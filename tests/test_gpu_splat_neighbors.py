"""Splat neighbourhood selection on the GPU (include/gsr.h "Splat neighbourhood selection"), through the C-ABI: every mode under every
op on a 6 M-splat cloud with planted floaters and small clumps, float and binary16 stores, against the serial C++ grid reference of
tests/neighbor_reference bit for bit (masks and stats); an instance range; a sequence of lasso, select_where, neighbourhood, hide, delete
and duplicate with the rule checked after every step; selections between asynchronous frames with and without front / back overlap
against frames of the same masks set directly; the single-context rule, the budget and the argument checks; the Python mirror."""
import ctypes as C
import time

import numpy as np
import pytest

from godotgaussiansplatting_b200 import _lib
from tests import neighbor_reference as nr
from tests import property_reference as pref
from tests import selection_reference as sref
from tests.test_gpu_cutouts import cloud, view
from tests.test_gpu_sh_degree import ShCtx, set_instances
from tests.test_gpu_splat_delete import bits, count_of, delete, duplicate, masks_of, restore_host, store_of, stride_of
from tests.test_gpu_splat_selection import INST, LASSO, polygon, set_masks

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

F32 = np.float32
W, H = 320, 200
N = 12288 - 77
INV, STATE = _lib.GSR_ERR_INVALID, _lib.GSR_ERR_STATE


def neighborhood(c, mode, radius, count=1, op=sref.SET, instance=-1):
    q = _lib.GsrNeighborhood(mode, radius, count, instance)
    st = _lib.GsrNeighborhoodStats()
    rc = c.L.gsr_select_neighborhood(c.h, C.byref(q), op, C.byref(st))
    return rc, [st.participants, st.inside, st.candidates, st.clusters, st.largest_cluster]


def plane0_of(store, n=None):
    p = np.ascontiguousarray(store[0], dtype=F32)
    if n is not None:
        p = p.copy()
        p[n:, :3] = np.nan   # past the cloud: never tested (the range is bounded by n)
    return p


# ---- a 6 M-splat cloud with floaters and clumps ---------------------------------------------------------------------------------
C3 = 6_000_000


def c3_positions(rng, m, n):
    """A shell of radius 5 and thickness 0.1 (about 8 neighbours within 0.02), 3000 floaters in a box of 30, 400 clumps of 3..60."""
    p = np.zeros((m, 3), F32)
    k_fl, clumps = 3000, [int(x) for x in rng.integers(3, 60, 400)]
    body = n - k_fl - sum(clumps)
    d = rng.normal(size=(body, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    pts = [d * rng.uniform(4.95, 5.05, (body, 1)), rng.uniform(-15, 15, (k_fl, 3))]
    for k in clumps:
        pts.append(rng.uniform(-15, 15, 3) + rng.normal(size=(k, 3)) * 0.01)
    pts = np.concatenate(pts).astype(F32)
    p[:n] = pts[rng.permutation(n)]
    return p


@pytest.fixture(scope="module")
def c3_cloud():
    rng = np.random.default_rng(31)
    m, n = C3 + 77, C3 - 13
    xyz = c3_positions(rng, m, n)
    hid = rng.random(m) < 0.02
    sel = (rng.random(m) < 0.0005) & ~hid
    hid[n:] = sel[n:] = False
    plane0 = np.zeros((m, 4), F32)
    plane0[:, :3] = xyz
    plane0[n:, :3] = np.nan
    refs = {md: (0.02, 3, inside[:m], st) for md, (inside, st) in nr.ref_all_modes(plane0, hid, sel, 0, n, 0.02, 3).items()}
    return m, n, xyz, hid, sel, refs


@pytest.mark.parametrize("half", [False, True])
def test_full_size_is_the_reference(half, c3_cloud):
    m, n, xyz, hid, sel, refs = c3_cloud
    with ShCtx(m, 64, 64, 4, _lib.GSR_FLAG_SH_HALF if half else 0) as c:
        nbytes = int(c.L.gsr_splat_store_bytes(c.h))
        store = np.zeros(nbytes // 4, dtype=F32).reshape(-1, stride_of(m), 4)
        store[0, :m, :3] = xyz
        restore_host(c, store)
        _lib.check(c.L.gsr_set_splat_count(c.h, n), "count")
        for mode, (radius, thr, inside, want_st) in refs.items():
            for op in range(4):
                _lib.check(set_masks(c, hid, sel), "masks")
                rc, st = neighborhood(c, mode, radius, thr, op)
                assert rc == _lib.GSR_OK, _lib.lib().gsr_last_error()
                gh, gs = masks_of(c)
                np.testing.assert_array_equal(gh, hid)
                np.testing.assert_array_equal(gs, sref.combine(op, sel, inside, hid), err_msg=f"mode {mode} op {op}")
                assert st == want_st, (mode, op, st, want_st)
        assert 3000 <= refs[nr.SPARSE][3][1] < C3 // 4            # the floaters and the sparsest shell splats
        assert refs[nr.SMALL][3][3] > 400 and refs[nr.SMALL][3][1] > 3000


# ---- instances, sequences, frames ---------------------------------------------------------------------------------------------
def small_store(c):
    store = store_of(c)
    return store, count_of(c)


def test_instance_range():
    splat60 = cloud(N)
    with ShCtx(N + 100, W, H) as c:
        c.upload(splat60)
        set_instances(c, INST + [(N - 40, 100, INST[0][2])])
        store, n = small_store(c)
        hid = np.zeros(N + 100, bool)
        sel = np.zeros(N + 100, bool)
        sel[::97] = True
        _lib.check(set_masks(c, hid, sel), "masks")
        p0 = plane0_of(store, n)
        for k, (first, count, _) in enumerate(INST + [(N - 40, 100, None)]):
            cnt = max(0, min(count, n - first))
            for mode in nr.MODES:
                op = [sref.SET, sref.ADD, sref.TOGGLE, sref.SUBTRACT][mode]
                want, wst = nr.select_rule(p0, hid, sel, first, cnt, 0.05, mode, 3, op)
                rc, st = neighborhood(c, mode, 0.05, 3, op, k)
                assert rc == _lib.GSR_OK, _lib.lib().gsr_last_error()
                sel = want
                np.testing.assert_array_equal(masks_of(c)[1], sel, err_msg=f"instance {k} mode {mode}")
                assert st == wst


def test_sequence_with_other_edits():
    """Lasso, select_where, neighbourhoods, hide, delete and duplicate, the rule after every step."""
    splat60 = cloud(N)
    vp, _ = view()
    m = 2 * N
    with ShCtx(m, W, H) as c:
        c.upload(splat60)
        hid = np.zeros(m, bool)
        sel = np.zeros(m, bool)

        def check_step(what):
            gh, gs = masks_of(c)
            np.testing.assert_array_equal(gh, hid, err_msg=what)
            np.testing.assert_array_equal(gs, sel, err_msg=what)

        _lib.check(polygon(c, vp, LASSO, sref.SET), "lasso")
        hid, sel = masks_of(c)
        for step, (mode, radius, thr, op) in enumerate([(nr.GROW, 0.05, 1, sref.SET), (nr.SPARSE, 0.04, 2, sref.ADD),
                                                        (nr.SPARSE, 0.04, 4, sref.SET), (nr.CONNECTED, 0.03, 1, sref.ADD),
                                                        (nr.SMALL, 0.03, 50, sref.TOGGLE)]):
            store, n = small_store(c)
            want, wst = nr.select_rule(plane0_of(store, n), hid, sel, 0, n, radius, mode, thr, op)
            rc, st = neighborhood(c, mode, radius, thr, op)
            assert rc == _lib.GSR_OK and st == wst, (step, st, wst)
            sel = want
            check_step(f"step {step}")
            if step == 0:
                f = pref.filter_array([(pref.OPACITY, 0.0, 0.5, (0, 0, 0))])
                _lib.check(c.L.gsr_select_where(c.h, f, 1, -1, sref.SUBTRACT), "where")
                sel = pref.where_rule(store, False, hid, sel, 0, n, [(pref.OPACITY, 0.0, 0.5, (0, 0, 0))], sref.SUBTRACT)
                check_step("where")
            if step == 1:
                _lib.check(c.L.gsr_hide_selection(c.h), "hide")
                hid, sel = hid | sel, np.zeros(m, bool)
                check_step("hide")
                rc, k = delete(c)
                assert rc == _lib.GSR_OK
                hid, sel = masks_of(c)
                assert not hid.any() and count_of(c) == k
            if step == 2:
                rc, S = duplicate(c)
                assert rc == _lib.GSR_OK and S == int(sel.sum()) > 0
                hid, sel = masks_of(c)


@pytest.mark.parametrize("pipeline", [0, 1])
def test_selections_between_asynchronous_frames(pipeline):
    splat60 = cloud(N)
    vp, ub = view()
    m = N + 300
    with ShCtx(m, W, H) as c, ShCtx(m, W, H) as r:
        for x in (c, r):
            x.upload(splat60)
        _lib.check(c.L.gsr_debug_pipeline(c.h, pipeline), "pipeline")
        sel0 = np.zeros(m, bool)
        sel0[::151] = True
        _lib.check(set_masks(c, np.zeros(m, bool), sel0), "masks")
        host = [torch.empty((H, W, 4), dtype=torch.float32).pin_memory() for _ in range(4)]
        want = []
        steps = [(nr.GROW, 0.05, 1, sref.SET), (nr.CONNECTED, 0.03, 1, sref.ADD), (nr.SMALL, 0.03, 30, sref.SET)]
        for i, (mode, radius, thr, op) in enumerate(steps):
            c.render_async(vp, ub, host_ptr=host[i].data_ptr())
            rc, _ = neighborhood(c, mode, radius, thr, op)
            assert rc == _lib.GSR_OK
            if i == 1:
                _lib.check(c.L.gsr_hide_selection(c.h), "hide")
        c.render_async(vp, ub, host_ptr=host[3].data_ptr())
        c.sync()
        torch.cuda.synchronize()
        # the second context: the masks each frame saw, set directly
        store, n = small_store(r)
        p0 = plane0_of(store, n)
        hid, sel = np.zeros(m, bool), sel0.copy()
        _lib.check(set_masks(r, hid, sel), "masks")
        want.append(r.render(vp, ub))
        for i, (mode, radius, thr, op) in enumerate(steps):
            sel, _ = nr.select_rule(p0, hid, sel, 0, n, radius, mode, thr, op)
            if i == 1:
                hid, sel = hid | sel, np.zeros(m, bool)
            _lib.check(set_masks(r, hid, sel), "masks")
            want.append(r.render(vp, ub))
        np.testing.assert_array_equal(masks_of(c)[0], hid)
        np.testing.assert_array_equal(masks_of(c)[1], sel)
        for i in range(4):
            np.testing.assert_array_equal(bits(host[i].numpy()), bits(want[i]), err_msg=f"frame {i}")


# ---- refusals ----------------------------------------------------------------------------------------------------------------
def test_refusals():
    splat60 = cloud(N)
    with ShCtx(N, W, H) as c:
        c.upload(splat60)
        q = _lib.GsrNeighborhood(nr.SPARSE, 0.05, 1, -1)
        L = c.L
        assert L.gsr_select_neighborhood(c.h, None, 0, None) == INV
        for bad in [(7, 0.05, 1, -1), (-1, 0.05, 1, -1), (0, float("nan"), 1, -1), (0, float("inf"), 1, -1), (0, 0.0, 1, -1),
                    (0, -1.0, 1, -1), (0, 2.0 ** -61, 1, -1), (0, 2.0 ** 61, 1, -1), (0, 0.05, 0, -1), (3, 0.05, 0, -1), (0, 0.05, 1, 0),
                    (0, 0.05, 1, -2)]:
            assert L.gsr_select_neighborhood(c.h, C.byref(_lib.GsrNeighborhood(*bad)), 0, None) == INV, bad
        assert L.gsr_select_neighborhood(c.h, C.byref(q), 4, None) == INV
        # the order: mode before radius before count before op before instance
        assert L.gsr_select_neighborhood(c.h, C.byref(_lib.GsrNeighborhood(9, float("nan"), 0, 5)), 9, None) == INV
        assert b"mode" in L.gsr_last_error()
        assert L.gsr_select_neighborhood(c.h, C.byref(_lib.GsrNeighborhood(0, float("nan"), 0, 5)), 9, None) == INV
        assert b"radius" in L.gsr_last_error()
        assert L.gsr_select_neighborhood(c.h, C.byref(_lib.GsrNeighborhood(0, 1.0, 0, 5)), 9, None) == INV
        assert b"count" in L.gsr_last_error()
        assert L.gsr_select_neighborhood(c.h, C.byref(_lib.GsrNeighborhood(1, 1.0, 0, 5)), 9, None) == INV
        assert b"op" in L.gsr_last_error()
        assert L.gsr_select_neighborhood(c.h, C.byref(_lib.GsrNeighborhood(1, 1.0, 0, 5)), 0, None) == INV
        assert b"instance" in L.gsr_last_error()
        gh, gs = masks_of(c)
        assert not gh.any() and not gs.any()
        # the single-context rule
        c.set_band(0, 3)
        assert neighborhood(c, nr.SPARSE, 0.05)[0] == STATE
        c.set_band(0, (H + 15) // 16)


def test_over_budget_is_refused_quickly():
    m = C3
    rng = np.random.default_rng(5)
    with ShCtx(m, 64, 64, 1) as c:
        nbytes = int(c.L.gsr_splat_store_bytes(c.h))
        store = np.zeros(nbytes // 4, dtype=F32).reshape(-1, stride_of(m), 4)
        store[0, :m, :3] = rng.uniform(-1, 1, (m, 3)).astype(F32)
        restore_host(c, store)
        _lib.check(c.L.gsr_set_splat_count(c.h, m), "count")
        hid = np.zeros(m, bool)
        sel = rng.random(m) < 0.01
        _lib.check(set_masks(c, hid, sel), "masks")
        assert neighborhood(c, nr.SPARSE, 0.01)[0] == _lib.GSR_OK   # warm
        _lib.check(set_masks(c, hid, sel), "masks")
        t0 = time.perf_counter()
        rc, _ = neighborhood(c, nr.GROW, 100.0)
        dt = time.perf_counter() - t0
        assert rc == INV
        msg = _lib.lib().gsr_last_error().decode()
        assert str(m * m) in msg, msg
        assert dt < 1.0, dt
        gh, gs = masks_of(c)
        np.testing.assert_array_equal(gs, sel)
        assert not gh.any()


# ---- the Python mirror -----------------------------------------------------------------------------------------------------------
def test_python_mirror():
    from godotgaussiansplatting_b200 import camera as cam
    from godotgaussiansplatting_b200.rasterizer import GaussianSplattingRasterizer
    from godotgaussiansplatting_b200.synthetic import synthetic_ply
    r = GaussianSplattingRasterizer(synthetic_ply(3001, 4), (160, 96), None, cam.orbit_camera(25, aspect=160 / 96))
    r.init_gpu()
    try:
        st = r.select_neighborhood(_lib.GSR_NEIGHBOR_SMALL_CLUSTERS, 0.05, count=10)
        assert st["participants"] == 3001 and st["clusters"] >= 1 and st["largest_cluster"] >= 1
        assert r.selection_counts()[0] == st["inside"]
        keep = r.select_neighborhood(_lib.GSR_NEIGHBOR_SMALL_CLUSTERS, 0.05, count=st["largest_cluster"])
        assert keep["inside"] <= 3001 - st["largest_cluster"] and keep["clusters"] == st["clusters"]
        r.hide_selection()
        grow = r.select_neighborhood(_lib.GSR_NEIGHBOR_SPARSE, 0.05, count=1)
        assert grow["participants"] == 3001 - keep["inside"] and grow["clusters"] == 0
        r.rasterize()
    finally:
        r.cleanup_gpu()
