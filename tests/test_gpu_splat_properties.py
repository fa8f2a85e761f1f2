"""Splat property selection on the GPU (include/gsr.h "Splat property selection"), through the C-ABI: gsr_select_where and
gsr_splat_histogram on a 6 M-splat store of random words against the numpy rule of tests/property_reference bit for bit; instance
ranges; sequences mixed with region selections, hide, delete and duplicate; selections between asynchronous frames with and without
front / back overlap against frames of the same masks set directly; the single-context rule; the argument checks; the Python mirror."""
import ctypes as C

import numpy as np
import pytest

from godotgaussiansplatting_b200 import _lib
from tests import cutout_reference as cr
from tests import property_reference as pref
from tests import selection_reference as sref
from tests.test_gpu_cutouts import cloud, view
from tests.test_gpu_sh_degree import ShCtx, set_instances
from tests.test_gpu_splat_delete import count_of, delete, duplicate, masks_of, restore_host, store_of, stride_of
from tests.test_gpu_splat_selection import INST, LASSO, get_masks, polygon, set_masks, volume

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

F32, U32 = np.float32, np.uint32
FP, U64P = C.POINTER(C.c_float), C.POINTER(C.c_uint64)
INF = np.inf
W, H = 320, 200
N = 12288 - 77
INV, STATE = _lib.GSR_ERR_INVALID, _lib.GSR_ERR_STATE


def where(c, filters, op, instance=-1):
    arr = pref.filter_array(filters)
    return c.L.gsr_select_where(c.h, arr, len(filters), instance, op)


def hist(c, prop, edges, scope=_lib.GSR_HISTOGRAM_KEPT, instance=-1, rgb=(0.0, 0.0, 0.0)):
    f = pref.filter_array([(prop, 0.0, 0.0, rgb)])
    e = np.ascontiguousarray(edges, dtype=F32)
    counts = np.zeros(e.size + 2, dtype=np.uint64)
    mm = np.zeros(2, dtype=F32)
    rc = c.L.gsr_splat_histogram(c.h, f, instance, scope, e.ctypes.data_as(FP), e.size - 1, counts.ctypes.data_as(U64P), mm.ctypes.data_as(FP))
    return rc, counts, (float(mm[0]), float(mm[1]))


def assert_hist(got, want, msg=""):
    rc, counts, mm = got
    assert rc == _lib.GSR_OK, _lib.lib().gsr_last_error()
    np.testing.assert_array_equal(counts, want[0], err_msg=msg)
    assert np.array(mm, F32).view(U32).tolist() == np.array(want[1], F32).view(U32).tolist(), (msg, mm, want[1])


def quantile_edges(v, bins, lo=0.05, hi=0.95):
    fin = v[np.isfinite(v)]
    return np.unique(np.quantile(fin, np.linspace(lo, hi, bins + 1)).astype(F32))


# ---- a 6 M-splat store of random words ---------------------------------------------------------------------------------------
C3 = 6_000_000


@pytest.mark.parametrize("half", [False, True])
def test_full_size_is_the_rule(half):
    m = C3 + 77
    n = C3 - 13
    rng = np.random.default_rng(11 + half)
    with ShCtx(m, 64, 64, 4, _lib.GSR_FLAG_SH_HALF if half else 0) as c:
        nbytes = int(c.L.gsr_splat_store_bytes(c.h))
        store = rng.integers(0, 2 ** 32, size=nbytes // 4, dtype=U32).view(F32).reshape(-1, stride_of(m), 4)
        restore_host(c, store)
        _lib.check(c.L.gsr_set_splat_count(c.h, n), "count")
        hid, sel = rng.random(m) < 0.2, rng.random(m) < 0.3
        sel &= ~hid
        _lib.check(set_masks(c, hid, sel), "masks")
        rgb = (0.3, 0.5, 0.7)
        vals = {p: pref.values(store, half, p, rgb) for p in pref.PROPS}
        sets = []
        for p in pref.PROPS:
            fin = vals[p][:n][np.isfinite(vals[p][:n])]
            lo, hi = np.quantile(fin, [0.3, 0.6]).astype(F32)
            sets.append([(p, lo, hi, rgb)])
        sets.append([(pref.OPACITY, -INF, 0.0, rgb), (pref.SIZE, 0.0, INF, rgb), (pref.COLOR, 0.0, 1e30, rgb)])
        for i, f in enumerate(sets):
            for op in range(4):
                _lib.check(where(c, f, op), "where")
                sel = pref.where_rule(store, half, hid, sel, 0, n, f, op)
                gh, gs = masks_of(c)
                np.testing.assert_array_equal(gh, hid)
                np.testing.assert_array_equal(gs, sel, err_msg=f"set {i} op {op}")
            assert 1000 < pref.where_inside(store, half, 0, n, f).sum() < n - 1000
        for p in pref.PROPS:
            for bins in (1, 256, 1024):
                e = quantile_edges(vals[p][:n], bins)
                for scope in (0, 1):
                    assert_hist(hist(c, p, e, scope, rgb=rgb), pref.histogram_rule(store, half, hid, sel, 0, n, p, rgb, e, scope),
                                f"prop {p} bins {bins} scope {scope}")
        store[2, :, 2] = 1.0   # a saturated property: every opacity in the last bin
        restore_host(c, store)
        e = np.linspace(0.0, 1.0, 257).astype(F32)
        want = pref.histogram_rule(store, half, hid, sel, 0, n, pref.OPACITY, rgb, e, 0)
        assert want[0][255] > C3 // 2
        assert_hist(hist(c, pref.OPACITY, e), want, "saturated")


# ---- instances, sequences, frames ---------------------------------------------------------------------------------------------
def test_instance_ranges():
    splat60 = cloud(N)
    with ShCtx(N + 100, W, H) as c:
        c.upload(splat60)
        set_instances(c, INST + [(N - 40, 100, INST[0][2])])   # the last range reaches past the cloud
        store = store_of(c)
        n = count_of(c)
        assert n == N
        hid = np.zeros(N + 100, bool)
        sel = np.zeros(N + 100, bool)
        f = [(pref.OPACITY, 0.3, 0.9, (0, 0, 0)), (pref.ISOTROPY, 0.05, 1.0, (0, 0, 0))]
        e = np.linspace(0.0, 1.0, 33).astype(F32)
        for k, (first, count, _) in enumerate(INST + [(N - 40, 100, None)]):
            cnt = max(0, min(count, n - first))
            op = [sref.SET, sref.ADD, sref.TOGGLE, sref.SUBTRACT, sref.ADD][k]
            _lib.check(where(c, f, op, k), "where")
            sel = pref.where_rule(store, False, hid, sel, first, cnt, f, op)
            np.testing.assert_array_equal(get_masks(c)[1], sel, err_msg=f"instance {k}")
            assert_hist(hist(c, pref.OPACITY, e, instance=k), pref.histogram_rule(store, False, hid, sel, first, cnt, pref.OPACITY,
                                                                                   (0, 0, 0), e, 0))
        assert sel.sum() > 100
        assert where(c, f, 0, len(INST) + 1) == INV


def test_sequences_with_regions_hide_delete_duplicate():
    """Each step changes the store, the masks or the count; select_where and the histogram after it equal the rule on what the
    device holds then."""
    splat60 = cloud(N)
    vp, _ = view()
    M = N + 4000
    with ShCtx(M, W, H, 0, _lib.GSR_FLAG_SH_HALF) as c:
        c.upload(splat60)
        f_small = [(pref.SIZE, -INF, 2e-4, (0, 0, 0))]
        f_col = [(pref.COLOR, 0.0, 0.08, (0.6, 0.5, 0.4)), (pref.OPACITY, 0.2, INF, (0, 0, 0))]
        e = np.geomspace(1e-6, 1.0, 65).astype(F32)
        steps = [("poly", lambda: polygon(c, vp, LASSO, sref.SET)), ("where", f_small, sref.ADD),
                 ("vol", lambda: volume(c, cr.box([0.0, 0.1, 2.4], [0.3, 0.5, 0.3]), sref.SUBTRACT)), ("where", f_col, sref.TOGGLE),
                 ("hide", None), ("where", f_small, sref.SET), ("delete", None), ("where", f_col, sref.ADD), ("dup", None),
                 ("where", f_small, sref.SUBTRACT), ("where", f_col, sref.SET)]
        for i, step in enumerate(steps):
            kind = step[0]
            if kind in ("poly", "vol"):
                _lib.check(step[1](), kind)
            elif kind == "hide":
                _lib.check(c.L.gsr_hide_selection(c.h), "hide")
            elif kind == "delete":
                assert delete(c)[0] == _lib.GSR_OK
            elif kind == "dup":
                assert duplicate(c)[0] == _lib.GSR_OK
            else:
                store, (hid, sel), n = store_of(c), masks_of(c), count_of(c)
                _lib.check(where(c, step[1], step[2]), "where")
                want = pref.where_rule(store, True, hid, sel, 0, n, step[1], step[2])
                np.testing.assert_array_equal(masks_of(c)[1], want, err_msg=f"step {i}")
            store, (hid, sel), n = store_of(c), masks_of(c), count_of(c)
            for scope in (0, 1):
                assert_hist(hist(c, pref.SIZE, e, scope), pref.histogram_rule(store, True, hid, sel, 0, n, pref.SIZE, (0, 0, 0), e, scope),
                            f"step {i} scope {scope}")
        assert 0 < count_of(c) < M


@pytest.mark.parametrize("pipeline", [0, 1])
def test_selections_between_asynchronous_frames(pipeline):
    """select_where and hide_selection between asynchronous frames: each frame equals the frame of the same masks set directly."""
    splat60 = cloud(N)
    vp, ub = view()
    with ShCtx(N, W, H) as c, ShCtx(N, W, H) as d:
        c.upload(splat60)
        d.upload(splat60)
        store = store_of(c)
        _lib.check(c.L.gsr_debug_pipeline(c.h, pipeline), "pipeline")
        outs = [torch.zeros((H, W, 4), dtype=torch.float32, device="cuda") for _ in range(5)]
        torch.cuda.synchronize()
        hid, sel = np.zeros(N, bool), np.zeros(N, bool)
        states = []
        ops = [("where", [(pref.OPACITY, 0.0, 0.5, (0, 0, 0))], sref.SET), ("hide",),
               ("where", [(pref.SIZE, 1e-3, INF, (0, 0, 0)), (pref.ISOTROPY, -INF, 0.5, (0, 0, 0))], sref.ADD),
               ("where", [(pref.COLOR, 0.0, 0.1, (0.5, 0.5, 0.5))], sref.TOGGLE), ("hide",)]
        for i, o in enumerate(ops):
            if o[0] == "hide":
                _lib.check(c.L.gsr_hide_selection(c.h), "hide")
                hid, sel = hid | sel, np.zeros(N, bool)
            else:
                _lib.check(where(c, o[1], o[2]), "where")
                sel = pref.where_rule(store, False, hid, sel, 0, N, o[1], o[2])
            _lib.check(c.L.gsr_set_framebuffer_external(c.h, C.c_void_p(outs[i].data_ptr())), "fb")
            c.render_async(vp, ub)
            states.append((hid.copy(), sel.copy()))
        c.sync()
        for i, (h_, s_) in enumerate(states):
            _lib.check(set_masks(d, h_, s_), "masks")
            want = d.render(vp, ub)
            np.testing.assert_array_equal(outs[i].cpu().numpy().view(U32), np.ascontiguousarray(want).view(U32), err_msg=f"frame {i}")
        assert states[-1][0].sum() > 500


# ---- state rules and arguments --------------------------------------------------------------------------------------------------
def test_single_context_rule_and_masks_out_of_use():
    splat60 = cloud(N)
    with ShCtx(N, W, H) as c:
        c.upload(splat60)
        store = store_of(c)
        e = np.linspace(0.0, 1.0, 17).astype(F32)
        none = np.zeros(N, bool)
        want = pref.histogram_rule(store, False, None, None, 0, N, pref.OPACITY, (0, 0, 0), e, 0)
        assert_hist(hist(c, pref.OPACITY, e), want, "masks not in use")
        nothing = hist(c, pref.OPACITY, e, _lib.GSR_HISTOGRAM_SELECTED)
        assert not nothing[1].any() and nothing[2] == (INF, -INF)
        c.set_band(0, 3)   # the histogram left the masks out of use, or the band would be refused
        assert where(c, [(pref.OPACITY, 0.0, 1.0, (0, 0, 0))], sref.SET) == STATE
        assert_hist(hist(c, pref.OPACITY, e), want, "sharded")
        gh, gs = get_masks(c)
        assert not gh.any() and not gs.any()
        c.set_band(0, (H + 15) // 16)
        _lib.check(where(c, [(pref.OPACITY, 0.0, 0.5, (0, 0, 0))], sref.SET), "where")
        assert c.L.gsr_set_band(c.h, 0, 3) == STATE   # now the masks are in use
        sel = pref.where_rule(store, False, none, none, 0, N, [(pref.OPACITY, 0.0, 0.5, (0, 0, 0))], sref.SET)
        assert_hist(hist(c, pref.OPACITY, e, _lib.GSR_HISTOGRAM_SELECTED),
                    pref.histogram_rule(store, False, none, sel, 0, N, pref.OPACITY, (0, 0, 0), e, 1))
        _lib.check(c.L.gsr_clear_splat_masks(c.h), "clear")
        nothing = hist(c, pref.OPACITY, e, _lib.GSR_HISTOGRAM_SELECTED)
        assert not nothing[1].any()


def test_argument_checks_keep_the_state():
    splat60 = cloud(N)
    with ShCtx(N, W, H) as c:
        c.upload(splat60)
        ok = [(pref.OPACITY, 0.0, 0.5, (0, 0, 0))]
        _lib.check(where(c, ok, sref.SET), "where")
        before = get_masks(c)
        L = c.L
        assert L.gsr_select_where(c.h, None, 1, -1, 0) == INV
        arr = pref.filter_array(ok * 9)
        assert L.gsr_select_where(c.h, arr, 0, -1, 0) == INV
        assert L.gsr_select_where(c.h, arr, 9, -1, 0) == INV
        for bad in ([(5, 0.0, 1.0, (0, 0, 0))], [(-1, 0.0, 1.0, (0, 0, 0))], [(pref.OPACITY, np.nan, 1.0, (0, 0, 0))],
                    [(pref.OPACITY, 0.0, np.nan, (0, 0, 0))], [(pref.COLOR, 0.0, 1.0, (0.0, np.inf, 0.0))],
                    [(pref.COLOR, 0.0, 1.0, (np.nan, 0.0, 0.0))]):
            assert where(c, ok + bad, sref.SET) == INV, bad
        assert where(c, ok, 4) == INV and where(c, ok, -1) == INV
        assert where(c, ok, sref.SET, instance=0) == INV and where(c, ok, sref.SET, instance=-2) == INV
        _lib.check(where(c, [(pref.OPACITY, -INF, INF, (np.nan, 0, 0))], sref.ADD), "rgb ignored outside colour")
        _lib.check(where(c, [(pref.OPACITY, -INF, INF, (0, 0, 0))], sref.SUBTRACT), "undo")
        after = get_masks(c)
        np.testing.assert_array_equal(after[1], before[1] & False)
        _lib.check(where(c, ok, sref.SET), "where")
        np.testing.assert_array_equal(get_masks(c)[1], before[1])
        e = np.linspace(0.0, 1.0, 5).astype(F32)
        counts = np.full(8, 7, dtype=np.uint64)
        f = pref.filter_array(ok)
        ep = e.ctypes.data_as(FP)
        cp = counts.ctypes.data_as(U64P)
        assert L.gsr_splat_histogram(c.h, None, -1, 0, ep, 4, cp, None) == INV
        assert L.gsr_splat_histogram(c.h, f, -1, 0, None, 4, cp, None) == INV
        assert L.gsr_splat_histogram(c.h, f, -1, 0, ep, 4, None, None) == INV
        assert L.gsr_splat_histogram(c.h, f, -1, 0, ep, 0, cp, None) == INV
        big = np.arange(1026, dtype=F32)
        assert L.gsr_splat_histogram(c.h, f, -1, 0, big.ctypes.data_as(FP), 1025, cp, None) == INV
        for bad_e in ([0, 1, 1, 2, 3], [0, 2, 1, 3, 4], [0, 1, np.inf, 3, 4], [np.nan, 1, 2, 3, 4]):
            be = np.array(bad_e, F32)
            assert L.gsr_splat_histogram(c.h, f, -1, 0, be.ctypes.data_as(FP), 4, cp, None) == INV, bad_e
        assert hist(c, 7, e)[0] == INV
        assert hist(c, pref.OPACITY, e, scope=2)[0] == INV
        assert hist(c, pref.OPACITY, e, instance=0)[0] == INV
        assert hist(c, pref.COLOR, e, rgb=(0, 0, np.inf))[0] == INV
        assert (counts == 7).all()
        assert hist(c, pref.OPACITY, e)[0] == _lib.GSR_OK   # minmax may be NULL:
        assert L.gsr_splat_histogram(c.h, f, -1, 0, ep, 4, cp, None) == _lib.GSR_OK
        np.testing.assert_array_equal(get_masks(c)[1], before[1])


def test_python_mirror():
    from godotgaussiansplatting_b200 import camera as cam
    from godotgaussiansplatting_b200.rasterizer import GaussianSplattingRasterizer, splat_filter
    from godotgaussiansplatting_b200.synthetic import synthetic_ply
    r = GaussianSplattingRasterizer(synthetic_ply(3001, 4), (160, 96), None, cam.orbit_camera(25, aspect=160 / 96))
    r.init_gpu()
    try:
        counts, below, above, nan, (lo, hi) = r.splat_histogram(_lib.GSR_PROP_OPACITY, np.linspace(0.0, 1.0, 11))
        assert int(counts.sum()) + below + above + nan == 3001 and lo <= hi
        below_half = float(np.nextafter(F32(0.5), F32(0.0)))   # v <= below_half <=> v < 0.5, the edge of bin 5
        r.select_where([(_lib.GSR_PROP_OPACITY, -np.inf, below_half), splat_filter(_lib.GSR_PROP_SIZE, 0.0, np.inf)])
        s, h = r.selection_counts()
        assert s == int(counts[:5].sum()) + below and h == 0
        r.hide_selection()
        kept = r.splat_histogram(_lib.GSR_PROP_OPACITY, np.linspace(0.0, 1.0, 11))
        assert int(kept[0].sum()) + kept[1] + kept[2] + kept[3] == 3001 - s
        r.select_where([(_lib.GSR_PROP_COLOR_DISTANCE, 0.0, 3.0, (0.5, 0.5, 0.5))], _lib.GSR_SELECT_ADD)
        sel = r.splat_histogram(_lib.GSR_PROP_OPACITY, np.linspace(0.0, 1.0, 11), _lib.GSR_HISTOGRAM_SELECTED)
        assert int(sel[0].sum()) + sel[1] + sel[2] + sel[3] == r.selection_counts()[0] > 0
        r.rasterize()
    finally:
        r.cleanup_gpu()
