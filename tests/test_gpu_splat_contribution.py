"""Splat contribution on the GPU (include/gsr.h gsr_set_splat_contribution), through the C-ABI with torch CUDA tensors as the caller's
buffers: every case of tests/variant_matrix drawn with the depth compositor plus contribution over three cameras into one buffer, bit for
bit against the contribution oracle, with rgba and depth unchanged; the state rules and refusals; the reset's ordering between
enqueued frames; the overflow re-render and GSR_FLAG_STATIC_CAPACITY; select_where and splat_histogram on the four properties against
numpy on the downloaded buffer; and the telescoping sum of the weights against the coverage alpha."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

from godotgaussiansplatting_b200 import _lib
from godotgaussiansplatting_b200.rasterizer import CONTRIBUTION_DTYPE, pack_instance_appearance, splat_filter, unpack_mask
from tests import contribution_reference as cref
from tests import variant_matrix as vm
from tests.gsr_direct import Ctx
from tests.scenes import make_scene
from tests.test_gpu_sh_degree import ShCtx, set_instances
from tests.test_gpu_splat_ids import last_frame_lists
from tests.test_gpu_variant_matrix import N, RAGGED, SIZE, flags_of, set_cutouts

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
bits = vm.bits


def ptr(t):
    return C.c_void_p(t.data_ptr())


def contrib_buffer(slots):
    t = torch.zeros(slots * 32, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    return t


def download(t):
    torch.cuda.synchronize()
    return t.cpu().numpy().view(CONTRIBUTION_DTYPE).copy()


def set_contrib(c, t, slots=None):
    return c.L.gsr_set_splat_contribution(c.h, None if t is None else ptr(t), c.max_splats if slots is None else slots)


def frames_of(c):
    n = C.c_uint32(0)
    _lib.check(c.L.gsr_splat_contribution_frames(c.h, C.byref(n)), "gsr_splat_contribution_frames")
    return int(n.value)


# ---- every variant-matrix case -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("i", range(len(vm.CASES)), ids=vm.IDS)
def test_case_with_contribution_is_the_reference(i):
    case = dataclasses.replace(vm.CASES[i], compositor="depth")
    fr = vm.frame_of(case, N, SIZE, RAGGED)
    ref = vm.reference(fr)
    ranges = [(f, k) for f, k, _ in fr.inst] if case.inst else None
    n_records = fr.drawn
    L = _lib.lib()
    want = cref.zeros(fr.n)
    with ShCtx(fr.n, fr.w, fr.h, case.store_bands, flags_of(case), factor=16) as c:
        c.upload(fr.splat60)
        if case.store_bands != case.bands:
            _lib.check(c.degree(case.bands - 1), "gsr_set_sh_degree")
        if case.aa:
            _lib.check(L.gsr_set_antialiasing(c.h, C.c_float(case.v)), "gsr_set_antialiasing")
        if case.dord:
            _lib.check(L.gsr_set_depth_order(c.h, _lib.GSR_DEPTH_ORDER_VIEW_DEPTH), "gsr_set_depth_order")
        if case.cut:
            set_cutouts(c, fr.vols)
        if case.inst:
            set_instances(c, fr.inst)
            if fr.app is not None:
                app = pack_instance_appearance(fr.app)
                _lib.check(L.gsr_set_instance_appearance(c.h, app, len(app)), "gsr_set_instance_appearance")
        Zt = None if fr.Z is None else torch.from_numpy(fr.Z).cuda()
        depth = torch.full((fr.h, fr.w), float("nan"), dtype=torch.float32, device="cuda")
        acc = contrib_buffer(fr.n)
        _lib.check(L.gsr_set_depth_compositing(c.h, None if Zt is None else ptr(Zt), ptr(depth)), "gsr_set_depth_compositing")
        _lib.check(set_contrib(c, acc), "gsr_set_splat_contribution")
        for k, frame in enumerate((25, 22, 28)):
            vp, ub = (fr.vp, fr.ub) if k == 0 else vm.camera(case, fr.w, fr.h, frame=frame)
            rgba = c.render(vp, ub, heatmap=1.0 if case.heat else 0.0)
            c.sync()
            if k == 0:   # the case's own camera: the frame is the composed reference's
                np.testing.assert_array_equal(bits(rgba), bits(ref["rgba"]))
                np.testing.assert_array_equal(bits(depth.cpu().numpy()), bits(ref["depth"]))
            recs, vals, bnds = last_frame_lists(c, n_records)
            cref.accumulate(want, recs, vals, bnds, fr.w, fr.h, vp, fr.Z, case.contract, ranges)
        got = download(acc)
        assert frames_of(c) == 3
    cref.assert_same(got, want)
    assert (got["pixels"] > 0).any()


# ---- the rules -----------------------------------------------------------------------------------------------------------------
def oracle_frame(c, n, vp, w, h, buf=None):
    recs, vals, bnds = last_frame_lists(c, n)
    return cref.accumulate(cref.zeros(n) if buf is None else buf, recs, vals, bnds, w, h, vp)


def test_state_and_argument_rules():
    n, w, h = 6000, 160, 120
    splat60, vp, ub = make_scene(n, 2, w, h, frame=13, scale_boost=0.5)
    with Ctx(n, w, h) as c:
        c.upload(splat60)
        L = c.L
        depth = torch.empty((h, w), dtype=torch.float32, device="cuda")
        scene = torch.full((h, w), float("inf"), dtype=torch.float32, device="cuda")
        motion = torch.empty((h, w, 2), dtype=torch.float32, device="cuda")
        ids = torch.empty((h, w, 2), dtype=torch.int32, device="cuda")
        a, b = contrib_buffer(n), contrib_buffer(n)
        assert set_contrib(c, a) == _lib.GSR_ERR_STATE                        # depth compositing is off
        assert L.gsr_reset_splat_contribution(c.h) == _lib.GSR_ERR_STATE      # no buffer
        f = splat_filter(_lib.GSR_PROP_CONTRIBUTION, 0.0, 1.0)
        assert L.gsr_select_where(c.h, C.byref(f), 1, -1, 0) == _lib.GSR_ERR_STATE
        _lib.check(L.gsr_set_depth_compositing(c.h, ptr(scene), ptr(depth)), "gsr_set_depth_compositing")
        assert set_contrib(c, a, n - 1) == _lib.GSR_ERR_INVALID               # slots != max_splats
        for bad in (depth, scene):
            assert set_contrib(c, bad) == _lib.GSR_ERR_INVALID                # aliases a plane
        _lib.check(L.gsr_set_motion_vectors(c.h, ptr(motion)), "gsr_set_motion_vectors")
        assert set_contrib(c, a) == _lib.GSR_ERR_STATE                        # motion vectors are on
        _lib.check(L.gsr_set_motion_vectors(c.h, None), "gsr_set_motion_vectors")
        _lib.check(L.gsr_set_splat_ids(c.h, ptr(ids)), "gsr_set_splat_ids")
        assert set_contrib(c, ids) == _lib.GSR_ERR_INVALID                    # aliases the ID plane
        assert set_contrib(c, a) == _lib.GSR_ERR_STATE                        # splat IDs are on
        _lib.check(L.gsr_set_splat_ids(c.h, None), "gsr_set_splat_ids")
        _lib.check(set_contrib(c, a), "gsr_set_splat_contribution")
        assert L.gsr_set_motion_vectors(c.h, ptr(motion)) == _lib.GSR_ERR_STATE   # and they refuse while it is on
        assert L.gsr_set_splat_ids(c.h, ptr(ids)) == _lib.GSR_ERR_STATE
        c.render(vp, ub)
        want = oracle_frame(c, n, vp, w, h)
        cref.assert_same(download(a), want)
        assert not download(b).view(np.uint8).any()
        st = c.stats()
        c.pick((st.tiles_y // 2) * st.tiles_x + st.tiles_x // 2)                # gsr_pick does not accumulate
        cref.assert_same(download(a), want)
        # NULL switches the mode off
        _lib.check(set_contrib(c, None), "gsr_set_splat_contribution")
        c.render(vp, ub)
        cref.assert_same(download(a), want)
        # depth compositing off switches it off, and so does gsr_resize
        _lib.check(set_contrib(c, a), "gsr_set_splat_contribution")
        _lib.check(L.gsr_set_depth_compositing(c.h, None, None), "gsr_set_depth_compositing")
        _lib.check(L.gsr_set_depth_compositing(c.h, None, ptr(depth)), "gsr_set_depth_compositing")
        c.render(vp, ub)
        cref.assert_same(download(a), want)
        _lib.check(set_contrib(c, a), "gsr_set_splat_contribution")
        c.resize(w, h)
        _lib.check(L.gsr_set_depth_compositing(c.h, None, ptr(depth)), "gsr_set_depth_compositing")
        c.render(vp, ub)
        cref.assert_same(download(a), want)


def test_reset_is_ordered_between_enqueued_frames():
    n, w, h = 6000, 160, 120
    splat60, vp0, ub0 = make_scene(n, 3, w, h, frame=10, scale_boost=0.5)
    _, vp1, ub1 = make_scene(n, 3, w, h, frame=40, scale_boost=0.5)
    with Ctx(n, w, h, factor=1000) as c:
        c.upload(splat60)
        depth = torch.empty((h, w), dtype=torch.float32, device="cuda")
        _lib.check(c.L.gsr_set_depth_compositing(c.h, None, ptr(depth)), "gsr_set_depth_compositing")
        acc = contrib_buffer(n)
        _lib.check(set_contrib(c, acc), "gsr_set_splat_contribution")
        c.render_async(vp0, ub0)
        c.render_async(vp1, ub1)
        _lib.check(c.L.gsr_reset_splat_contribution(c.h), "gsr_reset_splat_contribution")   # after both, before the next
        c.render_async(vp1, ub1)
        c.sync()
        assert frames_of(c) == 1
        cref.assert_same(download(acc), oracle_frame(c, n, vp1, w, h))


def test_overflow_rerender_is_counted_once():
    n, w, h = 6000, 160, 120
    splat60, vp, ub = make_scene(n, 2, w, h, frame=13, scale_boost=1.0)
    _, pvp, pub = make_scene(n, 2, w, h, frame=10, scale_boost=1.0)
    pvp[14] -= np.float32(40.0)   # far away: few pairs, the capacity stays small
    with Ctx(n, w, h, factor=1) as c:   # the second synchronous render overflows and is rendered again
        c.upload(splat60)
        depth = torch.empty((h, w), dtype=torch.float32, device="cuda")
        _lib.check(c.L.gsr_set_depth_compositing(c.h, None, ptr(depth)), "gsr_set_depth_compositing")
        acc = contrib_buffer(n)
        _lib.check(set_contrib(c, acc), "gsr_set_splat_contribution")
        c.render(pvp, pub)
        want = oracle_frame(c, n, pvp, w, h)
        m0 = c.stats().duplicates
        c.render(vp, ub)
        assert c.stats().capacity > 3 * m0, "the frame did not overflow"
        oracle_frame(c, n, vp, w, h, want)
        assert frames_of(c) == 2
        cref.assert_same(download(acc), want)


def test_static_capacity_adds_nothing():
    n, w, h = 6000, 160, 120
    splat60, vp, ub = make_scene(n, 2, w, h, frame=13, scale_boost=1.0)
    with ShCtx(n, w, h, 0, _lib.GSR_FLAG_STATIC_CAPACITY, factor=1) as c:
        c.upload(splat60)
        depth = torch.empty((h, w), dtype=torch.float32, device="cuda")
        _lib.check(c.L.gsr_set_depth_compositing(c.h, None, ptr(depth)), "gsr_set_depth_compositing")
        acc = contrib_buffer(n)
        _lib.check(set_contrib(c, acc), "gsr_set_splat_contribution")
        out = np.empty((h, w, 4), dtype=np.float32)
        rc = c.L.gsr_render(c.h, np.ascontiguousarray(vp, dtype=np.float32).ctypes.data_as(C.POINTER(C.c_float)), ub, 0.0,
                            C.c_void_p(out.ctypes.data))
        assert rc in (_lib.GSR_OK, _lib.GSR_ERR_OVERFLOW)
        assert c.stats().overflow, "the frame did not overflow its static capacity"
        assert frames_of(c) == 0
        assert not download(acc).view(np.uint8).any()


# ---- the properties and the telescoping sum ------------------------------------------------------------------------------------
def test_properties_and_telescoping_sum():
    n, w, h = 8000, 200, 150
    splat60, _, _ = make_scene(n, 4, w, h, frame=0, scale_boost=0.5)
    with Ctx(n, w, h, factor=64) as c:
        c.upload(splat60)
        L = c.L
        depth = torch.empty((h, w), dtype=torch.float32, device="cuda")
        _lib.check(L.gsr_set_depth_compositing(c.h, None, ptr(depth)), "gsr_set_depth_compositing")
        acc = contrib_buffer(n)
        _lib.check(set_contrib(c, acc), "gsr_set_splat_contribution")
        _lib.check(L.gsr_debug_pipeline(c.h, 1), "gsr_debug_pipeline")   # front / back overlap: the selections wait for the compositor
        prev = cref.zeros(n)
        for frame in (5, 20, 35):
            _, vp, ub = make_scene(n, 4, w, h, frame=frame, scale_boost=0.5)
            rgba = c.render(vp, ub)
            now = download(acc)
            # per view: sum of q(w) / 2^24 against sum of 1 - t (telescoping; each hit's w and q round by at most 2^-25 each)
            dw = (now["weight"] - prev["weight"]).astype(np.float64).sum() * 2.0 ** -24
            hits = float((now["pixels"] - prev["pixels"]).sum())
            cover = rgba[..., 3].astype(np.float64).sum()
            assert abs(dw - cover) <= (hits + w * h) * 2.0 ** -24, (dw, cover, hits)
            prev = now
        w_all = cref.prop_values(np.zeros((1, n, 4), np.float32), False, cref.CONTRIBUTION, None, prev)
        thr = float(np.quantile(w_all, 0.3))
        for filters in ([(cref.CONTRIBUTION, -np.inf, thr)], [(cref.PEAK, 0.05, 0.5), (cref.VIEWS, 2.0, 3.0)], [(cref.PIXELS, 10.0, np.inf)]):
            c.render_async(*make_scene(n, 4, w, h, frame=50, scale_boost=0.5)[1:])   # an enqueued frame the selection must follow
            arr = (_lib.GsrSplatFilter * len(filters))(*[splat_filter(*f) for f in filters])
            _lib.check(L.gsr_select_where(c.h, arr, len(filters), -1, _lib.GSR_SELECT_SET), "gsr_select_where")
            c.sync()
            buf = download(acc)
            sel = np.zeros(((n + 31) // 32,), dtype=np.uint32)
            hid = np.zeros_like(sel)
            u32p = C.POINTER(C.c_uint32)
            _lib.check(L.gsr_get_splat_masks(c.h, hid.ctypes.data_as(u32p), sel.ctypes.data_as(u32p), sel.size), "gsr_get_splat_masks")
            want = np.ones(n, dtype=bool)
            for prop, lo, hi in filters:
                v = cref.prop_values(np.zeros((1, n, 4), np.float32), False, prop, None, buf)
                want &= (np.float32(lo) <= v) & (v <= np.float32(hi))
            np.testing.assert_array_equal(unpack_mask(sel, n), want)
        for prop in cref.CONTRIB_PROPS:
            buf = download(acc)
            v = cref.prop_values(np.zeros((1, n, 4), np.float32), False, prop, None, buf)
            edges = np.unique(np.quantile(v, np.linspace(0.0, 1.0, 33)).astype(np.float32))
            if edges.size < 2:
                edges = np.array([0.0, 1.0], dtype=np.float32)
            counts = np.zeros(edges.size + 2, dtype=np.uint64)
            mm = np.zeros(2, dtype=np.float32)
            f = splat_filter(prop)
            fp = C.POINTER(C.c_float)
            _lib.check(L.gsr_splat_histogram(c.h, C.byref(f), -1, _lib.GSR_HISTOGRAM_KEPT, edges.ctypes.data_as(fp), edges.size - 1,
                                             counts.ctypes.data_as(C.POINTER(C.c_uint64)), mm.ctypes.data_as(fp)), "gsr_splat_histogram")
            want, (lo, hi) = cref.histogram_rule(np.zeros((1, n, 4), np.float32), False, None, None, 0, n, prop, edges, buf)
            np.testing.assert_array_equal(counts, want)
            assert (float(mm[0]), float(mm[1])) == (lo, hi)
