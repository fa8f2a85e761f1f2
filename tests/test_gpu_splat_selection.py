"""Splat selection on the GPU (include/gsr.h "Splat selection"), through the C-ABI: the selection kernels against the numpy rules of
tests/selection_reference bit for bit, frames with masks against the composed reference (RGBA, stats, pairs, records), the ordering of
operations between frames with and without front / back overlap, select-what-you-see on the library's own ID plane, get / set / counts,
masks across uploads, resizes and instance layouts, the single-context rule, the argument checks, and the default path once cleared."""
import ctypes as C

import numpy as np
import pytest

from godotgaussiansplatting_b200 import _lib
from godotgaussiansplatting_b200.rasterizer import pack_mask, splat_sources, unpack_mask
from tests import cutout_reference as cr
from tests import ortho_reference as oref
from tests import selection_reference as sref
from tests.gsr_direct import REC_DTYPE
from tests.test_gpu_cutouts import check, cloud, cutouts, default_frame, view
from tests.test_cutouts import crop_set
from tests.test_gpu_sh_degree import ShCtx, set_instances
from tests.test_instances import SCALED, rigid

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

W, H = 320, 200
N = 12288 - 77   # not a multiple of 32
FP = C.POINTER(C.c_float)
U32P = C.POINTER(C.c_uint32)


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def seeded_masks(n, seed, hidden=0.3, selected=0.1):
    rng = np.random.default_rng(seed)
    hid = rng.random(n) < hidden
    sel = (rng.random(n) < selected) & ~hid
    return hid, sel


def set_masks(c, hid, sel):
    h, s = pack_mask(hid, c.max_splats), pack_mask(sel, c.max_splats)
    return c.L.gsr_set_splat_masks(c.h, h.ctypes.data_as(U32P), s.ctypes.data_as(U32P), h.size)


def get_masks(c):
    words = (c.max_splats + 31) // 32
    h, s = np.zeros(words, np.uint32), np.zeros(words, np.uint32)
    _lib.check(c.L.gsr_get_splat_masks(c.h, h.ctypes.data_as(U32P), s.ctypes.data_as(U32P), words), "gsr_get_splat_masks")
    return unpack_mask(h, c.max_splats), unpack_mask(s, c.max_splats)


def counts(c):
    s, h = C.c_uint64(0), C.c_uint64(0)
    _lib.check(c.L.gsr_splat_mask_counts(c.h, C.byref(s), C.byref(h)), "gsr_splat_mask_counts")
    return int(s.value), int(h.value)


def polygon(c, vp, xy, op, instance=-1, ms=1.0):
    vp = np.ascontiguousarray(vp, dtype=np.float32)
    v = np.ascontiguousarray(xy, dtype=np.float32)
    return c.L.gsr_select_polygon(c.h, vp.ctypes.data_as(FP), ms, instance, v.ctypes.data_as(FP), v.size // 2, op)


def volume(c, vol, op, instance=-1, ms=1.0):
    return c.L.gsr_select_volume(c.h, cutouts([vol]), ms, instance, op)


def style(c, rgb, s):
    return c.L.gsr_set_selection_style(c.h, (C.c_float * 3)(*rgb), s)


LASSO = np.array([[40, 30], [290, 20], [200, 100], [300, 190], [20, 170], [150, 100]], dtype=np.float32)   # concave
STAR = np.array([[160, 10], [200, 190], [20, 70], [300, 70], [110, 190]], dtype=np.float32)                # self-intersecting
RECT = np.array([[0, 0], [W - 1, 0], [W - 1, 100], [0, 100]], dtype=np.float32)                         # horizontal edges
INST = [(0, 5000, rigid(4)), (4000, 6000, SCALED), (N - 301, 301, rigid(5)), (7, 4001, rigid(6))]


@pytest.mark.parametrize("inst", [False, True])
def test_region_operations_are_the_rules(inst):
    splat60 = cloud(N)
    vp, ub = view()
    with ShCtx(N, W, H) as c:
        c.upload(splat60)
        if inst:
            set_instances(c, INST)
        hid = np.zeros(N, bool)
        sel = np.zeros(N, bool)
        steps = []
        for i, (kind, arg, op) in enumerate([("poly", LASSO, sref.SET), ("poly", STAR, sref.TOGGLE), ("poly", RECT, sref.ADD),
                                             ("vol", cr.box([0.1, 0.0, 2.6], 0.4, cr.ELLIPSOID, space=cr.SOURCE), sref.SUBTRACT),
                                             ("vol", cr.box([0.0, 0.1, 2.4], [0.3, 0.5, 0.3], cr.BOX, space=cr.FRAME), sref.ADD),
                                             ("all", None, sref.TOGGLE), ("poly", LASSO[:4], sref.SUBTRACT)]):
            k = (i % len(INST)) if inst else -1
            instance = (INST[k][0], INST[k][1], INST[k][2]) if inst else None
            if kind == "poly":
                _lib.check(polygon(c, vp, arg, op, k), "polygon")
                inside = sref.polygon_set(splat60, N, vp, W, H, arg, instance=instance)
            elif kind == "vol":
                _lib.check(volume(c, arg, op, k), "volume")
                inside = sref.volume_set(splat60, N, arg[0], arg[1], arg[3], instance=instance)
            else:
                _lib.check(c.L.gsr_select_all(c.h, op), "all")
                inside = np.ones(N, bool)
            sel = sref.combine(op, sel, inside, hid)
            steps.append(inside.sum())
            if i == 3:
                _lib.check(c.L.gsr_hide_selection(c.h), "hide")
                hid, sel = hid | sel, np.zeros(N, bool)
            gh, gs = get_masks(c)
            np.testing.assert_array_equal(gh, hid, err_msg=f"step {i}")
            np.testing.assert_array_equal(gs, sel, err_msg=f"step {i}")
            assert counts(c) == (int(sel.sum()), int(hid.sum()))
        assert min(steps) > 50 and max(steps[:5]) < N   # every region cuts the cloud


@pytest.mark.parametrize("variant", ["plain", "instances", "highlight_off", "depth", "orthographic_cut"])
def test_frames_with_masks_are_the_reference(variant):
    splat60 = cloud(N)
    ortho = variant == "orthographic_cut"
    vp, ub = oref.ortho_camera(W, H, size=2.6, near=0.5, far=4.5, frame=25) if ortho else view()
    inst = INST if variant == "instances" else None
    hid, sel = seeded_masks(N, 5)
    st = ((0.2, 0.9, 3.0), 0.0 if variant == "highlight_off" else 0.35)
    vols = crop_set(splat60, "mixed", seed=3) if ortho else []
    Z = None
    if variant == "depth":
        V = np.asarray(vp, dtype=np.float64)[:16].reshape(4, 4)
        d = -(splat60[:, 0:3].astype(np.float64) @ V[:3, 2] + V[3, 2])
        Z = np.full((H, W), float(np.median(d)), dtype=np.float32)
    ref = sref.oracle_frame(splat60, vp, ub, hid, sel, st, vols, inst, scene_depth=Z, ortho=ortho)
    with ShCtx(N, W, H, 0, _lib.GSR_FLAG_ORTHOGRAPHIC if ortho else 0) as c:
        c.upload(splat60)
        if inst is not None:
            set_instances(c, inst)
        if vols:
            _lib.check(c.L.gsr_set_cutouts(c.h, cutouts(vols), len(vols)), "cutouts")
        depth = None
        if Z is not None:
            Zt = torch.from_numpy(Z).cuda()
            depth = torch.zeros((H, W), dtype=torch.float32, device="cuda")
            torch.cuda.synchronize()
            _lib.check(c.L.gsr_set_depth_compositing(c.h, C.c_void_p(Zt.data_ptr()), C.c_void_p(depth.data_ptr())), "depth")
        _lib.check(style(c, *st), "style")
        _lib.check(set_masks(c, hid, sel), "set masks")
        rgba = c.render(vp, ub)
        c.sync()
        check(c, rgba, ref, len(ref["records"]))
        if depth is not None:
            np.testing.assert_array_equal(bits(depth.cpu().numpy()), bits(ref["depth"]))
        assert ref["visible"] > 500


def test_empty_masks_and_zero_strength_are_the_default_frame():
    splat60 = cloud(N)
    vp, ub = view()
    want = default_frame(splat60, vp, ub, N)
    with ShCtx(N, W, H) as c:
        c.upload(splat60)
        before = c.render(vp, ub)
        launches = c.stats().kernel_launches
        _lib.check(c.L.gsr_select_all(c.h, sref.SUBTRACT), "in use, empty")
        np.testing.assert_array_equal(bits(c.render(vp, ub)), bits(want.rgba))
        _lib.check(c.L.gsr_select_all(c.h, sref.SET), "all selected")
        _lib.check(style(c, (1.0, 0.5, 0.0), 0.0), "strength 0")
        np.testing.assert_array_equal(bits(c.render(vp, ub)), bits(want.rgba))
        _lib.check(c.L.gsr_clear_splat_masks(c.h), "clear")
        assert counts(c) == (0, 0)
        after = c.render(vp, ub)
        np.testing.assert_array_equal(bits(after), bits(before))
        assert c.stats().kernel_launches == launches


@pytest.mark.parametrize("pipeline", [0, 1])
def test_operations_between_frames_follow_the_stream(pipeline):
    """select, frame, add, frame, hide, frame, set, frame, clear, frame -- asynchronous frames; each against the masks at its place."""
    splat60 = cloud(N)
    vp, ub = view()
    st = sref.DEFAULT_STYLE
    with ShCtx(N, W, H) as c:
        c.upload(splat60)
        _lib.check(c.L.gsr_debug_pipeline(c.h, pipeline), "pipeline")
        outs = [torch.zeros((H, W, 4), dtype=torch.float32, device="cuda") for _ in range(5)]
        torch.cuda.synchronize()
        hid, sel = np.zeros(N, bool), np.zeros(N, bool)
        states = []

        def frame(i):
            _lib.check(c.L.gsr_set_framebuffer_external(c.h, C.c_void_p(outs[i].data_ptr())), "fb")
            c.render_async(vp, ub)
            states.append((hid.copy(), sel.copy()))

        inside = sref.polygon_set(splat60, N, vp, W, H, LASSO)
        _lib.check(polygon(c, vp, LASSO, sref.SET), "select")
        sel = sref.combine(sref.SET, sel, inside, hid)
        frame(0)
        vol = cr.box([0.0, 0.1, 2.4], [0.3, 0.5, 0.3])
        _lib.check(volume(c, vol, sref.ADD), "add")
        sel = sref.combine(sref.ADD, sel, sref.volume_set(splat60, N, vol[0], vol[1], vol[3]), hid)
        frame(1)
        _lib.check(c.L.gsr_hide_selection(c.h), "hide")
        hid, sel = hid | sel, np.zeros(N, bool)
        frame(2)
        inside = sref.polygon_set(splat60, N, vp, W, H, STAR)
        _lib.check(polygon(c, vp, STAR, sref.SET), "set")
        sel = sref.combine(sref.SET, sel, inside, hid)
        frame(3)
        _lib.check(c.L.gsr_clear_splat_masks(c.h), "clear")
        hid, sel = np.zeros(N, bool), np.zeros(N, bool)
        frame(4)
        c.sync()
        for i, (h_, s_) in enumerate(states):
            ref = sref.oracle_frame(splat60, vp, ub, h_, s_, st)
            np.testing.assert_array_equal(bits(outs[i].cpu().numpy()), bits(ref["rgba"]), err_msg=f"frame {i}")


@pytest.mark.parametrize("inst", [False, True])
def test_select_ids_is_the_plane_sources(inst):
    splat60 = cloud(N)
    vp, ub = view()
    with ShCtx(N, W, H) as c:
        c.upload(splat60)
        if inst:
            set_instances(c, INST)
        depth = torch.zeros((H, W), dtype=torch.float32, device="cuda")
        ids = torch.zeros((H, W, 2), dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        _lib.check(c.L.gsr_set_depth_compositing(c.h, None, C.c_void_p(depth.data_ptr())), "depth")
        _lib.check(c.L.gsr_set_splat_ids(c.h, C.c_void_p(ids.data_ptr())), "ids")
        c.render(vp, ub)
        c.sync()
        plane = ids.cpu().numpy().view(np.uint32)
        ranges = [(f, n) for f, n, _ in INST] if inst else None
        src = splat_sources(plane, ranges)
        for rect in [(0, 0, W, H), (33, 17, 201, 150)]:
            x0, y0, x1, y1 = rect
            _lib.check(c.L.gsr_select_ids(c.h, C.c_void_p(ids.data_ptr()), x0, y0, x1, y1, sref.SET), "select ids")
            want = np.zeros(N, bool)
            s = src[y0:y1, x0:x1].reshape(-1)
            want[s[s != _lib.GSR_NO_ID].astype(np.int64)] = True
            np.testing.assert_array_equal(get_masks(c)[1], want)
            np.testing.assert_array_equal(want, sref.id_set(plane, N, rect, ranges))
            assert want.sum() > 100
        # hiding what was seen: no ID of the next frame reports a hidden splat
        _lib.check(c.L.gsr_hide_selection(c.h), "hide")
        c.render(vp, ub)
        c.sync()
        src2 = splat_sources(ids.cpu().numpy().view(np.uint32), ranges)
        hid = get_masks(c)[0]
        seen = src2[src2 != _lib.GSR_NO_ID].astype(np.int64)
        assert not hid[seen].any()


def test_get_set_counts_and_survival():
    splat60 = cloud(N)
    vp, ub = view()
    hid, sel = seeded_masks(N, 9)
    with ShCtx(N, W, H) as c:
        c.upload(splat60)
        assert get_masks(c)[0].sum() == 0 and counts(c) == (0, 0)
        _lib.check(set_masks(c, hid, sel), "set")
        assert counts(c) == (int(sel.sum()), int(hid.sum()))
        c.upload(splat60[:1000], first=0)
        c.resize(W + 16, H)
        set_instances(c, INST)
        set_instances(c, [])
        gh, gs = get_masks(c)
        np.testing.assert_array_equal(gh, hid)
        np.testing.assert_array_equal(gs, sel)
        c.resize(W, H)
        ref = sref.oracle_frame(splat60, vp, ub, hid, sel)
        check(c, c.render(vp, ub), ref, N)


def test_overflow_and_static_capacity():
    splat60 = cloud(N)
    vp, ub = view()
    hid, sel = seeded_masks(N, 11, hidden=0.2)
    ref = sref.oracle_frame(splat60, vp, ub, hid, sel)
    with ShCtx(N, W, H, factor=1) as c:   # the first synchronous frame overflows and is rendered again
        c.upload(splat60)
        _lib.check(set_masks(c, hid, sel), "set")
        assert ref["m"] > N
        check(c, c.render(vp, ub), ref, N)
    with ShCtx(N, W, H, 0, _lib.GSR_FLAG_STATIC_CAPACITY, factor=64) as c:
        c.upload(splat60)
        _lib.check(set_masks(c, hid, sel), "set")
        check(c, c.render(vp, ub), ref, N)


def test_single_context_rule_and_argument_checks():
    splat60 = cloud(N)
    vp, ub = view()
    INV, STATE = _lib.GSR_ERR_INVALID, _lib.GSR_ERR_STATE
    with ShCtx(N, W, H) as c:
        c.upload(splat60)
        words = (N + 31) // 32
        z = np.zeros(words, np.uint32)
        # a sharded context refuses every call that puts the masks in use
        c.set_band(0, 3)
        assert c.L.gsr_select_all(c.h, 0) == STATE
        assert polygon(c, vp, RECT, 0) == STATE
        assert volume(c, cr.box([0, 0, 0], 1.0), 0) == STATE
        assert c.L.gsr_set_splat_masks(c.h, z.ctypes.data_as(U32P), z.ctypes.data_as(U32P), words) == STATE
        assert c.L.gsr_clear_splat_masks(c.h) == 0
        c.set_band(0, (H + 15) // 16)
        # masks in use refuse every call that would shard the context; clear lifts the refusal
        _lib.check(c.L.gsr_select_all(c.h, 0), "all")
        assert c.L.gsr_set_band(c.h, 0, 3) == STATE
        assert c.L.gsr_set_row_interleave(c.h, 0, 2) == STATE
        _lib.check(c.L.gsr_clear_splat_masks(c.h), "clear")
        _lib.check(c.L.gsr_set_band(c.h, 0, 3), "band after clear")
        c.set_band(0, (H + 15) // 16)
        _lib.check(c.L.gsr_select_all(c.h, 0), "all")
        before = get_masks(c)
        # GSR_ERR_INVALID keeps the state
        assert c.L.gsr_select_all(c.h, 4) == INV
        assert polygon(c, vp, RECT[:2], 0) == INV
        assert polygon(c, vp, np.zeros((65, 2), np.float32), 0) == INV
        assert polygon(c, vp, np.array([[0, 0], [np.nan, 1], [3, 4]], np.float32), 0) == INV
        assert polygon(c, vp, RECT, 0, instance=0) == INV   # no instances
        assert polygon(c, vp, RECT, 0, instance=-2) == INV
        bad = cr.volume(np.full((3, 4), np.inf))
        assert volume(c, bad, 0) == INV
        assert c.L.gsr_select_volume(c.h, None, 1.0, -1, 0) == INV
        ids = torch.zeros((H, W, 2), dtype=torch.int32, device="cuda")
        for rect in [(-1, 0, 5, 5), (0, 0, W + 1, 5), (0, 0, 5, H + 1), (5, 0, 4, 5)]:
            assert c.L.gsr_select_ids(c.h, C.c_void_p(ids.data_ptr()), *rect, 0) == INV
        assert c.L.gsr_get_splat_masks(c.h, z.ctypes.data_as(U32P), z.ctypes.data_as(U32P), words + 1) == INV
        z1 = np.zeros(words + 1, np.uint32)
        assert c.L.gsr_set_splat_masks(c.h, z1.ctypes.data_as(U32P), z1.ctypes.data_as(U32P), words + 1) == INV
        assert c.L.gsr_set_splat_masks(c.h, z.ctypes.data_as(U32P), z.ctypes.data_as(U32P), words - 1) == INV
        for shape, space in ((2, cr.FRAME), (cr.BOX, 2), (-1, cr.SOURCE)):
            assert volume(c, cr.box([0, 0, 2.5], 1.0, shape, space=space), 0) == INV
        for a, b in zip(get_masks(c), before):
            np.testing.assert_array_equal(a, b)
        set_instances(c, INST)
        assert polygon(c, vp, RECT, 0, instance=len(INST)) == INV   # past the layout
        assert volume(c, cr.box([0, 0, 2.5], 1.0), 0, instance=len(INST)) == INV
        for a, b in zip(get_masks(c), before):
            np.testing.assert_array_equal(a, b)
        _lib.check(polygon(c, vp, RECT, sref.ADD, instance=len(INST) - 1), "the last instance")
        set_instances(c, [])
        _lib.check(c.L.gsr_select_all(c.h, sref.SET), "back to all")
        before = get_masks(c)
        full = np.full(words, 0xFFFFFFFF, np.uint32)
        assert c.L.gsr_set_splat_masks(c.h, z.ctypes.data_as(U32P), full.ctypes.data_as(U32P), words) == INV   # bits past max_splats
        one = np.zeros(words, np.uint32)
        one[3] = 1
        assert c.L.gsr_set_splat_masks(c.h, one.ctypes.data_as(U32P), one.ctypes.data_as(U32P), words) == INV   # overlap
        assert style(c, (1.0, np.nan, 0.0), 0.5) == INV
        assert style(c, (1.0, 17.0, 0.0), 0.5) == INV
        assert style(c, (1.0, 0.5, 0.0), 1.5) == INV
        assert style(c, (1.0, 0.5, 0.0), -0.1) == INV
        after = get_masks(c)
        np.testing.assert_array_equal(before[0], after[0])
        np.testing.assert_array_equal(before[1], after[1])
    cfg = _lib.GsrConfig(0, 0, 100, 10, 0)
    h = C.c_void_p()
    L = _lib.lib()
    _lib.check(L.gsr_create(C.byref(cfg), C.byref(h)), "create")
    try:   # no size yet
        ids = torch.zeros((2, 2, 2), dtype=torch.int32, device="cuda")
        assert L.gsr_select_ids(h, C.c_void_p(ids.data_ptr()), 0, 0, 1, 1, 0) == STATE
    finally:
        L.gsr_destroy(h)


def test_python_mirror():
    from godotgaussiansplatting_b200 import camera as cam
    from godotgaussiansplatting_b200.rasterizer import GaussianSplattingRasterizer
    from godotgaussiansplatting_b200.synthetic import synthetic_ply
    r = GaussianSplattingRasterizer(synthetic_ply(3001, 4), (160, 96), None, cam.orbit_camera(25, aspect=160 / 96))
    r.init_gpu()
    try:
        r.select_all()
        assert r.selection_counts() == (3001, 0)
        r.select_polygon([[0, 0], [159, 0], [159, 40], [0, 40]], _lib.GSR_SELECT_SUBTRACT)
        hid, sel = r.splat_masks()
        r.hide_selection()
        assert r.selection_counts() == (0, int(sel.sum()))
        r.set_splat_masks(hid, sel)
        np.testing.assert_array_equal(r.splat_masks()[1], sel)
        r.set_selection_style((0, 1, 0), 0.8)
        r.rasterize()
        r.clear_splat_masks()
        assert r.selection_counts() == (0, 0)
    finally:
        r.cleanup_gpu()


# ---- every projection and compositor variant with masks in use ------------------------------------------------------------------
MATRIX_N = 10240
MATRIX_STYLE = ((0.25, 1.5, 0.75), 0.4)


def render_masked_case(fr, hid, sel):
    """tests/test_gpu_variant_matrix's draw of a case, with the masks and the style set before the case's frames."""
    from godotgaussiansplatting_b200.rasterizer import pack_instance_appearance
    from tests.test_gpu_variant_matrix import flags_of, set_cutouts
    case = fr.case
    L = _lib.lib()
    heat = 1.0 if case.heat else 0.0
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
            set_instances(c, fr.prev_inst if fr.prev_inst is not None else fr.inst)
            if fr.app is not None:
                app = pack_instance_appearance(fr.app)
                _lib.check(L.gsr_set_instance_appearance(c.h, app, len(app)), "gsr_set_instance_appearance")
        _lib.check(style(c, *MATRIX_STYLE), "gsr_set_selection_style")
        _lib.check(set_masks(c, hid, sel), "gsr_set_splat_masks")
        depth = motion = None
        if case.compositor != "plain":
            Zt = None if fr.Z is None else torch.from_numpy(fr.Z).cuda()
            depth = torch.full((fr.h, fr.w), float("nan"), dtype=torch.float32, device="cuda")
            torch.cuda.synchronize()
            _lib.check(L.gsr_set_depth_compositing(c.h, None if Zt is None else C.c_void_p(Zt.data_ptr()), C.c_void_p(depth.data_ptr())),
                       "gsr_set_depth_compositing")
        if case.compositor == "motion":
            motion = torch.full((fr.h, fr.w, 2), float("nan"), dtype=torch.float32, device="cuda")
            torch.cuda.synchronize()
            _lib.check(L.gsr_set_motion_vectors(c.h, C.c_void_p(motion.data_ptr())), "gsr_set_motion_vectors")
            c.render(fr.pvp, fr.pub, heatmap=heat)
            if case.inst:
                set_instances(c, fr.inst)
        rgba = c.render(fr.vp, fr.ub, heatmap=heat)
        c.sync()
        st = c.stats()
        m = int(min(st.duplicates, st.capacity))
        T = st.tiles_x * st.tiles_y
        return dict(rgba=rgba, depth=None if depth is None else depth.cpu().numpy(), motion=None if motion is None else motion.cpu().numpy(),
                    stats=st, keys=c.copy(_lib.GSR_BUF_KEYS, m, np.uint32), values=c.copy(_lib.GSR_BUF_VALUES, m, np.uint32),
                    bounds=c.copy(_lib.GSR_BUF_BOUNDS, T * 2, np.uint32).reshape(T, 2),
                    records=c.copy(_lib.GSR_BUF_RECORDS, fr.drawn, REC_DTYPE))


def _matrix_cases():
    from tests import variant_matrix as vm
    return range(len(vm.CASES)), vm.IDS


@pytest.mark.parametrize("i", _matrix_cases()[0], ids=_matrix_cases()[1])
def test_variant_matrix_with_masks(i):
    """Every case of tests/variant_matrix on its CUT = true projection kernel (masks in use route every case there), with a seeded
    hidden and selected mask and a non-zero highlight, bit for bit against the composed reference."""
    from tests import variant_matrix as vm
    case = vm.CASES[i]
    fr = vm.frame_of(case, MATRIX_N, (320, 192), (321, 181))
    hid, sel = seeded_masks(fr.n, 100 + i, hidden=0.25, selected=0.2)
    ref = sref.variant_frame(fr, hid, sel, MATRIX_STYLE)
    vm.assert_both_phase2_paths(ref)   # the highlight runs in the bulk and in the per-lane colour path
    ids = np.unique(ref["values"])
    assert np.isin(ids, ref["selected_ids"]).sum() > 20
    got = render_masked_case(fr, hid, sel)
    st = got["stats"]
    assert (st.duplicates, st.visible, st.last_tile, bool(st.overflow)) == (ref["m"], ref["visible"], ref["last_tile"], False)
    np.testing.assert_array_equal(got["keys"], ref["keys"])
    np.testing.assert_array_equal(got["values"], ref["values"])
    np.testing.assert_array_equal(got["bounds"], ref["bounds"])
    for w in ("image_pos", "pos_xy", "conic", "pos_z", "color"):
        np.testing.assert_array_equal(bits(got["records"][w][ids]), bits(ref["records"][w][ids]), err_msg=f"record word {w}")
    np.testing.assert_array_equal(bits(got["rgba"]), bits(ref["rgba"]))
    assert st.staged == ref["staged"]
    if got["depth"] is not None:
        np.testing.assert_array_equal(bits(got["depth"]), bits(ref["depth"]))
    assert (got["motion"] is None) == (case.compositor != "motion")
    if got["motion"] is not None:
        np.testing.assert_array_equal(bits(got["motion"]), bits(ref["motion"]))
