"""Cutout frames on the GPU (include/gsr.h gsr_set_cutouts), through the C-ABI: every frame with a set is bit for bit the composed
reference's (tests/cutout_reference) in RGBA, keys, values, bounds, records of drawn ids and stats; an empty set restores the default
frame; each async frame follows the set it was enqueued with; the single-context rules and the argument checks hold; gsr_pick never
returns a cut splat; and the Python mirror sets it."""
import ctypes as C

import numpy as np
import pytest

from godotgaussiansplatting_b200 import _lib
from godotgaussiansplatting_b200 import camera as cam
from godotgaussiansplatting_b200.ply_file import PlyFile, swizzle_splats
from godotgaussiansplatting_b200.rasterizer import GaussianSplattingRasterizer
from godotgaussiansplatting_b200.synthetic import synthetic_ply_table
from oracle import oracle as orc
from tests import cutout_reference as cr
from tests import ortho_reference as oref
from tests.gsr_direct import REC_DTYPE
from tests.scenes import make_scene
from tests.test_cutouts import crop_set
from tests.test_gpu_sh_degree import ShCtx, set_instances
from tests.test_sh_degree import zero_splat_coeffs

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

W, H = 320, 200


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def cloud(n, seed=3):
    t62 = synthetic_ply_table(n, seed)
    t62[:, 55:58] += 0.5
    t62[:, 9:54] += 0.02
    return swizzle_splats(t62, 0.0)


def view(width=W, height=H, frame=25):
    _, vp, ub = make_scene(16, 1, width, height, frame=frame)
    return vp, ub


def cutouts(vols):
    arr = (_lib.GsrCutout * max(1, len(vols)))()
    for k, (c12, shape, action, space) in enumerate(vols):
        arr[k].to_local[:] = [float(v) for v in np.asarray(c12, dtype=np.float32)]
        arr[k].shape, arr[k].action, arr[k].space = int(shape), int(action), int(space)
    return arr


def set_cut(c, vols):
    return c.L.gsr_set_cutouts(c.h, cutouts(vols), len(vols))


def default_frame(splat60, vp, ub, n):
    return orc.frame(splat60, vp, orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8)), cap=64 * n)


def check(c, rgba, ref, drawn, overflow=False):
    np.testing.assert_array_equal(bits(rgba), bits(ref["rgba"]))
    st = c.stats()
    assert st.duplicates == ref["m"] and st.visible == ref["visible"] and st.last_tile == ref["last_tile"]
    assert bool(st.overflow) == overflow
    m = int(min(st.duplicates, st.capacity))
    T = st.tiles_x * st.tiles_y
    np.testing.assert_array_equal(c.copy(_lib.GSR_BUF_KEYS, m, np.uint32), ref["keys"])
    np.testing.assert_array_equal(c.copy(_lib.GSR_BUF_VALUES, m, np.uint32), ref["values"])
    np.testing.assert_array_equal(c.copy(_lib.GSR_BUF_BOUNDS, T * 2, np.uint32).reshape(T, 2), ref["bounds"])
    recs = c.copy(_lib.GSR_BUF_RECORDS, drawn, REC_DTYPE)
    ids = np.unique(ref["values"])
    np.testing.assert_array_equal(bits(recs[ids].view(np.float32)), bits(ref["records"][ids].view(np.float32)))


VARIANTS = ["plain", "heatmap", "uncontracted", "instances_frame", "instances_source", "orthographic", "aa_0.3", "reduced_store",
            "depth_order", "depth_compositing", "ragged"]


@pytest.mark.parametrize("variant", VARIANTS)
def test_frames_are_the_cutout_reference(variant):
    n = 12288
    splat60 = cloud(n)
    w, h = (321, 181) if variant == "ragged" else (W, H)
    ortho = variant == "orthographic"
    vp, ub = oref.ortho_camera(w, h, size=2.6, near=0.5, far=4.5, frame=25) if ortho else view(w, h)
    v = 0.3 if variant == "aa_0.3" else 0.0
    flags = (_lib.GSR_FLAG_UNCONTRACTED_BLEND if variant == "uncontracted" else 0) | (_lib.GSR_FLAG_ORTHOGRAPHIC if ortho else 0)
    heat = 1.0 if variant == "heatmap" else 0.0
    bands = 2 if variant == "reduced_store" else 0
    src = zero_splat_coeffs(splat60, 2) if bands else splat60
    inst = None
    if variant.startswith("instances"):   # overlapping and repeated ranges
        from tests.test_instances import SCALED, rigid
        inst = [(0, 5000, rigid(4)), (4000, 6000, SCALED), (n - 301, 301, rigid(5)), (0, 5000, rigid(6))]
    kind = "source" if variant == "instances_source" else "mixed"
    vols = crop_set(splat60, kind, cr.positions(splat60, 1.0, inst)[1], seed=3)
    Z = None
    if variant == "depth_compositing":   # a scene plane through the middle of the cloud
        V = np.asarray(vp, dtype=np.float64)[:16].reshape(4, 4)
        d = -(splat60[:, 0:3].astype(np.float64) @ V[:3, 2] + V[3, 2])
        Z = np.full((h, w), float(np.median(d)), dtype=np.float32)
    ref = cr.oracle_frame(src, vp, ub, vols, v, ortho, heat, contract=variant != "uncontracted", inst=inst, scene_depth=Z,
                          depth_order=variant == "depth_order")
    assert ref["visible"] > 500
    with ShCtx(n, w, h, bands, flags) as c:
        c.upload(splat60)
        if inst is not None:
            set_instances(c, inst)
        if v:
            _lib.check(c.L.gsr_set_antialiasing(c.h, C.c_float(v)), "gsr_set_antialiasing")
        if variant == "depth_order":
            _lib.check(c.L.gsr_set_depth_order(c.h, _lib.GSR_DEPTH_ORDER_VIEW_DEPTH), "gsr_set_depth_order")
        depth = None
        if Z is not None:
            Zt = torch.from_numpy(Z).cuda()
            depth = torch.zeros((h, w), dtype=torch.float32, device="cuda")
            torch.cuda.synchronize()
            _lib.check(c.L.gsr_set_depth_compositing(c.h, C.c_void_p(Zt.data_ptr()), C.c_void_p(depth.data_ptr())), "depth")
        _lib.check(set_cut(c, vols), "gsr_set_cutouts")
        rgba = c.render(vp, ub, heatmap=heat)
        c.sync()
        check(c, rgba, ref, len(ref["records"]))
        if depth is not None:
            np.testing.assert_array_equal(bits(depth.cpu().numpy()), bits(ref["depth"]))
        if variant == "plain":   # more orbit frames on the same context, then the set switched off
            for f in (3, 40, 77):
                vpf, ubf = view(frame=f)
                check(c, c.render(vpf, ubf), cr.oracle_frame(splat60, vpf, ubf, vols), n)
            _lib.check(c.L.gsr_set_cutouts(c.h, None, 0), "off")
            want = default_frame(splat60, vp, ub, n)
            np.testing.assert_array_equal(bits(c.render(vp, ub)), bits(want.rgba))
            m = int(c.stats().duplicates)
            assert m == want.duplicates
            np.testing.assert_array_equal(c.copy(_lib.GSR_BUF_KEYS, m, np.uint32), want.keys)
            np.testing.assert_array_equal(c.copy(_lib.GSR_BUF_VALUES, m, np.uint32), want.values)


def test_static_capacity_truncates_after_the_filter():
    n = 12288
    splat60 = cloud(n, seed=4)
    vp, ub = view()
    vols = crop_set(splat60, "remove_ellipsoid", seed=2)
    with ShCtx(n, W, H, 0, _lib.GSR_FLAG_STATIC_CAPACITY, factor=1) as c:
        c.upload(splat60)
        _lib.check(set_cut(c, vols), "gsr_set_cutouts")
        c.L.gsr_render(c.h, np.ascontiguousarray(vp, dtype=np.float32).ctypes.data_as(C.POINTER(C.c_float)), ub, 0.0, None)
        cap = int(c.stats().capacity)
        ref = cr.oracle_frame(splat60, vp, ub, vols, cap=cap)
        assert ref["m"] > cap
        out = np.empty((H, W, 4), dtype=np.float32)
        rc = c.L.gsr_render(c.h, np.ascontiguousarray(vp, dtype=np.float32).ctypes.data_as(C.POINTER(C.c_float)), ub, 0.0,
                            C.c_void_p(out.ctypes.data))
        assert rc in (_lib.GSR_OK, _lib.GSR_ERR_OVERFLOW)
        check(c, out, ref, n, overflow=True)


def test_a_set_that_removes_everything_gives_an_empty_frame():
    n = 12288
    splat60 = cloud(n, seed=6)
    vp, ub = view()
    nothing = [cr.volume(np.concatenate([np.eye(3) * 1e-6, np.zeros((3, 1))], axis=1), cr.BOX, cr.REMOVE)]
    with ShCtx(n, W, H) as c:
        c.upload(splat60)
        _lib.check(set_cut(c, nothing), "gsr_set_cutouts")
        rgba = c.render(vp, ub)
        st = c.stats()
        assert st.duplicates == 0 and st.visible == 0 and st.last_tile == -1
        assert np.isfinite(rgba).all()
        np.testing.assert_array_equal(bits(rgba), bits(cr.oracle_frame(splat60, vp, ub, nothing)["rgba"]))


@pytest.mark.parametrize("overlap", [0, 1], ids=["serial", "overlap"])
def test_sets_change_between_async_frames(overlap):
    n = 12288
    splat60 = cloud(n, seed=9)
    sets = [crop_set(splat60, "keep_box", seed=1), [], crop_set(splat60, "mixed", seed=2), crop_set(splat60, "remove_ellipsoid", seed=3),
            [], crop_set(splat60, "source", seed=4)]
    frames = [view(frame=20 + k) for k in range(len(sets))]
    with ShCtx(n, W, H) as c:
        c.upload(splat60)
        _lib.check(c.L.gsr_debug_pipeline(c.h, overlap), "gsr_debug_pipeline")
        hosts = [torch.empty((H, W, 4), dtype=torch.float32, pin_memory=True) for _ in frames]
        for vols, (vp, ub), hb in zip(sets, frames, hosts):
            _lib.check(set_cut(c, vols), "gsr_set_cutouts")
            c.render_async(vp, ub, host_ptr=hb.data_ptr())
        c.sync()
    for k, (vols, (vp, ub), hb) in enumerate(zip(sets, frames, hosts)):
        want = cr.oracle_frame(splat60, vp, ub, vols)["rgba"] if vols else default_frame(splat60, vp, ub, n).rgba
        np.testing.assert_array_equal(bits(hb.numpy()), bits(want), err_msg=f"frame {k}")


def test_state_rules_and_invalid_sets():
    n = 4096
    splat60 = cloud(n)
    vp, ub = view()
    handles = (C.c_ubyte * 128)()
    blob = (C.c_ubyte * _lib.GSR_GROUP_BLOB_BYTES)()
    vols = crop_set(splat60, "mixed", seed=5)
    with ShCtx(n, W, H) as c:
        c.upload(splat60)
        L = c.L
        want = cr.oracle_frame(splat60, vp, ub, vols)
        _lib.check(set_cut(c, vols), "gsr_set_cutouts")
        good = vols[0]
        bad_sets = [[good] * 17, [(np.where(np.arange(12) == 4, np.nan, good[0]).astype(np.float32),) + good[1:]],
                    [(np.where(np.arange(12) == 11, np.inf, good[0]).astype(np.float32),) + good[1:]],
                    [good, (good[0], 2, cr.KEEP, cr.FRAME)], [(good[0], cr.BOX, 2, cr.FRAME)], [(good[0], cr.BOX, cr.KEEP, -1)]]
        for bad in bad_sets:
            assert set_cut(c, bad) == _lib.GSR_ERR_INVALID
        assert L.gsr_set_cutouts(c.h, None, 3) == _lib.GSR_ERR_INVALID
        check(c, c.render(vp, ub), want, n)   # the previous set is kept
        # a singular to_local (a flat slab) is a valid volume
        slab = np.zeros((3, 4))
        slab[2, 2] = 1.0
        assert set_cut(c, [cr.volume(slab)]) == _lib.GSR_OK
        _lib.check(set_cut(c, vols), "back")
        # while a set is active, the multi-context calls are refused
        assert L.gsr_set_band(c.h, 0, 3) == _lib.GSR_ERR_STATE
        assert L.gsr_set_row_interleave(c.h, 0, 2) == _lib.GSR_ERR_STATE
        assert L.gsr_peer_export_framebuffers(c.h, handles) == _lib.GSR_ERR_STATE
        assert L.gsr_peer_import_framebuffers(c.h, handles) == _lib.GSR_ERR_STATE
        assert L.gsr_group_export(c.h, blob) == _lib.GSR_ERR_STATE
        check(c, c.render(vp, ub), want, n)
        # and a non-empty set is refused on a multi-context setup (an empty one is not)
        _lib.check(L.gsr_set_cutouts(c.h, None, 0), "off")
        for setup, undo in ((lambda: L.gsr_set_band(c.h, 0, 3), lambda: L.gsr_set_band(c.h, 0, (H + 15) // 16)),
                            (lambda: L.gsr_set_row_interleave(c.h, 0, 2), lambda: L.gsr_set_row_interleave(c.h, 0, 1)),
                            (lambda: L.gsr_peer_export_framebuffers(c.h, handles), lambda: L.gsr_resize(c.h, W, H))):
            _lib.check(setup(), "setup")
            assert set_cut(c, vols) == _lib.GSR_ERR_STATE
            assert set_cut(c, []) == _lib.GSR_OK
            _lib.check(undo(), "undo")
        _lib.check(set_cut(c, vols), "on")
        c.resize(W, H)   # keeps the set
        check(c, c.render(vp, ub), want, n)


def test_pick_never_returns_a_cut_splat():
    n = 12288
    splat60 = cloud(n, seed=8)
    vp, ub = view()
    vols = crop_set(splat60, "mixed", seed=6)
    ref = cr.oracle_frame(splat60, vp, ub, vols)
    with ShCtx(n, W, H) as c:
        c.upload(splat60)
        _lib.check(set_cut(c, vols), "gsr_set_cutouts")
        c.render(vp, ub)
        T = c.stats().tiles_x * c.stats().tiles_y
        counts = ref["bounds"][:, 1].astype(np.int64) - ref["bounds"][:, 0].astype(np.int64)
        tiles = np.nonzero(counts > 0)[0][::7]
        assert len(tiles) > 10
        cut_ids = np.setdiff1d(np.unique(orc.project(splat60, vp, orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8)), cap=64 * n).values),
                               np.unique(ref["values"]))
        assert len(cut_ids) > 100
        cut_pos = {tuple(bits(splat60[i, 0:3].astype(np.float32))) for i in cut_ids}
        prev = np.zeros(4, dtype=np.float32)
        picked = 0
        for t in tiles:   # gsr_pick's buffer persists across calls like the reference's: carry the oracle's along
            prev = orc.render(ref["records"], ref["values"], ref["bounds"], W, H, 0.0, target_tile=int(t), pick=prev)[2]
            out = c.pick(int(t))
            np.testing.assert_array_equal(bits(out), bits(prev))
            assert tuple(bits(out[:3].copy())) not in cut_pos
            picked += out[3] > 0
        assert picked > 10 and T > 0


def test_large_frame_with_a_crop_box():
    n, w, h = 1_500_000, 1280, 720
    splat60, vp, ub = make_scene(n, 7, w, h, frame=12)
    sp = splat60[:, 0:3]
    c0 = np.median(sp, axis=0)
    half = np.median(np.abs(sp - c0), axis=0) * 1.6
    vols = [cr.box(c0, half)]
    ref = cr.oracle_frame(splat60, vp, ub, vols)
    uncut = orc.project(splat60, vp, orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8)), cap=64 * n).visible
    assert 0.15 * uncut < ref["visible"] < 0.85 * uncut
    with ShCtx(n, w, h) as c:
        c.upload(splat60)
        _lib.check(set_cut(c, vols), "gsr_set_cutouts")
        check(c, c.render(vp, ub), ref, n)


def test_rasterizer_set_cutouts():
    n = 12288
    t62 = synthetic_ply_table(n, 12)
    t62[:, 55:58] += 0.5
    ply = PlyFile.from_array(t62)
    r = GaussianSplattingRasterizer(ply, (W, H), None, cam.orbit_camera(25, aspect=W / H))
    # a Godot box around the cloud's bulk (its Godot positions are F p: x and y negated)
    splat60 = swizzle_splats(t62, 0.0)
    p = splat60[:, 0:3].astype(np.float64) * np.array([-1.0, -1.0, 1.0])
    c0 = np.median(p, axis=0)
    T = np.concatenate([np.diag(np.median(np.abs(p - c0), axis=0) * 1.5), c0[:, None]], axis=1)
    r.set_cutouts([(T, _lib.GSR_CUTOUT_BOX, _lib.GSR_CUTOUT_KEEP, _lib.GSR_CUTOUT_FRAME)])   # before init_gpu: applied there
    r.init_gpu()
    try:
        out = np.empty((H, W, 4), dtype=np.float32)
        r.rasterize(time=10.0, out_host=out)
        vp, ub = r.camera_push_constants, r.uniforms_bytes(10.0)
        from godotgaussiansplatting_b200.rasterizer import cutout_to_local
        vols = [cr.volume(cutout_to_local(T, r.basis_override))]
        ref = cr.oracle_frame(splat60, vp, ub, vols)
        assert 0 < ref["visible"] < orc.project(splat60, vp, orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8)), cap=64 * n).visible
        np.testing.assert_array_equal(bits(out), bits(ref["rgba"]))
        r.set_cutouts([])
        r.rasterize(time=10.0, out_host=out)
        vp, ub = r.camera_push_constants, r.uniforms_bytes(10.0)
        np.testing.assert_array_equal(bits(out), bits(default_frame(splat60, vp, ub, n).rgba))
    finally:
        r.cleanup_gpu()
