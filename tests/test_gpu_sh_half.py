"""The binary16 SH store (include/gsr.h GSR_FLAG_SH_HALF) on the GPU, through the C-ABI: every frame of a binary16 store is bit for bit
the frame of the float store holding the cloud whose coefficients were rounded to binary16 once (the unchanged oracle's frame of that
cloud where the oracle covers the variant), the stored planes are the emulated ingest's, and the store keeps the single-context rules."""
import ctypes as C

import numpy as np
import pytest

from godotgaussiansplatting_b200 import _lib
from godotgaussiansplatting_b200.ply_file import PlyFile, degree_properties, narrow_table, swizzle_splats
from oracle import oracle as orc
from tests import ortho_reference as oref
from tests.gsr_direct import REC_DTYPE
from tests.test_gpu_sh_degree import H, W, ShCtx, check, oracle_frame, scene, set_instances
from tests.test_sh_half import F32, emu, half_planes, half_planes_count, layout_ints, rounded

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

HALF = _lib.GSR_FLAG_SH_HALF


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def appearance(c, rows):
    arr = (_lib.GsrInstanceAppearance * len(rows))()
    for k, (tint, opacity, draw) in enumerate(rows):
        arr[k].tint[:] = list(tint)
        arr[k].opacity, arr[k].draw_count = opacity, draw
    _lib.check(c.L.gsr_set_instance_appearance(c.h, arr, len(rows)), "gsr_set_instance_appearance")


def cutouts(c, splat60):
    """A KEEP box around the bulk of the cloud and a REMOVE ellipsoid inside it, both in frame space."""
    p = np.asarray(splat60[:, 0:3], dtype=np.float64)
    med = np.median(p, axis=0)
    half = np.median(np.abs(p - med), axis=0) * 1.5 + 1e-3
    arr = (_lib.GsrCutout * 2)()
    for i, (scale, shape, action) in enumerate(((half, _lib.GSR_CUTOUT_BOX, _lib.GSR_CUTOUT_KEEP),
                                                (half * 0.4, _lib.GSR_CUTOUT_ELLIPSOID, _lib.GSR_CUTOUT_REMOVE))):
        A = np.diag(1.0 / scale)
        arr[i].to_local[:] = [float(v) for v in np.concatenate([A.T.reshape(-1), -A @ med])]   # [A | t] column-major
        arr[i].shape, arr[i].action, arr[i].space = shape, action, _lib.GSR_CUTOUT_FRAME
    _lib.check(c.L.gsr_set_cutouts(c.h, arr, 2), "gsr_set_cutouts")


def taps(c, drawn):
    st = c.stats()
    m = int(min(st.duplicates, st.capacity))
    T = st.tiles_x * st.tiles_y
    return dict(m=int(st.duplicates), v=int(st.visible), keys=c.copy(_lib.GSR_BUF_KEYS, m, np.uint32), values=c.copy(_lib.GSR_BUF_VALUES, m, np.uint32),
                bounds=c.copy(_lib.GSR_BUF_BOUNDS, 2 * T, np.uint32), records=c.copy(_lib.GSR_BUF_RECORDS, drawn, REC_DTYPE))


def same_frame(a, b, rgba_a, rgba_b, drawn):
    np.testing.assert_array_equal(bits(rgba_a), bits(rgba_b))
    ta, tb = taps(a, drawn), taps(b, drawn)
    assert (ta["m"], ta["v"]) == (tb["m"], tb["v"]) and ta["m"] > 0
    for k in ("keys", "values", "bounds"):
        np.testing.assert_array_equal(ta[k], tb[k], err_msg=k)
    ids = np.unique(tb["values"])
    np.testing.assert_array_equal(bits(ta["records"][ids].view(np.float32)), bits(tb["records"][ids].view(np.float32)))


GPU_VS_GPU = ["ortho", "aa", "depth_order", "cutouts", "appearance", "ortho_aa_depth_order_cutouts"]


@pytest.mark.parametrize("variant", GPU_VS_GPU)
@pytest.mark.parametrize("degree", [3, 1])
def test_frames_are_the_float_store_of_the_rounded_cloud(variant, degree):
    """The variants the oracle does not cover directly: against the float store's frame of the rounded cloud (itself checked against
    the per-feature references by their own tests)."""
    n = 12288
    t62, vp, ub = scene(n, seed=21)
    splat60 = swizzle_splats(t62, 0.0)
    flags = _lib.GSR_FLAG_ORTHOGRAPHIC if "ortho" in variant else 0
    if "ortho" in variant:
        vp, _ = oref.ortho_camera(W, H, size=3.0, near=0.5, far=40.0, frame=25)
    inst = None
    drawn = n
    with ShCtx(n, W, H, 4, flags | HALF) as a, ShCtx(n, W, H, 4, flags) as b:
        a.upload(splat60)
        b.upload(rounded(splat60))
        for c in (a, b):
            _lib.check(c.degree(degree), "gsr_set_sh_degree")
            if "aa" in variant:
                _lib.check(c.L.gsr_set_antialiasing(c.h, 0.3), "aa")
            if "depth_order" in variant:
                _lib.check(c.L.gsr_set_depth_order(c.h, 1), "depth order")
            if "cutouts" in variant:
                cutouts(c, splat60)
            if variant == "appearance":
                from tests.test_instances import SCALED, rigid
                inst = [(0, 5000, rigid(4)), (4000, 6000, SCALED), (n - 301, 301, rigid(5))]
                set_instances(c, inst)
                appearance(c, [((0.5, 1.0, 2.0), 0.5, 2**64 - 1), ((1.0, 1.0, 1.0), 1.0, 3000), ((1.0, 0.25, 1.0), 0.75, 100)])
                drawn = sum((k + 31) // 32 for _, k, _ in inst) * 32
        same_frame(a, b, a.render(vp, ub), b.render(vp, ub), drawn)


VARIANTS = ["plain", "ragged", "heatmap", "instances", "depth_plane", "uncontracted"]


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("bands", [1, 2, 3, 4])
def test_frames_are_the_oracle_of_the_rounded_cloud(bands, variant):
    n = 12001 if variant == "ragged" else 12288
    t62, vp, ub = scene(n, seed=3 + bands)
    splat60 = swizzle_splats(t62, 0.0)
    flags = _lib.GSR_FLAG_UNCONTRACTED_BLEND if variant == "uncontracted" else 0
    heat = 1.0 if variant == "heatmap" else 0.0
    inst = None
    if variant == "instances":
        from tests.test_instances import SCALED, rigid
        inst = [(0, 5000, rigid(4)), (4000, 6000, SCALED), (n - 301, 301, rigid(5))]
    for store in sorted({bands, 4}):   # a store of `bands`, and a 4-band store rendered at degree bands - 1
        want = rounded(splat60, bands)
        Z = None
        if variant == "depth_plane":
            u = orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8))
            pr = orc.project(want, vp, u, cap=64 * n)
            V = np.asarray(vp, dtype=np.float32)
            r = pr.records[np.unique(pr.values)]
            d = -(((V[2] * r["pos_xy"][:, 0] + V[6] * r["pos_xy"][:, 1]) + V[10] * r["pos_z"]) + V[14] * np.float32(1.0))
            Z = np.full((H, W), np.inf, dtype=np.float32)
            Z[:, W // 2:] = np.median(d)
        ref = oracle_frame(want, vp, ub, heat, flags == 0, inst, Z, Z is not None)
        assert ref["visible"] > 0
        with ShCtx(n, W, H, store, flags | HALF) as c:
            c.upload(splat60)
            if store != bands:
                _lib.check(c.degree(bands - 1), "gsr_set_sh_degree")
            depth = None
            if Z is not None:
                Zt = torch.from_numpy(Z).cuda()
                depth = torch.zeros((H, W), dtype=torch.float32, device="cuda")
                torch.cuda.synchronize()
                _lib.check(c.L.gsr_set_depth_compositing(c.h, C.c_void_p(Zt.data_ptr()), C.c_void_p(depth.data_ptr())), "depth")
            if inst is not None:
                set_instances(c, inst)
            rgba = c.render(vp, ub, heatmap=heat)
            check(c, rgba, ref, sum((k + 31) // 32 for _, k, _ in inst) * 32 if inst else n)
            if depth is not None:
                c.sync()
                np.testing.assert_array_equal(bits(depth.cpu().numpy()), bits(ref["depth"]))


def test_c3_size_frame_is_the_float_store_of_the_rounded_cloud():
    """6 M splats at 1080p: GPU against GPU."""
    from godotgaussiansplatting_b200.synthetic import synthetic_ply_table
    from tests.scenes import make_scene
    n, w, h = 6_000_000, 1920, 1080
    splat60 = swizzle_splats(synthetic_ply_table(n, 7), 0.0)
    _, vp, ub = make_scene(16, 1, w, h, frame=25)
    with ShCtx(n, w, h, 4, HALF) as a:
        a.upload(splat60)
        rgba_a = a.render(vp, ub)
        ta = taps(a, n)
    splat60 = rounded(splat60)
    with ShCtx(n, w, h, 4, 0) as b:
        b.upload(splat60)
        rgba_b = b.render(vp, ub)
        tb = taps(b, n)
    np.testing.assert_array_equal(bits(rgba_a), bits(rgba_b))
    assert (ta["m"], ta["v"]) == (tb["m"], tb["v"]) and ta["m"] > 1_000_000
    for k in ("keys", "values", "bounds"):
        np.testing.assert_array_equal(ta[k], tb[k], err_msg=k)


@pytest.mark.parametrize("bands", [1, 2, 3, 4])
def test_stored_planes_are_the_emulated_ingest(bands):
    n, first = 3000, 0
    stride = (n + 255) // 256 * 256
    P = 3 + half_planes_count(bands)
    t62, _, _ = scene(n)
    t62[::5, 9:54] *= 1e5      # saturated coefficients
    t62[1::5, 9:54] *= 1e-6    # subnormal halves
    splat60 = swizzle_splats(t62, 0.0)

    def emulated(fn):
        soa = np.zeros((P, stride, 4), dtype=F32)
        fn(soa)
        return soa

    with ShCtx(n, W, H, bands, HALF) as c:
        size = P * stride * 4   # 16 (3 + P_h) bytes per splat of the stride
        c.upload(splat60)
        got = c.copy(_lib.GSR_BUF_SPLATS, size, np.float32)
        want = emulated(lambda s: emu().emu_sh_half_aos_to_soa(splat60.ctypes.data, n, s.ctypes.data, stride, first, P))
        np.testing.assert_array_equal(bits(got), bits(want.reshape(-1)))
        np.testing.assert_array_equal(bits(got), bits(half_planes(splat60, bands, stride).reshape(-1)))
        big = np.empty(size * 4 + 1, dtype=np.uint8)
        assert c.L.gsr_debug_copy(c.h, _lib.GSR_BUF_SPLATS, C.c_void_p(big.ctypes.data), big.nbytes) == _lib.GSR_ERR_INVALID
        # gsr_upload_ply_raw
        _lib.check(c.L.gsr_upload_ply_raw(c.h, t62.ctypes.data_as(C.POINTER(C.c_float)), 62, 0, n, 0.0), "gsr_upload_ply_raw")
        np.testing.assert_array_equal(bits(c.copy(_lib.GSR_BUF_SPLATS, size, np.float32)), bits(want.reshape(-1)))
        # gsr_upload_ply with a degree-1 layout
        narrow = np.ascontiguousarray(narrow_table(t62, 1, normals=False))
        lay = PlyFile.from_array(narrow, degree_properties(1, False)).layout()
        _lib.check(c.upload_ply(narrow, lay), "gsr_upload_ply")
        want = emulated(lambda s: emu().emu_sh_half_ply_to_soa(narrow.ctypes.data, layout_ints(lay).ctypes.data, n, 0.0, s.ctypes.data, stride, 0, P, -1))
        np.testing.assert_array_equal(bits(c.copy(_lib.GSR_BUF_SPLATS, size, np.float32)), bits(want.reshape(-1)))
        # gsr_upload_ply_filtered
        f = np.random.default_rng(2).uniform(-0.01, 0.05, size=(n, 1)).astype(F32)
        table = np.ascontiguousarray(np.concatenate([narrow, f], axis=1))
        lay = PlyFile.from_array(table, degree_properties(1, False, ("filter_3D",))).layout()
        assert lay.filter_3d == table.shape[1] - 1
        L = _lib.GsrPlyLayout(lay.nprops, lay.sh_degree, lay.x, lay.f_dc, lay.f_rest, lay.opacity, lay.scale, lay.rot)
        _lib.check(c.L.gsr_upload_ply_filtered(c.h, table.ctypes.data_as(C.POINTER(C.c_float)), C.byref(L), lay.filter_3d, 0, n, 0.0), "filtered")
        want = emulated(lambda s: emu().emu_sh_half_ply_to_soa(table.ctypes.data, layout_ints(lay).ctypes.data, n, 0.0, s.ctypes.data, stride, 0, P,
                                                               int(lay.filter_3d)))
        np.testing.assert_array_equal(bits(c.copy(_lib.GSR_BUF_SPLATS, size, np.float32)), bits(want.reshape(-1)))


def test_state_rules():
    n = 4096
    L = _lib.lib()
    blob = (C.c_ubyte * _lib.GSR_GROUP_BLOB_BYTES)()
    handles = (C.c_ubyte * 128)()
    with ShCtx(n, W, H, 4, HALF) as c:   # a binary16 store at the full degree: single-context only all the same
        assert L.gsr_set_band(c.h, 0, 3) == _lib.GSR_ERR_STATE
        assert L.gsr_set_row_interleave(c.h, 0, 2) == _lib.GSR_ERR_STATE
        assert L.gsr_group_export(c.h, blob) == _lib.GSR_ERR_STATE
        assert L.gsr_peer_export_framebuffers(c.h, handles) == _lib.GSR_ERR_STATE
        assert L.gsr_peer_import_framebuffers(c.h, handles) == _lib.GSR_ERR_STATE
        _lib.check(L.gsr_set_band(c.h, 0, (H + 15) // 16), "full band")
        _lib.check(L.gsr_set_row_interleave(c.h, 0, 1), "row_mod 1")
        assert c.degree(4) == _lib.GSR_ERR_INVALID and c.degree(-2) == _lib.GSR_ERR_INVALID
        for d in (0, 1, 2, 3, -1):
            _lib.check(c.degree(d), f"degree {d}")
    with ShCtx(n, W, H, 2, HALF) as c:
        assert c.degree(2) == _lib.GSR_ERR_INVALID
        _lib.check(c.degree(1), "degree 1")


@pytest.mark.parametrize("overlap", [0, 1], ids=["serial", "overlap"])
def test_degree_changes_between_async_frames(overlap):
    n = 12288
    t62, vp, ub = scene(n, seed=9)
    splat60 = swizzle_splats(t62, 0.0)
    degrees = [3, 0, 2, -1, 1, 0]
    with ShCtx(n, W, H, 4, HALF) as c:
        c.upload(splat60)
        _lib.check(c.L.gsr_debug_pipeline(c.h, overlap), "gsr_debug_pipeline")
        hosts = [torch.empty((H, W, 4), dtype=torch.float32, pin_memory=True) for _ in degrees]
        for d, hb in zip(degrees, hosts):
            _lib.check(c.degree(d), "gsr_set_sh_degree")
            c.render_async(vp, ub, host_ptr=hb.data_ptr())
        c.sync()
        for d, hb in zip(degrees, hosts):
            ref = oracle_frame(rounded(splat60, 4 if d < 0 else d + 1), vp, ub)
            np.testing.assert_array_equal(bits(hb.numpy()), bits(ref["rgba"]), err_msg=f"degree {d}")
