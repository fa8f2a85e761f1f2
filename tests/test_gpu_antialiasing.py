"""Anti-aliased trainings on the GPU (include/gsr.h gsr_set_antialiasing, gsr_upload_ply_filtered), through the C-ABI: every anti-aliased
frame is bit for bit the anti-aliased oracle's (tests/aa_reference), switching the filter off gives the default frame, the setting follows
the frames it was enqueued with, the single-context rules hold, and the filtered ingest stores what its emulation stores."""
import ctypes as C

import numpy as np
import pytest

from godotgaussiansplatting_b200 import _lib
from godotgaussiansplatting_b200 import camera as cam
from godotgaussiansplatting_b200.ply_file import PlyFile, swizzle_splats
from godotgaussiansplatting_b200.rasterizer import GaussianSplattingRasterizer
from godotgaussiansplatting_b200.synthetic import synthetic_ply_table
from oracle import oracle as orc
from tests import aa_reference as aref
from tests import ortho_reference as oref
from tests.scenes import make_scene
from tests.test_antialiasing import mip_table
from tests.test_gpu_sh_degree import ShCtx, check, set_instances
from tests.test_sh_degree import expected_planes, sh_planes, zero_splat_coeffs

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

W, H = 320, 200


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def cloud(n, seed=3):
    t62 = synthetic_ply_table(n, seed)
    t62[:, 55:58] += 0.5
    t62[:, 9:54] += 0.02   # every coefficient non-zero
    return swizzle_splats(t62, 0.0)


def view(width=W, height=H, frame=25):
    _, vp, ub = make_scene(16, 1, width, height, frame=frame)
    return vp, ub


def aa(c, v):
    return c.L.gsr_set_antialiasing(c.h, C.c_float(v))


VARIANTS = ["plain", "heatmap", "uncontracted", "instances", "depth_plane", "orthographic", "v_0.1", "v_2.0"]


@pytest.mark.parametrize("variant", VARIANTS)
def test_frames_are_the_aa_oracle(variant):
    n = 12288
    splat60 = cloud(n)
    v = {"v_0.1": 0.1, "v_2.0": 2.0}.get(variant, 0.3)
    ortho = variant == "orthographic"
    vp, ub = oref.ortho_camera(W, H, size=2.6, near=0.5, far=4.5, frame=25) if ortho else view()
    flags = (_lib.GSR_FLAG_UNCONTRACTED_BLEND if variant == "uncontracted" else 0) | (_lib.GSR_FLAG_ORTHOGRAPHIC if ortho else 0)
    heat = 1.0 if variant == "heatmap" else 0.0
    inst = None
    if variant == "instances":
        from tests.test_instances import SCALED, rigid
        inst = [(0, 5000, rigid(4)), (4000, 6000, SCALED), (n - 301, 301, rigid(5))]
    Z = None
    if variant == "depth_plane":   # an occluding plane: half the frame at the cloud's median view depth
        pr = aref.project(splat60, vp, orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8)), v)
        V = np.asarray(vp, dtype=np.float32)
        r = pr.records[np.unique(pr.values)]
        d = -(((V[2] * r["pos_xy"][:, 0] + V[6] * r["pos_xy"][:, 1]) + V[10] * r["pos_z"]) + V[14] * np.float32(1.0))
        Z = np.full((H, W), np.inf, dtype=np.float32)
        Z[:, W // 2:] = np.median(d)
    ref = aref.oracle_frame(splat60, vp, ub, v, ortho, heat, contract=variant != "uncontracted", inst=inst, scene_depth=Z, depth=Z is not None)
    assert ref["visible"] > 1000
    with ShCtx(n, W, H, 0, flags) as c:
        c.upload(splat60)
        depth = None
        if Z is not None:
            Zt = torch.from_numpy(Z).cuda()
            depth = torch.zeros((H, W), dtype=torch.float32, device="cuda")
            torch.cuda.synchronize()
            _lib.check(c.L.gsr_set_depth_compositing(c.h, C.c_void_p(Zt.data_ptr()), C.c_void_p(depth.data_ptr())), "depth")
        if inst is not None:
            set_instances(c, inst)
        _lib.check(aa(c, v), "gsr_set_antialiasing")
        rgba = c.render(vp, ub, heatmap=heat)
        check(c, rgba, ref, len(ref["records"]))
        if depth is not None:
            c.sync()
            np.testing.assert_array_equal(bits(depth.cpu().numpy()), bits(ref["depth"]))
            assert np.isfinite(ref["depth"]).any()


@pytest.mark.parametrize("degree", [0, 1, 2])
def test_reduced_sh_stores_and_degrees(degree):
    n = 12288
    splat60 = cloud(n, seed=7 + degree)
    vp, ub = view()
    ref = aref.oracle_frame(zero_splat_coeffs(splat60, degree + 1), vp, ub, 0.3)
    with ShCtx(n, W, H, degree + 1) as c:   # a reduced store
        c.upload(splat60)
        _lib.check(aa(c, 0.3), "gsr_set_antialiasing")
        check(c, c.render(vp, ub), ref, n)
    with ShCtx(n, W, H, 4) as c:            # a degree-3 store rendered lower
        c.upload(splat60)
        _lib.check(c.degree(degree), "gsr_set_sh_degree")
        _lib.check(aa(c, 0.3), "gsr_set_antialiasing")
        check(c, c.render(vp, ub), ref, n)


@pytest.mark.parametrize("size", [(1, 1), (17, 13), (321, 181)], ids=["1x1", "17x13", "321x181"])
def test_ragged_frame_sizes(size):
    w, h = size
    n = 12001
    splat60 = cloud(n, seed=5)
    vp, ub = view(w, h)
    ref = aref.oracle_frame(splat60, vp, ub, 0.1)
    with ShCtx(n, w, h) as c:
        c.upload(splat60)
        _lib.check(aa(c, 0.1), "gsr_set_antialiasing")
        check(c, c.render(vp, ub), ref, n)


def test_more_drawn_ids_than_splats_grow_the_capacity():
    from tests.test_instances import rigid
    n = 4096
    splat60, vp, ub = make_scene(n, 3, W, H, frame=5, scale_boost=0.5)
    inst = [(0, n, rigid(30 + k, 0.3, 0.5)) for k in range(6)]   # D = 6 N
    ref = aref.oracle_frame(splat60, vp, ub, 0.3, inst=inst)
    with ShCtx(n, W, H, 0, 0, factor=1) as c:
        c.upload(splat60)
        set_instances(c, inst)
        _lib.check(aa(c, 0.3), "gsr_set_antialiasing")
        rgba = c.render(vp, ub)   # overflows the initial capacity: grows and renders again
        check(c, rgba, ref, len(ref["records"]))


def test_switching_off_gives_the_default_frame_and_resize_keeps_it():
    n = 12288
    splat60 = cloud(n, seed=8)
    vp, ub = view()
    with ShCtx(n, W, H) as a, ShCtx(n, W, H) as b:
        a.upload(splat60)
        b.upload(splat60)
        want = a.render(vp, ub)
        m = int(a.stats().duplicates)
        _lib.check(aa(b, 0.3), "on")
        on = b.render(vp, ub)
        assert not np.array_equal(bits(on), bits(want))
        _lib.check(aa(b, 0.0), "off")
        np.testing.assert_array_equal(bits(b.render(vp, ub)), bits(want))
        for which in (_lib.GSR_BUF_KEYS, _lib.GSR_BUF_VALUES):
            np.testing.assert_array_equal(b.copy(which, m, np.uint32), a.copy(which, m, np.uint32))
        _lib.check(aa(b, 0.3), "on")
        b.resize(W, H)   # keeps the setting
        np.testing.assert_array_equal(bits(b.render(vp, ub)), bits(on))


@pytest.mark.parametrize("overlap", [0, 1], ids=["serial", "overlap"])
def test_setting_changes_between_async_frames(overlap):
    n = 12288
    splat60 = cloud(n, seed=9)
    vs = [0.0, 0.3, 0.1, 0.0, 2.0, 0.3]
    frames = [view(frame=20 + k) for k in range(len(vs))]
    with ShCtx(n, W, H) as c:
        c.upload(splat60)
        _lib.check(c.L.gsr_debug_pipeline(c.h, overlap), "gsr_debug_pipeline")
        hosts = [torch.empty((H, W, 4), dtype=torch.float32, pin_memory=True) for _ in frames]
        for v, (vp, ub), hb in zip(vs, frames, hosts):
            _lib.check(aa(c, v), "gsr_set_antialiasing")
            c.render_async(vp, ub, host_ptr=hb.data_ptr())
        c.sync()
    for k, (v, (vp, ub), hb) in enumerate(zip(vs, frames, hosts)):
        if v:
            want = aref.oracle_frame(splat60, vp, ub, v)["rgba"]
        else:
            want = orc.frame(splat60, vp, orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8)), cap=64 * n).rgba
        np.testing.assert_array_equal(bits(hb.numpy()), bits(want), err_msg=f"frame {k}")


def test_state_rules_and_invalid_variances():
    n = 4096
    splat60 = cloud(n)
    vp, ub = view()
    handles = (C.c_ubyte * 128)()
    blob = (C.c_ubyte * _lib.GSR_GROUP_BLOB_BYTES)()
    with ShCtx(n, W, H) as c:
        c.upload(splat60)
        L = c.L
        want = aref.oracle_frame(splat60, vp, ub, 0.3)
        _lib.check(aa(c, 0.3), "gsr_set_antialiasing")
        for bad in (-0.1, float("nan"), float("inf"), -float("inf"), 64.5):
            assert aa(c, bad) == _lib.GSR_ERR_INVALID
        check(c, c.render(vp, ub), want, n)   # the previous state is kept
        assert aa(c, 64.0) == _lib.GSR_OK and aa(c, 0.3) == _lib.GSR_OK
        # while the filter is on, the multi-context calls are refused
        assert L.gsr_set_band(c.h, 0, 3) == _lib.GSR_ERR_STATE
        assert L.gsr_set_row_interleave(c.h, 0, 2) == _lib.GSR_ERR_STATE
        assert L.gsr_peer_export_framebuffers(c.h, handles) == _lib.GSR_ERR_STATE
        assert L.gsr_peer_import_framebuffers(c.h, handles) == _lib.GSR_ERR_STATE
        assert L.gsr_group_export(c.h, blob) == _lib.GSR_ERR_STATE
        check(c, c.render(vp, ub), want, n)
        # and turning it on is refused on a multi-context setup
        _lib.check(aa(c, 0.0), "off")
        for setup, undo in ((lambda: L.gsr_set_band(c.h, 0, 3), lambda: L.gsr_set_band(c.h, 0, (H + 15) // 16)),
                            (lambda: L.gsr_set_row_interleave(c.h, 0, 2), lambda: L.gsr_set_row_interleave(c.h, 0, 1)),
                            (lambda: L.gsr_peer_export_framebuffers(c.h, handles), lambda: L.gsr_resize(c.h, W, H))):
            _lib.check(setup(), "setup")
            assert aa(c, 0.3) == _lib.GSR_ERR_STATE
            assert aa(c, 0.0) == _lib.GSR_OK
            _lib.check(undo(), "undo")
        _lib.check(aa(c, 0.3), "on")
        check(c, c.render(vp, ub), want, n)


def test_filtered_upload_stores_the_emulated_ingest():
    n, stride = 3000, 3072
    table, names = mip_table(n, seed=6)
    lay = PlyFile.from_array(table, names).layout()
    glay = _lib.GsrPlyLayout(lay.nprops, lay.sh_degree, lay.x, lay.f_dc, lay.f_rest, lay.opacity, lay.scale, lay.rot)
    ptr = table.ctypes.data_as(C.POINTER(C.c_float))
    want = aref.emu_ply_to_soa(table, lay, 0.0, 15, stride)
    np.testing.assert_array_equal(bits(want[:, :n]), bits(expected_planes(swizzle_splats(table, 0.0, lay), 4, n)))
    with ShCtx(n, W, H) as c:
        size = 15 * stride * 4
        _lib.check(c.L.gsr_upload_ply_filtered(c.h, ptr, C.byref(glay), lay.filter_3d, 0, n, 0.0), "gsr_upload_ply_filtered")
        got = c.copy(_lib.GSR_BUF_SPLATS, size, np.float32).reshape(15, stride, 4)
        np.testing.assert_array_equal(bits(got[:, :n]), bits(want[:, :n]))
        # filter_3d = -1 is gsr_upload_ply, byte for byte
        _lib.check(c.L.gsr_upload_ply(c.h, ptr, C.byref(glay), 0, n, 0.0), "gsr_upload_ply")
        plain = c.copy(_lib.GSR_BUF_SPLATS, size, np.uint8)
        _lib.check(c.L.gsr_upload_ply_filtered(c.h, ptr, C.byref(glay), lay.filter_3d, 0, n, 0.0), "filtered again")
        _lib.check(c.L.gsr_upload_ply_filtered(c.h, ptr, C.byref(glay), -1, 0, n, 0.0), "gsr_upload_ply_filtered(-1)")
        np.testing.assert_array_equal(c.copy(_lib.GSR_BUF_SPLATS, size, np.uint8), plain)
        for bad in (-2, lay.nprops, 1000):
            assert c.L.gsr_upload_ply_filtered(c.h, ptr, C.byref(glay), bad, 0, n, 0.0) == _lib.GSR_ERR_INVALID
    with ShCtx(n, W, H, 2) as c:   # a reduced store keeps the first planes of the same splats
        _lib.check(c.L.gsr_upload_ply_filtered(c.h, ptr, C.byref(glay), lay.filter_3d, 0, n, 0.0), "gsr_upload_ply_filtered")
        got = c.copy(_lib.GSR_BUF_SPLATS, (3 + sh_planes(2)) * stride * 4, np.float32).reshape(-1, stride, 4)
        np.testing.assert_array_equal(bits(got[:, :n]), bits(aref.emu_ply_to_soa(table, lay, 0.0, 3 + sh_planes(2), stride)[:, :n]))


@pytest.mark.parametrize("device_ingest", [False, True], ids=["host", "device"])
def test_mip_splatting_ply_renders_through_the_rasterizer(device_ingest):
    n = 12288
    t62 = synthetic_ply_table(n, 12)
    t62[:, 55:58] += 0.5
    f = np.random.default_rng(12).uniform(0.0, 0.02, n).astype(np.float32)
    names = [f"{p}" for p in PlyFile.from_array(t62).properties] + ["filter_3D"]
    table = np.concatenate([t62, f[:, None]], axis=1)
    ply = PlyFile.from_array(table, names)
    camera = cam.orbit_camera(25, aspect=W / H)
    r = GaussianSplattingRasterizer(ply, (W, H), None, camera)
    assert r._antialiasing == 0.1
    r.init_gpu(device_ingest=device_ingest)
    try:
        out = np.empty((H, W, 4), dtype=np.float32)
        r.rasterize(time=10.0, out_host=out)
        vp = r.camera_push_constants
        ub = r.uniforms_bytes(10.0)
        ref = aref.oracle_frame(swizzle_splats(table, 0.0, ply.layout()), vp, ub, 0.1)
        assert ref["visible"] > 1000
        np.testing.assert_array_equal(bits(out), bits(ref["rgba"]))
    finally:
        r.cleanup_gpu()
