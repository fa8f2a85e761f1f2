"""Orthographic cameras on the GPU (include/gsr.h GSR_FLAG_ORTHOGRAPHIC), through the C-ABI: every orthographic frame is bit for bit
the orthographic oracle's (tests/ortho_reference), perspective frames of a flagged context are the unflagged context's, and the
single-context rules hold."""
import ctypes as C

import numpy as np
import pytest

from godotgaussiansplatting_b200 import _lib
from godotgaussiansplatting_b200 import camera as cam
from godotgaussiansplatting_b200.ply_file import swizzle_splats
from godotgaussiansplatting_b200.synthetic import synthetic_ply_table
from oracle import oracle as orc
from tests import ortho_reference as oref
from tests.gsr_direct import Ctx
from tests.scenes import make_scene
from tests.test_gpu_sh_degree import ShCtx, check, set_instances
from tests.test_sh_degree import zero_splat_coeffs

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

ORTHO = _lib.GSR_FLAG_ORTHOGRAPHIC
W, H = 320, 200


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def cloud(n, seed=3):
    t62 = synthetic_ply_table(n, seed)
    t62[:, 55:58] += 0.5
    t62[:, 9:54] += 0.02   # every coefficient non-zero
    return swizzle_splats(t62, 0.0)


def ortho_view(width, height, frame=25, size=2.6, near=0.5, far=4.5):
    return oref.ortho_camera(width, height, size=size, near=near, far=far, frame=frame)


def test_c2_view_renders_the_cloud_that_perspective_culls():
    """The synthetic cloud 2.5 units in front of the default camera at 320x180, size 4, Godot's default near / far."""
    splat60, _, _ = make_scene(20000, 2, 320, 180)
    vp, ub = oref.ortho_camera(320, 180, size=4.0, near=0.05, far=4000.0)
    ref = oref.oracle_frame(splat60, vp, ub)
    assert ref["visible"] > 19000
    np.testing.assert_array_equal(bits(oref.frame(splat60, vp, ub)["rgba"]), bits(ref["rgba"]))
    with ShCtx(20000, 320, 180, 0, ORTHO) as c:
        c.upload(splat60)
        rgba = c.render(vp, ub)
        check(c, rgba, ref, 20000)
        assert (rgba[..., :3] > 0).any()
    with Ctx(20000, 320, 180) as c:   # without the flag: the perspective path, which culls the whole cloud (the parent's behaviour)
        c.upload(splat60)
        rgba = c.render(vp, ub)
        assert c.stats().visible == 0 and not rgba[..., :3].any()


VARIANTS = ["plain", "heatmap", "uncontracted", "instances", "depth_plane", "far_4000"]


@pytest.mark.parametrize("variant", VARIANTS)
def test_frames_are_the_ortho_oracle(variant):
    n = 12288
    splat60 = cloud(n)
    vp, ub = ortho_view(W, H, far=4000.0 if variant == "far_4000" else 4.5)
    flags = ORTHO | (_lib.GSR_FLAG_UNCONTRACTED_BLEND if variant == "uncontracted" else 0)
    heat = 1.0 if variant == "heatmap" else 0.0
    inst = None
    if variant == "instances":
        from tests.test_instances import SCALED, rigid
        inst = [(0, 5000, rigid(4)), (4000, 6000, SCALED), (n - 301, 301, rigid(5))]
    Z = None
    if variant == "depth_plane":   # an occluding plane given as orthographic linear depth: half the frame at the cloud's median depth
        pr = oref.project(splat60, vp, orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8)))
        V = np.asarray(vp, dtype=np.float32)
        r = pr.records[np.unique(pr.values)]
        d = -(((V[2] * r["pos_xy"][:, 0] + V[6] * r["pos_xy"][:, 1]) + V[10] * r["pos_z"]) + V[14] * np.float32(1.0))
        Z = np.full((H, W), np.inf, dtype=np.float32)
        Z[:, W // 2:] = np.median(d)
    ref = oref.oracle_frame(splat60, vp, ub, heat, contract=variant != "uncontracted", inst=inst, scene_depth=Z, depth=Z is not None)
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
        rgba = c.render(vp, ub, heatmap=heat)
        check(c, rgba, ref, len(ref["records"]))
        if depth is not None:
            c.sync()
            np.testing.assert_array_equal(bits(depth.cpu().numpy()), bits(ref["depth"]))
            assert np.isfinite(ref["depth"]).any()


@pytest.mark.parametrize("size", [(1, 1), (17, 13), (321, 181)], ids=["1x1", "17x13", "321x181"])
def test_ragged_frame_sizes(size):
    w, h = size
    n = 12001
    splat60 = cloud(n, seed=5)
    vp, ub = ortho_view(w, h)
    ref = oref.oracle_frame(splat60, vp, ub)
    with ShCtx(n, w, h, 0, ORTHO) as c:
        c.upload(splat60)
        check(c, c.render(vp, ub), ref, n)


@pytest.mark.parametrize("degree", [0, 1, 2])
def test_reduced_sh_stores_and_degrees(degree):
    n = 12288
    splat60 = cloud(n, seed=7 + degree)
    vp, ub = ortho_view(W, H)
    ref = oref.oracle_frame(zero_splat_coeffs(splat60, degree + 1), vp, ub)
    with ShCtx(n, W, H, degree + 1, ORTHO) as c:   # a reduced store
        c.upload(splat60)
        check(c, c.render(vp, ub), ref, n)
    with ShCtx(n, W, H, 4, ORTHO) as c:            # a degree-3 store rendered lower
        c.upload(splat60)
        _lib.check(c.degree(degree), "gsr_set_sh_degree")
        check(c, c.render(vp, ub), ref, n)


def test_pick():
    n = 12288
    splat60 = cloud(n, seed=6)
    vp, ub = ortho_view(W, H)
    ref = oref.oracle_frame(splat60, vp, ub)
    lengths = ref["bounds"][:, 1].astype(np.int64) - ref["bounds"][:, 0].astype(np.int64)
    with ShCtx(n, W, H, 0, ORTHO) as c:
        c.upload(splat60)
        c.render(vp, ub)
        busy = np.where(lengths > 0)[0]
        for tile in (int(np.argmax(lengths)), int(busy[np.argsort(lengths[busy])[len(busy) // 2]])):
            _, _, want = orc.render(ref["records"], ref["values"], ref["bounds"], W, H, 0.0, target_tile=tile, pick=np.zeros(4, np.float32))
            assert want[3] > 0   # the oracle picks a splat in this tile (a tile whose sampled pixels are empty leaves the buffer as it was)
            np.testing.assert_array_equal(bits(c.pick(tile)), bits(want))


@pytest.mark.parametrize("overlap", [0, 1], ids=["serial", "overlap"])
def test_perspective_and_orthographic_frames_alternate(overlap):
    n = 12288
    splat60 = cloud(n, seed=9)
    frames = []
    for k in range(6):
        if k % 2:
            frames.append(ortho_view(W, H, frame=20 + k, size=2.2 + 0.2 * k))
        else:
            _, vp, ub = make_scene(16, 1, W, H, frame=20 + k)
            frames.append((vp, ub))
    with ShCtx(n, W, H, 0, ORTHO) as c:
        c.upload(splat60)
        _lib.check(c.L.gsr_debug_pipeline(c.h, overlap), "gsr_debug_pipeline")
        hosts = [torch.empty((H, W, 4), dtype=torch.float32, pin_memory=True) for _ in frames]
        for (vp, ub), hb in zip(frames, hosts):
            c.render_async(vp, ub, host_ptr=hb.data_ptr())
        c.sync()
    for k, ((vp, ub), hb) in enumerate(zip(frames, hosts)):
        if k % 2:
            want = oref.oracle_frame(splat60, vp, ub)["rgba"]
        else:
            assert not oref.is_orthographic(vp)
            want = orc.frame(splat60, vp, orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8)), cap=64 * n).rgba
        np.testing.assert_array_equal(bits(hb.numpy()), bits(want), err_msg=f"frame {k}")


def test_flagged_perspective_frames_are_the_unflagged_ones():
    n = 12288
    splat60 = cloud(n, seed=10)
    c0 = cam.orbit_camera(30, aspect=W / H)
    proj = c0.get_camera_projection()
    views = [cam.pack_camera_push_constants(c0.get_camera_transform(), proj),
             cam.pack_camera_push_constants(c0.get_camera_transform(), proj, keep_w_row=True)]
    _, _, ub = make_scene(16, 1, W, H, frame=30)
    for flags in (0, _lib.GSR_FLAG_UNCONTRACTED_BLEND):
        with ShCtx(n, W, H, 0, flags) as a, ShCtx(n, W, H, 0, flags | ORTHO) as b:
            a.upload(splat60)
            b.upload(splat60)
            for vp in views:
                want = a.render(vp, ub)
                np.testing.assert_array_equal(bits(b.render(vp, ub)), bits(want))
                m = int(a.stats().duplicates)
                for which in (_lib.GSR_BUF_KEYS, _lib.GSR_BUF_VALUES):
                    np.testing.assert_array_equal(b.copy(which, m, np.uint32), a.copy(which, m, np.uint32))
            # an orthographic matrix packed the reference's way is a perspective frame on both
            o = cam.pack_camera_push_constants(c0.get_camera_transform(), cam.orthogonal(2.6, W / H, 0.5, 4.5))
            np.testing.assert_array_equal(bits(b.render(o, ub)), bits(a.render(o, ub)))


def test_state_rules():
    n = 4096
    splat60 = cloud(n)
    vp, ub = ortho_view(W, H)
    _, pvp, pub = make_scene(16, 1, W, H, frame=25)
    handles = (C.c_ubyte * 128)()
    with ShCtx(n, W, H, 0, ORTHO) as c:
        c.upload(splat60)
        L = c.L
        vpp = np.ascontiguousarray(vp, dtype=np.float32).ctypes.data_as(C.POINTER(C.c_float))
        want = oref.oracle_frame(splat60, vp, ub)
        for setup, undo in ((lambda: L.gsr_set_band(c.h, 0, 3), lambda: L.gsr_set_band(c.h, 0, (H + 15) // 16)),
                            (lambda: L.gsr_set_row_interleave(c.h, 0, 2), lambda: L.gsr_set_row_interleave(c.h, 0, 1)),
                            (lambda: L.gsr_peer_export_framebuffers(c.h, handles), lambda: L.gsr_resize(c.h, W, H))):
            _lib.check(setup(), "setup")
            assert L.gsr_render(c.h, vpp, ub, 0.0, None) == _lib.GSR_ERR_STATE
            assert L.gsr_render_async(c.h, vpp, ub, 0.0, None) == _lib.GSR_ERR_STATE
            _lib.check(L.gsr_render_async(c.h, np.ascontiguousarray(pvp).ctypes.data_as(C.POINTER(C.c_float)), pub, 0.0, None),
                       "a perspective frame is unaffected")
            c.sync()
            _lib.check(undo(), "undo")
            check(c, c.render(vp, ub), want, n)
