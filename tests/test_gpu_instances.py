"""Splat instances on the GPU (include/gsr.h gsr_set_instances), through the C-ABI: the identity instance against the default frame,
instanced frames against the instance oracle (tests/instance_reference) bit for bit, per-frame motion without host syncs, the Godot
transform convention against a moved camera, pick, and the state rules."""
import ctypes as C

import numpy as np
import pytest

from godotgaussiansplatting_b200 import _lib
from godotgaussiansplatting_b200 import camera as cam
from godotgaussiansplatting_b200.rasterizer import godot_to_frame
from oracle import oracle as orc
from tests import depth_reference as dref
from tests import instance_reference as iref
from tests.gsr_direct import REC_DTYPE, Ctx
from tests.scenes import make_scene, uniforms_bytes
from tests.test_instances import IDENTITY, SCALED, SHEARED, rigid, rotation, to_frame

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def uniforms(ub):
    return orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8))


def set_instances(c, inst):
    arr = (_lib.GsrInstance * max(1, len(inst)))()
    for k, (first, count, xf12) in enumerate(inst):
        arr[k].first, arr[k].count = int(first), int(count)
        arr[k].to_frame[:] = [float(v) for v in np.asarray(xf12, dtype=np.float32)]
    return c.L.gsr_set_instances(c.h, arr, len(inst))


def library_xf(c, n):
    return c.copy(_lib.GSR_BUF_INSTANCES, 24 * n, np.float32).reshape(n, 24)


def taps(c, drawn):
    """The stage outputs of the last frame (GSR_BUF_RECORDS holds D records in instanced mode)."""
    st = c.stats()
    m = int(min(st.duplicates, st.capacity))
    T = st.tiles_x * st.tiles_y
    return dict(stats=st, m=m, records=c.copy(_lib.GSR_BUF_RECORDS, drawn, REC_DTYPE), keys=c.copy(_lib.GSR_BUF_KEYS, m, np.uint32),
                values=c.copy(_lib.GSR_BUF_VALUES, m, np.uint32), bounds=c.copy(_lib.GSR_BUF_BOUNDS, T * 2, np.uint32).reshape(T, 2))


def check_against_oracle(c, splat60, vp, ub, inst, rgba, heat=0.0, depth=None, scene_depth=None, contract=True):
    ranges = [(f, n) for f, n, _ in inst]
    xf = library_xf(c, len(inst))
    for k, (_, _, x) in enumerate(inst):   # the library's A|t is the caller's, its inverse the float64 one rounded (up to the sign of zero)
        np.testing.assert_array_equal(bits(xf[k, :12]), bits(np.asarray(x, dtype=np.float32)))
        np.testing.assert_allclose(xf[k, 12:], iref.inverse(x)[12:], rtol=2e-7, atol=1e-7)
    ref = iref.frame(splat60, vp, uniforms(ub), ranges, xf, heatmap=heat, depth=depth is not None, scene_depth=scene_depth, contract=contract)
    np.testing.assert_array_equal(bits(rgba), bits(ref.rgba))
    t = taps(c, ref.proj.drawn)
    assert t["stats"].duplicates == ref.proj.duplicates and t["stats"].visible == ref.proj.visible
    assert t["stats"].staged == ref.staged and not t["stats"].overflow
    np.testing.assert_array_equal(t["keys"], ref.keys)
    np.testing.assert_array_equal(t["values"], ref.values)
    np.testing.assert_array_equal(t["bounds"], ref.bounds)
    ids = np.unique(ref.values)
    np.testing.assert_array_equal(bits(t["records"][ids].view(np.float32)), bits(ref.proj.records[ids].view(np.float32)))
    if depth is not None:
        c.sync()
        np.testing.assert_array_equal(bits(depth.cpu().numpy()), bits(ref.depth))
    return ref


N, W, H = 16384, 320, 200


@pytest.mark.parametrize("mode", ["spec", "uncontracted", "depth"])
def test_identity_instance_is_the_default_frame(mode):
    flags = _lib.GSR_FLAG_UNCONTRACTED_BLEND if mode == "uncontracted" else 0
    splat60, vp, ub = make_scene(N, 1, W, H, frame=40, scale_boost=0.5)
    with Ctx(N, W, H, flags=flags) as c:
        c.upload(splat60)
        depth = None
        if mode == "depth":
            depth = torch.zeros((H, W), dtype=torch.float32, device="cuda")
            torch.cuda.synchronize()
            _lib.check(c.L.gsr_set_depth_compositing(c.h, None, C.c_void_p(depth.data_ptr())), "gsr_set_depth_compositing")
        plain = c.render(vp, ub)
        base = taps(c, N)
        d0 = depth.cpu().numpy() if depth is not None else None
        _lib.check(set_instances(c, [(0, N, IDENTITY)]), "gsr_set_instances")
        got = c.render(vp, ub)
        t = taps(c, N)
        np.testing.assert_array_equal(bits(got), bits(plain))
        for k in ("keys", "values", "bounds"):
            np.testing.assert_array_equal(t[k], base[k])
        ids = np.unique(base["values"])
        assert (t["records"][ids].view(np.float32) == base["records"][ids].view(np.float32)).all()   # +-0 compare equal
        if depth is not None:
            c.sync()
            np.testing.assert_array_equal(bits(depth.cpu().numpy()), bits(d0))


def cases():
    q = N // 4
    return {
        "rigid": ([(0, N, rigid(3))], {}),
        "scaled": ([(0, N, SCALED)], {}),
        "sheared": ([(0, N, SHEARED)], {}),
        "three_disjoint": ([(0, 5000, rigid(4)), (5000, 6000, SCALED), (11000, N - 11000, rigid(5))], {}),
        "asset_x4": ([(0, q, to_frame(np.eye(3), [dx, dy, 0.0])) for dx, dy in ((0, 0), (0.6, 0), (0, 0.5), (0.6, 0.5))], {}),
        "ragged_tail": ([(100 * i + 3, c, rigid(20 + i)) for i, c in enumerate((1, 31, 32, 33, 257, 0))] + [(N - 301, 301, rigid(8))], {}),
        "heatmap": ([(0, 8000, rigid(6)), (4000, 8000, rigid(7))], dict(heat=1.0)),
        "depth_plane": ([(0, 8000, rigid(9)), (8000, 8000, SCALED)], dict(depth=True)),
    }


@pytest.mark.parametrize("case", list(cases()))
def test_frames_are_the_instance_oracle(case):
    inst, kw = cases()[case]
    splat60, vp, ub = make_scene(N, 2, W, H, frame=25, scale_boost=0.5)
    with Ctx(N, W, H) as c:
        c.upload(splat60)
        depth = Z = None
        if kw.get("depth"):
            probe = iref.project(splat60, vp, uniforms(ub), [(f, n) for f, n, _ in inst], np.stack([iref.inverse(x) for _, _, x in inst]))
            V = np.asarray(vp, dtype=np.float32)
            r = probe.records[np.unique(probe.values)]
            d = -(((V[2] * r["pos_xy"][:, 0] + V[6] * r["pos_xy"][:, 1]) + V[10] * r["pos_z"]) + V[14] * np.float32(1.0))
            Z = np.full((H, W), np.inf, dtype=np.float32)
            Z[:, W // 2:] = np.median(d)   # an occluding plane over the right half
            Zt = torch.from_numpy(Z).cuda()
            depth = torch.zeros((H, W), dtype=torch.float32, device="cuda")
            torch.cuda.synchronize()
            _lib.check(c.L.gsr_set_depth_compositing(c.h, C.c_void_p(Zt.data_ptr()), C.c_void_p(depth.data_ptr())), "depth")
        _lib.check(set_instances(c, inst), "gsr_set_instances")
        rgba = c.render(vp, ub, heatmap=kw.get("heat", 0.0))
        ref = check_against_oracle(c, splat60, vp, ub, inst, rgba, heat=kw.get("heat", 0.0), depth=depth, scene_depth=Z)
        assert ref.proj.visible > 0


def test_more_drawn_ids_than_splats_grow_the_capacity():
    n = 4096
    splat60, vp, ub = make_scene(n, 3, W, H, frame=5, scale_boost=0.5)
    inst = [(0, n, rigid(30 + k, 0.3, 0.5)) for k in range(6)]   # D = 6 N
    with Ctx(n, W, H, factor=1) as c:
        c.upload(splat60)
        _lib.check(set_instances(c, inst), "gsr_set_instances")
        assert c.stats().capacity >= 6 * n
        rgba = c.render(vp, ub)   # overflows the initial capacity: grows and renders again
        check_against_oracle(c, splat60, vp, ub, inst, rgba)
        hosts = [torch.empty((H, W, 4), dtype=torch.float32, pin_memory=True) for _ in range(3)]
        for hb in hosts:
            c.render_async(vp, ub, host_ptr=hb.data_ptr())
        c.sync()
        np.testing.assert_array_equal(bits(hosts[-1].numpy()), bits(rgba))


@pytest.mark.parametrize("overlap", [0, 1], ids=["serial", "overlap"])
def test_per_frame_motion_without_host_sync(overlap):
    n = 8192
    splat60, vp, ub = make_scene(n, 4, W, H, frame=60, scale_boost=0.5)
    frames = [[(0, 4096, rigid(40 + f)), (2048, 4096, rigid(50 + f)), (4096, 4096, to_frame(rotation([0, 1, 0], 0.2 * f), [0.1 * f, 0, 0]))]
              for f in range(5)]
    with Ctx(n, W, H) as c:
        c.upload(splat60)
        _lib.check(c.L.gsr_debug_pipeline(c.h, overlap), "gsr_debug_pipeline")
        _lib.check(set_instances(c, frames[0]), "gsr_set_instances")   # the layout (may synchronise)
        hosts = [torch.empty((H, W, 4), dtype=torch.float32, pin_memory=True) for _ in frames]
        for inst, hb in zip(frames, hosts):
            _lib.check(set_instances(c, inst), "gsr_set_instances")   # same layout: transforms only
            c.render_async(vp, ub, host_ptr=hb.data_ptr())
        c.sync()
        for f, (inst, hb) in enumerate(zip(frames, hosts)):
            ref = iref.frame(splat60, vp, uniforms(ub), [(a, b) for a, b, _ in inst], np.stack([iref.inverse(x) for _, _, x in inst]))
            np.testing.assert_array_equal(bits(hb.numpy()), bits(ref.rgba), err_msg=f"frame {f}")


def test_godot_transform_equals_the_inverse_camera():
    n, w, h = 12000, 256, 160
    splat60, _, _ = make_scene(n, 5, w, h, scale_boost=0.4)
    camera = cam.orbit_camera(20, aspect=w / h)
    R = rotation([0.1, 1.0, 0.2], 0.35)
    o = np.array([0.2, -0.1, 0.3])
    T = np.hstack([R, o[:, None]])
    # the camera T^-1 C: basis R^T * basis, position R^T (p - o)
    moved = cam.orbit_camera(20, aspect=w / h)
    moved.basis = (camera.basis.astype(np.float64) @ R).astype(np.float32)
    moved.global_position = (R.T @ (camera.global_position.astype(np.float64) - o)).astype(np.float32)
    vp = cam.pack_camera_push_constants(camera.get_camera_transform(), camera.get_camera_projection())
    vp2 = cam.pack_camera_push_constants(moved.get_camera_transform(), moved.get_camera_projection())
    ub, ub2 = uniforms_bytes(camera.global_position, 1.0, w, h, 10.0), uniforms_bytes(moved.global_position, 1.0, w, h, 10.0)
    with Ctx(n, w, h) as c:
        c.upload(splat60)
        want = c.render(vp2, ub2)
        _lib.check(set_instances(c, [(0, n, godot_to_frame(T, np.eye(3)).T.reshape(12))]), "gsr_set_instances")
        got = c.render(vp, ub)
    err = np.abs(got - want).max(axis=2)
    assert float((err <= 1e-3).mean()) >= 0.999
    assert want[..., :3].max() > 0.1


def test_pick_returns_the_frame_space_position_of_a_moved_instance():
    n = 8192
    splat60, vp, ub = make_scene(n, 6, W, H, frame=0, scale_boost=0.5)
    xf12 = rigid(70)
    with Ctx(n, W, H) as c:
        c.upload(splat60)
        _lib.check(set_instances(c, [(0, n, xf12)]), "gsr_set_instances")
        c.render(vp, ub)
        t = taps(c, n)
        lengths = t["bounds"][:, 1].astype(np.int64) - t["bounds"][:, 0].astype(np.int64)
        tile = int(np.argmax(lengths))
        p = c.pick(tile)
    assert p[3] > 0
    xf = iref.inverse(xf12)
    ids = np.unique(t["values"])
    w = np.stack([t["records"][ids]["pos_xy"][:, 0], t["records"][ids]["pos_xy"][:, 1], t["records"][ids]["pos_z"]], axis=1)
    hit = np.where((w == p[:3]).all(axis=1))[0]
    assert hit.size, "pick returned no record position"
    src = splat60[ids[hit[0]], :3][None]
    np.testing.assert_array_equal(bits(p[:3]), bits(iref.frame_position(xf, src)[0]))
    # back to Godot coordinates (basis_override = identity): F * frame position, the moved source splat
    godot = np.array([-p[0], -p[1], p[2]], dtype=np.float64)
    A, tt = xf[:9].astype(np.float64).reshape(3, 3).T, xf[9:12].astype(np.float64)
    F = np.diag([-1.0, -1.0, 1.0])
    np.testing.assert_allclose(godot, F @ (A @ src[0].astype(np.float64) + tt), atol=1e-5)


def test_state_rules_invalid_inputs_and_switching_off():
    n, w, h = 4096, 96, 64
    splat60, vp, ub = make_scene(n, 7, w, h)
    with Ctx(n, w, h) as fresh:
        fresh.upload(splat60)
        never = fresh.render(vp, ub)
    with Ctx(n, w, h) as c:
        c.upload(splat60)
        L = c.L
        inst = [(0, 2048, rigid(80)), (1024, 2048, rigid(81))]
        # not on a sharded context
        c.set_band(0, 2)
        assert set_instances(c, inst) == _lib.GSR_ERR_STATE
        c.set_band(0, 4)
        c.set_row_interleave(1, 2)
        assert set_instances(c, inst) == _lib.GSR_ERR_STATE
        c.set_row_interleave(0, 1)
        _lib.check(set_instances(c, inst), "gsr_set_instances")
        # ... and no sharding while instances are set
        assert L.gsr_set_band(c.h, 1, 3) == _lib.GSR_ERR_STATE
        assert L.gsr_set_row_interleave(c.h, 0, 2) == _lib.GSR_ERR_STATE
        handles = (C.c_ubyte * 128)()
        assert L.gsr_peer_export_framebuffers(c.h, handles) == _lib.GSR_ERR_STATE
        assert L.gsr_peer_import_framebuffers(c.h, handles) == _lib.GSR_ERR_STATE
        blob = c.group_export()
        buf = (C.c_ubyte * (2 * len(blob))).from_buffer_copy(blob + blob)
        assert L.gsr_group_attach(c.h, 0, 2, buf) == _lib.GSR_ERR_STATE
        before = c.render(vp, ub)
        xf_before = library_xf(c, 2)
        # invalid inputs: rejected, previous state kept
        bad = [
            [(0, n + 1, IDENTITY)],                                    # beyond max_splats
            [(n - 10, 11, IDENTITY)],
            [(0, 100, to_frame(np.zeros((3, 3)), [0, 0, 0]))],         # singular
            [(0, 100, to_frame(np.eye(3), [np.nan, 0, 0]))],           # non-finite
            [(0, 100, to_frame(np.eye(3), [np.inf, 0, 0]))],
        ]
        for b in bad:
            assert set_instances(c, b) == _lib.GSR_ERR_INVALID, b
        big = (_lib.GsrInstance * (_lib.GSR_MAX_INSTANCES + 1))()
        for k in range(_lib.GSR_MAX_INSTANCES + 1):
            big[k].count, big[k].to_frame[:] = 1, [float(v) for v in IDENTITY]
        assert L.gsr_set_instances(c.h, big, _lib.GSR_MAX_INSTANCES + 1) == _lib.GSR_ERR_INVALID
        np.testing.assert_array_equal(bits(library_xf(c, 2)), bits(xf_before))
        np.testing.assert_array_equal(bits(c.render(vp, ub)), bits(before))
        # resize keeps the instances
        c.resize(w, h)
        np.testing.assert_array_equal(bits(c.render(vp, ub)), bits(before))
        # off: the frame of a context that never used instances; the sharding calls work again
        _lib.check(set_instances(c, []), "gsr_set_instances(n = 0)")
        np.testing.assert_array_equal(bits(c.render(vp, ub)), bits(never))
        c.set_band(1, 3)
        c.set_band(0, 4)
