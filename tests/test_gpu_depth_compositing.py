"""Depth compositing on the GPU (include/gsr.h gsr_set_depth_compositing): composite_kernel<CONTRACT, true> against the oracle, bit for
bit, with torch CUDA tensors as the caller's scene-depth and depth-output planes; the default frame around it; the state rules."""
import ctypes as C

import numpy as np
import pytest

from godotgaussiansplatting_b200 import _lib
from oracle import oracle as orc
from tests import depth_reference as dref
from tests.gsr_direct import Ctx
from tests.scenes import make_scene

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def uniforms(ub):
    return orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8))


def splat_depths(records, vp):
    V = np.asarray(vp, dtype=np.float32)
    return -(((V[2] * records["pos_xy"][:, 0] + V[6] * records["pos_xy"][:, 1]) + V[10] * records["pos_z"]) + V[14] * np.float32(1.0))


class DepthPlanes:
    """The caller's device planes: scene depth (optional) and depth output, as torch CUDA tensors."""

    def __init__(self, w, h, Z=None):
        self.Z = None if Z is None else torch.from_numpy(np.ascontiguousarray(Z, dtype=np.float32)).cuda()
        self.out = torch.full((h, w), float("nan"), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()

    def enable(self, c):
        return c.L.gsr_set_depth_compositing(c.h, C.c_void_p(None if self.Z is None else self.Z.data_ptr()), C.c_void_p(self.out.data_ptr()))

    def read(self, c):
        c.sync()
        return self.out.cpu().numpy()


def disable(c):
    _lib.check(c.L.gsr_set_depth_compositing(c.h, None, None), "gsr_set_depth_compositing")


def plane(kind, w, h, d, seed=0):
    if kind == "none":
        return None
    if kind == "front":                      # in front of everything: nothing shows
        return np.zeros((h, w), dtype=np.float32)
    if kind == "half":                       # the lower half of the frame behind a plane at the median splat depth
        Z = np.full((h, w), np.inf, dtype=np.float32)
        Z[h // 2:] = np.median(d)
        return Z
    rng = np.random.default_rng(seed)        # per-pixel random depths with +inf, 0 and NaN mixed in
    Z = rng.uniform(d.min(), d.max(), size=(h, w)).astype(np.float32)
    p = rng.random((h, w))
    Z[p < 0.1] = np.inf
    Z[(p >= 0.1) & (p < 0.2)] = 0.0
    Z[(p >= 0.2) & (p < 0.3)] = np.nan
    return Z


#                   n      seed w    h    heat  flags                              scene kwargs
CASES = {
    "default_cam": (20000, 1, 640, 480, 0.0, 0, dict()),
    "orbit_ragged_heat": (9000, 5, 250, 130, 1.0, 0, dict(frame=37, scale_boost=0.5)),
    "load_in": (6000, 7, 192, 160, 0.0, 0, dict(time=0.6, scale_boost=1.0)),
    "uncontracted": (12000, 3, 333, 201, 0.0, _lib.GSR_FLAG_UNCONTRACTED_BLEND, dict(frame=80, scale_boost=1.0)),
}


@pytest.mark.parametrize("case", list(CASES))
def test_depth_frames_are_the_oracles_and_the_default_frame_is_unchanged(case):
    n, seed, w, h, heat, flags, kw = CASES[case]
    splat60, vp, ub = make_scene(n, seed, w, h, **kw)
    contract = not (flags & _lib.GSR_FLAG_UNCONTRACTED_BLEND)
    orc.set_blend_contraction(contract)
    try:
        base = orc.frame(splat60, vp, uniforms(ub), heatmap=heat, cap=1000 * n)
        d = splat_depths(base.records[base.values], vp)
        with Ctx(n, w, h, flags=flags) as c:
            c.upload(splat60)
            plain = c.render(vp, ub, heatmap=heat)
            np.testing.assert_array_equal(bits(plain), bits(base.rgba))
            for kind in ("none", "half", "mixed", "front"):
                Z = plane(kind, w, h, d, seed)
                ref = dref.frame_depth(splat60, vp, uniforms(ub), heatmap=heat, cap=1000 * n, scene_depth=Z, contract=contract)
                planes = DepthPlanes(w, h, Z)
                _lib.check(planes.enable(c), "gsr_set_depth_compositing")
                rgba = c.render(vp, ub, heatmap=heat)
                depth = planes.read(c)
                np.testing.assert_array_equal(bits(rgba), bits(ref.rgba), err_msg=f"rgba, plane {kind}")
                np.testing.assert_array_equal(bits(depth), bits(ref.depth), err_msg=f"depth, plane {kind}")
                assert c.stats().staged == ref.staged, kind
                if kind == "none":   # rgb is the plain frame's; only alpha differs
                    np.testing.assert_array_equal(bits(rgba[..., :3]), bits(plain[..., :3]))
                if kind == "front":
                    lengths = base.bounds[:, 1].astype(np.int64) - base.bounds[:, 0].astype(np.int64)
                    assert ref.staged == int(np.minimum(lengths[lengths > 0], 256).sum())
                    assert not rgba.any()
                disable(c)
                again = c.render(vp, ub, heatmap=heat)   # off again: the default frame, bit for bit
                np.testing.assert_array_equal(bits(again), bits(base.rgba), err_msg=f"default frame after plane {kind}")
                assert c.stats().staged == base.staged
    finally:
        orc.set_blend_contraction(True)


def test_async_frames_equal_synchronous_ones():
    n, w, h = 15000, 320, 200
    scenes = [make_scene(n, 2, w, h, frame=f, scale_boost=0.5) for f in (10, 11, 12)]
    splat60 = scenes[0][0]
    base = orc.frame(splat60, scenes[0][1], uniforms(scenes[0][2]), cap=1000 * n)
    Z = plane("mixed", w, h, splat_depths(base.records[base.values], scenes[0][1]), 5)
    with Ctx(n, w, h) as c:
        c.upload(splat60)
        planes = DepthPlanes(w, h, Z)
        _lib.check(planes.enable(c), "gsr_set_depth_compositing")
        sync_rgba, sync_depth = [], []
        for _, vp, ub in scenes:
            sync_rgba.append(c.render(vp, ub))
            sync_depth.append(planes.read(c))
        hosts = [torch.empty((h, w, 4), dtype=torch.float32, pin_memory=True) for _ in scenes]
        for (_, vp, ub), hb in zip(scenes, hosts):
            c.render_async(vp, ub, host_ptr=hb.data_ptr())
        last_depth = planes.read(c)
        for k, hb in enumerate(hosts):
            np.testing.assert_array_equal(bits(hb.numpy()), bits(sync_rgba[k]), err_msg=f"async frame {k}")
        np.testing.assert_array_equal(bits(last_depth), bits(sync_depth[-1]))
        ref = dref.frame_depth(splat60, scenes[-1][1], uniforms(scenes[-1][2]), cap=1000 * n, scene_depth=Z)
        np.testing.assert_array_equal(bits(last_depth), bits(ref.depth))


def test_state_rules_and_resize():
    n, w, h = 4000, 96, 64
    splat60, vp, ub = make_scene(n, 3, w, h)
    with Ctx(n, w, h) as c:
        c.upload(splat60)
        L = c.L
        planes = DepthPlanes(w, h, np.full((h, w), 2.0, dtype=np.float32))
        # a scene depth needs an output
        assert L.gsr_set_depth_compositing(c.h, C.c_void_p(planes.Z.data_ptr()), None) == _lib.GSR_ERR_INVALID
        # not on a sharded context
        c.set_band(0, 2)
        assert planes.enable(c) == _lib.GSR_ERR_STATE
        c.set_band(0, 4)
        c.set_row_interleave(1, 2)
        assert planes.enable(c) == _lib.GSR_ERR_STATE
        c.set_row_interleave(0, 1)
        _lib.check(planes.enable(c), "gsr_set_depth_compositing")
        # ... and no sharding while it is on
        assert L.gsr_set_band(c.h, 1, 3) == _lib.GSR_ERR_STATE
        _lib.check(L.gsr_set_band(c.h, 0, 4), "gsr_set_band (the full frame)")
        assert L.gsr_set_row_interleave(c.h, 0, 2) == _lib.GSR_ERR_STATE
        _lib.check(L.gsr_set_row_interleave(c.h, 0, 1), "gsr_set_row_interleave(0, 1)")
        handles = (C.c_ubyte * 128)()
        assert L.gsr_peer_export_framebuffers(c.h, handles) == _lib.GSR_ERR_STATE
        assert L.gsr_peer_import_framebuffers(c.h, handles) == _lib.GSR_ERR_STATE
        blob = c.group_export()
        buf = (C.c_ubyte * (2 * len(blob))).from_buffer_copy(blob + blob)
        assert L.gsr_group_attach(c.h, 0, 2, buf) == _lib.GSR_ERR_STATE
        # pick keeps the default path and leaves the depth-composited frame as it is
        rgba = c.render(vp, ub)
        depth = planes.read(c)
        assert (rgba[..., 3] < 1).all()
        busy = int(np.argmax(c.taps()["bounds"][:, 1].astype(np.int64) - c.taps()["bounds"][:, 0].astype(np.int64)))
        pick_depth = c.pick(busy)
        fb = c.copy(_lib.GSR_BUF_FRAMEBUFFER, w * h * 4, np.float32).reshape(h, w, 4)
        np.testing.assert_array_equal(bits(fb), bits(rgba))
        np.testing.assert_array_equal(bits(planes.read(c)), bits(depth))
        disable(c)
        c.render(vp, ub)
        np.testing.assert_array_equal(c.pick(busy), pick_depth)
        # a resize switches the mode off: the frame is opaque again and the old depth plane is not written
        _lib.check(planes.enable(c), "gsr_set_depth_compositing")
        planes.out.fill_(-1.0)
        torch.cuda.synchronize()
        c.resize(w, h)
        rgba = c.render(vp, ub)
        assert (rgba[..., 3] == 1).all()
        assert (planes.read(c) == -1.0).all()
