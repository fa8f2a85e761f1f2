"""Motion vectors on the GPU (include/gsr.h gsr_set_motion_vectors), through the C-ABI with torch CUDA tensors as the caller's planes:
composite_kernel<CONTRACT, true, true> against the motion oracle bit for bit, the unchanged depth-composited frame around it, the
previous-state rules across asynchronous instanced frames, and the state rules."""
import ctypes as C

import numpy as np
import pytest

from godotgaussiansplatting_b200 import _lib
from oracle import oracle as orc
from tests import instance_reference as iref
from tests import motion_reference as mref
from tests.gsr_direct import REC_DTYPE, Ctx
from tests.scenes import make_scene

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
F32 = np.float32


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def uni(ub):
    return orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8))


class Planes:
    def __init__(self, w, h):
        self.depth = torch.full((h, w), float("nan"), dtype=torch.float32, device="cuda")
        self.motion = torch.full((h, w, 2), float("nan"), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()

    def enable(self, c, motion=True):
        _lib.check(c.L.gsr_set_depth_compositing(c.h, None, C.c_void_p(self.depth.data_ptr())), "gsr_set_depth_compositing")
        if motion:
            _lib.check(c.L.gsr_set_motion_vectors(c.h, C.c_void_p(self.motion.data_ptr())), "gsr_set_motion_vectors")

    def read(self, c):
        c.sync()
        return self.depth.cpu().numpy(), self.motion.cpu().numpy()


def records_of_last_frame(c, n_records):
    st = c.stats()
    m = int(min(st.duplicates, st.capacity))
    T = st.tiles_x * st.tiles_y
    recs = c.copy(_lib.GSR_BUF_RECORDS, n_records, REC_DTYPE).view(orc.RECORD_DTYPE)
    return recs, c.copy(_lib.GSR_BUF_VALUES, m, np.uint32), c.copy(_lib.GSR_BUF_BOUNDS, T * 2, np.uint32).reshape(T, 2)


def oracle_of_last_frame(c, n_records, vp, pvp, w, h, contract=True, prev_pos=None, heat=0.0):
    recs, vals, bnds = records_of_last_frame(c, n_records)
    m = mref.splat_motion(recs, vp, pvp, w, h, prev_pos)
    return mref.render_motion(recs, vals, bnds, w, h, vp, m, None, heat, contract)


CASES = {
    "default_cam": (20000, 1, 640, 480, 0.0, 0, None),
    "orbit_ragged_heat": (9000, 5, 250, 130, 1.0, 0, 37),
    "uncontracted": (12000, 3, 333, 201, 0.0, _lib.GSR_FLAG_UNCONTRACTED_BLEND, 80),
}


@pytest.mark.parametrize("case", list(CASES))
def test_consecutive_frames_are_the_oracle_and_motion_changes_nothing_else(case):
    n, seed, w, h, heat, flags, frame = CASES[case]
    contract = not (flags & _lib.GSR_FLAG_UNCONTRACTED_BLEND)
    f0 = 3 if frame is None else frame - 2
    splat60, pvp, pub = make_scene(n, seed, w, h, frame=f0, scale_boost=0.5)
    _, vp, ub = make_scene(n, seed, w, h, frame=frame, scale_boost=0.5)
    with Ctx(n, w, h, flags=flags, factor=1000) as c:
        c.upload(splat60)
        p = Planes(w, h)
        p.enable(c, motion=False)
        c.render(pvp, pub, heatmap=heat)
        rgba0 = c.render(vp, ub, heatmap=heat)
        depth0, _ = p.read(c)
        _lib.check(c.L.gsr_set_motion_vectors(c.h, C.c_void_p(p.motion.data_ptr())), "gsr_set_motion_vectors")
        c.render(pvp, pub, heatmap=heat)
        rgba = c.render(vp, ub, heatmap=heat)
        depth, mo = p.read(c)
        np.testing.assert_array_equal(bits(rgba), bits(rgba0))
        np.testing.assert_array_equal(bits(depth), bits(depth0))
        o_rgba, o_depth, o_mo, o_staged = oracle_of_last_frame(c, n, vp, pvp, w, h, contract, heat=heat)
        np.testing.assert_array_equal(bits(rgba), bits(o_rgba))
        np.testing.assert_array_equal(bits(depth), bits(o_depth))
        np.testing.assert_array_equal(bits(mo), bits(o_mo))
        assert c.stats().staged == o_staged
        assert np.abs(mo).max() > 0


def test_zero_motion_first_frame_static_camera_reset_and_resize():
    n, w, h = 6000, 160, 120
    splat60, vp, ub = make_scene(n, 2, w, h, frame=10)
    _, vp2, ub2 = make_scene(n, 2, w, h, frame=14)
    with Ctx(n, w, h) as c:
        c.upload(splat60)
        p = Planes(w, h)
        p.enable(c)
        c.render(vp, ub)                       # the context's first frame
        assert not bits(p.read(c)[1]).any()
        c.render(vp, ub)                       # a static camera
        assert not bits(p.read(c)[1]).any()
        c.render(vp2, ub2)                     # moved
        assert np.abs(p.read(c)[1]).max() > 0
        _lib.check(c.L.gsr_reset_motion(c.h), "gsr_reset_motion")
        c.render(vp, ub)                       # the frame after a camera cut
        assert not bits(p.read(c)[1]).any()
        c.resize(w, h)
        p = Planes(w, h)
        p.enable(c)
        c.render(vp2, ub2)                     # the first frame after a resize
        assert not bits(p.read(c)[1]).any()


def to_frame(t, ang):
    cs, sn = np.cos(ang), np.sin(ang)
    A = np.array([[cs, -sn, 0], [sn, cs, 0], [0, 0, 1]], dtype=np.float64)
    return np.concatenate([A.T.reshape(9), np.asarray(t, dtype=np.float64)]).astype(F32)


def set_instances(c, ranges, xfs):
    arr = (_lib.GsrInstance * len(ranges))()
    for k, ((first, count), x) in enumerate(zip(ranges, xfs)):
        arr[k].first, arr[k].count = first, count
        arr[k].to_frame[:] = [float(v) for v in x]
    _lib.check(c.L.gsr_set_instances(c.h, arr, len(ranges)), "gsr_set_instances")


@pytest.mark.parametrize("overlap", [0, 1])
def test_instances_across_async_frames(overlap):
    n, w, h, F = 3000, 128, 96, 20
    splat60, _, _ = make_scene(n, 9, w, h, scale_boost=0.5)
    layouts = [[(0, 1500), (1000, 2000), (0, 3000)], [(0, 2000), (500, 2500)]]
    frames = []
    for f in range(F):
        lay = layouts[0] if f < 10 else layouts[1]
        xfs = [to_frame((0.02 * f * (k + 1), 0.01 * k, 0.0), 0.03 * f * (k - 1)) for k in range(len(lay))]
        _, vp, ub = make_scene(16, 9, w, h, frame=f)
        frames.append((lay, xfs, vp, ub))
    with Ctx(n, w, h, factor=1000) as c:
        c.upload(splat60)
        _lib.check(c.L.gsr_debug_pipeline(c.h, overlap), "gsr_debug_pipeline")
        depth = torch.empty((h, w), dtype=torch.float32, device="cuda")
        _lib.check(c.L.gsr_set_depth_compositing(c.h, None, C.c_void_p(depth.data_ptr())), "gsr_set_depth_compositing")
        motion = [torch.full((h, w, 2), float("nan"), dtype=torch.float32, device="cuda") for _ in range(F)]
        torch.cuda.synchronize()
        for f, (lay, xfs, vp, ub) in enumerate(frames):
            set_instances(c, lay, xfs)
            _lib.check(c.L.gsr_set_motion_vectors(c.h, C.c_void_p(motion[f].data_ptr())), "gsr_set_motion_vectors")
            c.render_async(vp, ub)
        c.sync()
        for f, (lay, xfs, vp, ub) in enumerate(frames):
            u = uni(ub)
            xf = np.stack([iref.inverse(x) for x in xfs])
            fr = iref.frame(splat60, vp, u, lay, xf, depth=True)
            if f == 0:
                pvp, prev_xfs = vp, xfs
            else:
                pvp = frames[f - 1][2]
                prev_xfs = frames[f - 1][1] if frames[f - 1][0] == lay else xfs   # a new layout: no instance motion
            pp = mref.instance_prev_positions(splat60, lay, prev_xfs, u.model_scale, fr.proj.drawn)
            m = mref.splat_motion(fr.proj.records, vp, pvp, w, h, pp)
            _, _, o_mo, _ = mref.render_motion(fr.proj.records, fr.values, fr.bounds, w, h, vp, m)
            np.testing.assert_array_equal(bits(motion[f].cpu().numpy()), bits(o_mo), err_msg=f"frame {f}")
            if f == 10:   # the new layout's first frame: camera motion only
                m_cam = mref.splat_motion(fr.proj.records, vp, pvp, w, h, None)
                np.testing.assert_array_equal(bits(m[np.unique(fr.values)]), bits(m_cam[np.unique(fr.values)]))


@pytest.mark.parametrize("combo", ["view_depth_order", "antialiasing", "cutouts", "sh_half", "appearance"])
def test_combinations_render_as_the_oracle(combo):
    n, w, h = 8000, 200, 150
    splat60, pvp, pub = make_scene(n, 6, w, h, frame=50, scale_boost=0.5)
    _, vp, ub = make_scene(n, 6, w, h, frame=53, scale_boost=0.5)
    flags = _lib.GSR_FLAG_SH_HALF if combo == "sh_half" else 0
    with Ctx(n, w, h, flags=flags, factor=1000) as c:
        c.upload(splat60)
        L = c.L
        n_rec, prev_pos, ranges, xfs = n, None, None, None
        if combo == "view_depth_order":
            _lib.check(L.gsr_set_depth_order(c.h, _lib.GSR_DEPTH_ORDER_VIEW_DEPTH), "gsr_set_depth_order")
        elif combo == "antialiasing":
            _lib.check(L.gsr_set_antialiasing(c.h, 0.1), "gsr_set_antialiasing")
        elif combo == "cutouts":
            cut = (_lib.GsrCutout * 1)()
            cut[0].to_local[:] = [2.0, 0, 0, 0, 2.0, 0, 0, 0, 2.0, 0, 0, -5.0]
            cut[0].shape, cut[0].action, cut[0].space = _lib.GSR_CUTOUT_ELLIPSOID, _lib.GSR_CUTOUT_REMOVE, _lib.GSR_CUTOUT_FRAME
            _lib.check(L.gsr_set_cutouts(c.h, cut, 1), "gsr_set_cutouts")
        elif combo == "appearance":
            ranges = [(0, 5000), (2000, 6000)]
            xfs = [to_frame((0.1, 0, 0), 0.1), to_frame((-0.1, 0.05, 0.1), -0.1)]
            set_instances(c, ranges, xfs)
            app = (_lib.GsrInstanceAppearance * 2)()
            for k, (op, cnt) in enumerate([(0.5, 4000), (1.0, _lib.GSR_DRAW_ALL)]):
                app[k].tint[:] = [1.0, 0.5, 2.0]
                app[k].opacity, app[k].draw_count = op, cnt
            _lib.check(L.gsr_set_instance_appearance(c.h, app, 2), "gsr_set_instance_appearance")
        p = Planes(w, h)
        p.enable(c)
        c.render(pvp, pub)
        if combo == "appearance":
            prev_xfs = xfs
            xfs = [to_frame((0.15, 0.02, 0), 0.12), xfs[1]]
            set_instances(c, ranges, xfs)
            _, n_rec = iref.layout(ranges)
            prev_pos = mref.instance_prev_positions(splat60, ranges, prev_xfs, 1.0, n_rec)
        rgba = c.render(vp, ub)
        depth, mo = p.read(c)
        o_rgba, o_depth, o_mo, _ = oracle_of_last_frame(c, n_rec, vp, pvp, w, h, prev_pos=prev_pos)
        np.testing.assert_array_equal(bits(rgba), bits(o_rgba))
        np.testing.assert_array_equal(bits(depth), bits(o_depth))
        np.testing.assert_array_equal(bits(mo), bits(o_mo))
        assert np.abs(mo).max() > 0


def test_state_rules_overflow_and_pick():
    n, w, h = 6000, 160, 120
    splat60, vp, ub = make_scene(n, 2, w, h, frame=13, scale_boost=1.0)
    _, pvp, pub = make_scene(n, 2, w, h, frame=10, scale_boost=1.0)
    pvp[14] -= F32(40.0)   # the previous camera far behind: small footprints, few pairs, the capacity does not grow
    with Ctx(n, w, h, factor=1) as c:   # a small duplicate capacity: the second synchronous render overflows and re-renders
        c.upload(splat60)
        L = c.L
        p = Planes(w, h)
        assert L.gsr_set_motion_vectors(c.h, C.c_void_p(p.motion.data_ptr())) == _lib.GSR_ERR_STATE
        p.enable(c, motion=False)
        assert L.gsr_set_motion_vectors(c.h, C.c_void_p(p.depth.data_ptr())) == _lib.GSR_ERR_INVALID
        _lib.check(L.gsr_set_motion_vectors(c.h, C.c_void_p(p.motion.data_ptr())), "gsr_set_motion_vectors")
        c.render(pvp, pub)
        m0 = c.stats().duplicates
        rgba = c.render(vp, ub)
        assert c.stats().capacity > 3 * m0, "the frame did not overflow"   # (growing ahead of need stops at 3 x the pairs seen)
        depth, mo = p.read(c)
        o_rgba, o_depth, o_mo, _ = oracle_of_last_frame(c, n, vp, pvp, w, h)
        np.testing.assert_array_equal(bits(mo), bits(o_mo))   # the motion from the true previous frame
        # pick neither changes motion_out nor the next frame's motion
        st = c.stats()
        c.pick((st.tiles_y // 2) * st.tiles_x + st.tiles_x // 2)
        np.testing.assert_array_equal(bits(p.read(c)[1]), bits(mo))
        c.render(vp, ub)
        assert not bits(p.read(c)[1]).any()   # previous == this frame: still the history of the rendered frames
        # depth compositing off stops the writes
        _lib.check(L.gsr_set_depth_compositing(c.h, None, None), "gsr_set_depth_compositing")
        p.motion.fill_(float("nan"))
        torch.cuda.synchronize()
        c.render(pvp, pub)
        assert np.isnan(p.read(c)[1]).all()
        assert L.gsr_set_motion_vectors(c.h, C.c_void_p(p.motion.data_ptr())) == _lib.GSR_ERR_STATE
