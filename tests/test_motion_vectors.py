"""Motion vectors (include/gsr.h gsr_set_motion_vectors) on the CPU: composite_kernel<CONTRACT, true, true> on the kernel emulator
against the motion oracle, bit for bit; rgba and depth against the depth-compositing reference; zero motion for an unchanged frame;
and the sign and axis convention against a float64 projection, independent of both implementations."""
import numpy as np
import pytest

from godotgaussiansplatting_b200 import _lib
from oracle import oracle as orc
from tests import depth_reference as dref
from tests import instance_reference as iref
from tests import motion_reference as mref
from tests import ortho_reference as oref
from tests.scenes import make_scene, uniforms_bytes

F32 = np.float32


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def uni(ub):
    return orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8))


def check_frame(records, values, bounds, W, H, vp, prev_vp, motion, Z=None, heat=0.0, contract=True, instances=None):
    """Emulated kernel == oracle (rgba, depth, motion, staged), and rgba / depth == the depth-compositing reference.  Returns the motion."""
    o_rgba, o_depth, o_mo, o_staged = mref.render_motion(records, values, bounds, W, H, vp, motion, Z, heat, contract)
    e_rgba, e_depth, e_mo, e_staged = mref.emu_composite_motion(0 if contract else 1, records, values, bounds, W, H, vp, prev_vp, Z, heat,
                                                                instances)
    np.testing.assert_array_equal(bits(e_rgba), bits(o_rgba))
    np.testing.assert_array_equal(bits(e_depth), bits(o_depth))
    np.testing.assert_array_equal(bits(e_mo), bits(o_mo))
    assert e_staged == o_staged
    d_rgba, d_depth, d_staged = dref.render_depth(records, values, bounds, W, H, vp, Z, heat, contract)
    np.testing.assert_array_equal(bits(o_rgba), bits(d_rgba))
    np.testing.assert_array_equal(bits(o_depth), bits(d_depth))
    assert o_staged == d_staged
    check_frame.rgba = o_rgba
    return o_mo


#                   n      seed w    h    heat  flags                              scene kwargs
CASES = {
    "default_cam": (20000, 1, 640, 480, 0.0, 0, dict()),
    "orbit_ragged_heat": (9000, 5, 250, 130, 1.0, 0, dict(frame=37, scale_boost=0.5)),
    "load_in": (6000, 7, 192, 160, 0.0, 0, dict(time=0.6, scale_boost=1.0)),
    "uncontracted": (12000, 3, 333, 201, 0.0, _lib.GSR_FLAG_UNCONTRACTED_BLEND, dict(frame=80, scale_boost=1.0)),
}


def prev_camera(n, seed, w, h, kw):
    """The previous frame's view_proj: the orbit frame before (or a nearby orbit frame for the default camera)."""
    f = kw.get("frame")
    return make_scene(16, seed, w, h, frame=(f - 2) if f is not None else 3)[1]


@pytest.mark.parametrize("case", list(CASES))
def test_kernel_is_the_oracle(case):
    n, seed, w, h, heat, flags, kw = CASES[case]
    contract = not (flags & _lib.GSR_FLAG_UNCONTRACTED_BLEND)
    splat60, vp, ub = make_scene(n, seed, w, h, **kw)
    pvp = prev_camera(n, seed, w, h, kw)
    fr = orc.frame(splat60, vp, uni(ub), heatmap=heat, cap=1000 * n)
    m = mref.splat_motion(fr.records, vp, pvp, w, h)
    assert np.count_nonzero(m[fr.values]) > 0
    mo = check_frame(fr.records, fr.values, fr.bounds, w, h, vp, pvp, m, None, heat, contract)
    assert np.abs(mo).max() > 0
    # a scene depth that occludes the lower half
    d = -(((vp[2] * fr.records["pos_xy"][:, 0] + vp[6] * fr.records["pos_xy"][:, 1]) + vp[10] * fr.records["pos_z"]) + vp[14])
    Z = np.full((h, w), np.inf, dtype=F32)
    Z[h // 2:] = np.median(d[fr.values])
    check_frame(fr.records, fr.values, fr.bounds, w, h, vp, pvp, m, Z, heat, contract)


def test_unchanged_frame_has_exactly_zero_motion():
    n, w, h = 9000, 250, 130
    splat60, vp, ub = make_scene(n, 5, w, h, frame=37, scale_boost=0.5)
    fr = orc.frame(splat60, vp, uni(ub), cap=1000 * n)
    m = mref.splat_motion(fr.records, vp, vp, w, h)
    assert not bits(m).any()
    mo = check_frame(fr.records, fr.values, fr.bounds, w, h, vp, vp, m)
    assert not bits(mo).any()   # +0.0 everywhere, not -0.0


def instanced_scene(n=8000, w=200, h=150):
    splat60, vp, ub = make_scene(n, 11, w, h, frame=20, scale_boost=0.5)
    ranges = [(0, 3000), (3000, 2500), (1000, 4000)]
    eye = np.eye(3, dtype=F32)
    def to_frame(t, ang=0.0):
        c, s = np.cos(ang), np.sin(ang)
        A = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]], dtype=np.float64)
        return np.concatenate([A.T.reshape(9), np.asarray(t, dtype=np.float64)]).astype(F32)
    cur = [to_frame((0.2, 0.0, 0.0)), to_frame((0.0, 0.1, 0.3), 0.1), to_frame((-0.3, 0.05, 0.2), -0.2)]
    prev = [to_frame((0.25, -0.02, 0.0)), cur[1].copy(), to_frame((-0.3, 0.0, 0.25), -0.15)]   # moved, unchanged, moved
    return splat60, vp, ub, ranges, cur, prev


@pytest.mark.parametrize("contract", [True, False])
def test_instances_moved_unchanged_and_new_layout(contract):
    splat60, vp, ub, ranges, cur, prev = instanced_scene()
    u = uni(ub)
    W, H = u.dims[0], u.dims[1]
    pvp = make_scene(16, 11, W, H, frame=19)[1]
    xf = np.stack([iref.inverse(x) for x in cur])
    orc.set_blend_contraction(contract)
    try:
        fr = iref.frame(splat60, vp, u, ranges, xf, depth=True, contract=contract)
    finally:
        orc.set_blend_contraction(True)
    recs = fr.proj.records
    for prev_xf in (prev, cur):   # the moved layout, then a new layout (each instance is its own previous state)
        pp = mref.instance_prev_positions(splat60, ranges, prev_xf, u.model_scale, fr.proj.drawn)
        m = mref.splat_motion(recs, vp, pvp, W, H, pp)
        check_frame(recs, fr.values, fr.bounds, W, H, vp, pvp, m, contract=contract,
                    instances=(splat60, splat60.shape[0], ranges, np.stack(prev_xf), u.model_scale))
    # the unchanged instance: p' == p bit for bit
    pp = mref.instance_prev_positions(splat60, ranges, cur, u.model_scale, fr.proj.drawn)
    vis = np.unique(fr.values)
    np.testing.assert_array_equal(bits(pp[vis, 0]), bits(recs["pos_xy"][vis, 0]))
    np.testing.assert_array_equal(bits(pp[vis, 2]), bits(recs["pos_z"][vis]))
    # unchanged transforms and camera: exactly +0.0
    m = mref.splat_motion(recs, vp, vp, W, H, pp)
    mo = check_frame(recs, fr.values, fr.bounds, W, H, vp, vp, m, contract=contract,
                     instances=(splat60, splat60.shape[0], ranges, np.stack(cur), u.model_scale))
    assert not bits(mo).any()


def test_orthographic_pair():
    n, w, h = 8000, 160, 120
    splat60 = make_scene(n, 4, w, h, scale_boost=0.5)[0]
    vp, ub = oref.ortho_camera(w, h, frame=30)
    pvp, _ = oref.ortho_camera(w, h, frame=28)
    fr = oref.oracle_frame(splat60, vp, ub, depth=True)
    m = mref.splat_motion(fr["records"], vp, pvp, w, h)
    mo = check_frame(fr["records"], fr["values"], fr["bounds"], w, h, vp, pvp, m)
    assert np.abs(mo).max() > 0


# ---- the convention, against float64 ----------------------------------------------------------------------------------------
def pix64(vp32, p):
    M = np.asarray(vp32, dtype=F32).astype(np.float64)
    V, P = M[:16].reshape(4, 4), M[16:].reshape(4, 4)   # [c][r]
    view = np.concatenate([p, np.ones((len(p), 1))], axis=1) @ V
    clip = view @ P
    return np.stack([(clip[:, 0] / clip[:, 3] + 1) * 0.5, (clip[:, 1] / clip[:, 3] + 1) * 0.5], axis=1)


def isolated_splats(vp, n=5, depth=3.0, spread=0.8):
    V = np.asarray(vp, dtype=np.float64)[:16].reshape(4, 4)
    R, t = V[:3, :3].T, V[3, :3]
    eye = -np.linalg.solve(R, t)
    right, up, fwd = R[0], R[1], -R[2]
    offs = np.linspace(-spread, spread, n)
    p = np.array([eye + depth * fwd + a * right + 0.5 * a * up for a in offs])
    s = np.zeros((n, 60), dtype=F32)
    s[:, 0:3] = p
    s[:, 4] = s[:, 7] = s[:, 9] = 0.01 ** 2
    s[:, 10] = 0.99
    s[:, 12:15] = 1.0
    return s, s[:, 0:3].astype(np.float64)


def check_centres(mo, rgba, cur, prev):
    """The motion at every covered splat's centre pixel is the float64 difference.  (The last occupied tile of a frame is dropped by
    the reference's tile ranges, so one splat may be missing.)"""
    checked = 0
    for k in range(len(cur)):
        x, y = int(np.rint(cur[k][0])), int(np.rint(cur[k][1]))
        if rgba[y, x, 3] < 0.5:
            continue
        np.testing.assert_allclose(mo[y, x], prev[k] - cur[k], atol=1e-3)
        checked += 1
    assert checked >= len(cur) - 1


def test_convention_camera_translation_and_rotation():
    w, h = 320, 240
    _, vp, ub = make_scene(16, 1, w, h, frame=40)
    s, p = isolated_splats(vp)
    moved = vp.copy()
    moved[12] += F32(0.05)           # the previous camera 0.05 further along the view's x translation
    rotated = make_scene(16, 1, w, h, frame=42)[1]   # a previous camera two orbit steps away
    fr = orc.frame(s, vp, uni(ub), cap=100000)
    dims = np.array([w - 1, h - 1], dtype=np.float64)
    for pvp in (moved, rotated):
        m = mref.splat_motion(fr.records, vp, pvp, w, h)
        mo = check_frame(fr.records, fr.values, fr.bounds, w, h, vp, pvp, m)
        check_centres(mo, check_frame.rgba, pix64(vp, p) * dims, pix64(pvp, p) * dims)


def test_convention_instance_translation():
    w, h = 320, 240
    _, vp, ub = make_scene(16, 1, w, h, frame=40)
    s, p = isolated_splats(vp)
    u = uni(ub)
    cur = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], dtype=F32)
    prev = cur.copy()
    prev[9:12] = (0.03, -0.02, 0.01)
    ranges = [(0, len(s))]
    fr = iref.frame(s, vp, u, ranges, np.stack([iref.inverse(cur)]), depth=True)
    pp = mref.instance_prev_positions(s, ranges, [prev], u.model_scale, fr.proj.drawn)
    m = mref.splat_motion(fr.proj.records, vp, vp, w, h, pp)
    mo = check_frame(fr.proj.records, fr.values, fr.bounds, w, h, vp, vp, m,
                     instances=(s, len(s), ranges, np.stack([prev]), u.model_scale))
    dims = np.array([w - 1, h - 1], dtype=np.float64)
    check_centres(mo, check_frame.rgba, pix64(vp, p) * dims, pix64(vp, p + prev[9:12].astype(np.float64)) * dims)
