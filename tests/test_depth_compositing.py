"""Depth compositing (include/gsr.h gsr_set_depth_compositing) on the CPU: the mode's oracle (tests/depth_reference) against an
independent float64 restatement and against the default frame of oracle/, and composite_kernel<CONTRACT, true> compiled for the CPU
(on top of tests/kernel_emu) against that oracle, bit for bit."""
import math

import numpy as np
import pytest

from godotgaussiansplatting_b200 import camera as cam
from godotgaussiansplatting_b200.ply_file import swizzle_splats
from godotgaussiansplatting_b200.synthetic import synthetic_ply_table
from oracle import oracle as orc
from tests import depth_reference as dref
from tests.scenes import make_scene, uniforms_bytes

SPEC, UNCONTRACTED = 0, 1   # composite_kernel<true, true> / <false, true>


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def uniforms(ub):
    return orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8))


def splat_depths(records, vp):
    """d = -(((V2*x + V6*y) + V10*z) + V14) in binary32, in the order the library evaluates it."""
    V = np.asarray(vp, dtype=np.float32)
    x, y = records["pos_xy"][:, 0], records["pos_xy"][:, 1]
    z = records["pos_z"]
    return -(((V[2] * x + V[6] * y) + V[10] * z) + V[14] * np.float32(1.0))


def depth_frame(splat60, vp, ub, scene_depth=None, heat=0.0, quirks=True, contract=True):
    return dref.frame_depth(splat60, vp, uniforms(ub), heatmap=heat, quirks=quirks, cap=40 * splat60.shape[0], scene_depth=scene_depth,
                            contract=contract)


@pytest.mark.parametrize("contract", [True, False], ids=["spec", "uncontracted"])
@pytest.mark.parametrize("heat", [0.0, 1.0])
def test_without_scene_depth_rgb_is_the_default_frame(contract, heat):
    n, w, h = 5000, 150, 100
    splat60, vp, ub = make_scene(n, 11, w, h, frame=23, scale_boost=0.5)
    orc.set_blend_contraction(contract)
    try:
        ref = orc.frame(splat60, vp, uniforms(ub), heatmap=heat, cap=40 * n)
    finally:
        orc.set_blend_contraction(True)
    fr = depth_frame(splat60, vp, ub, heat=heat, contract=contract)
    np.testing.assert_array_equal(bits(fr.rgba[..., :3]), bits(ref.rgba[..., :3]))
    assert fr.staged == ref.staged
    cov = fr.rgba[..., 3]
    assert (cov >= 0).all() and (cov < 1).all() and cov.max() > 0.5
    # depth: finite exactly where something was blended, and inside the range of the splats' depths where the coverage is not tiny
    # (1 - t cancels in binary32 at coverages near one ulp)
    d = splat_depths(fr.records[fr.values], vp)
    assert np.array_equal(np.isfinite(fr.depth), cov > 0)
    fin = fr.depth[cov >= 0.01]
    assert fin.size > 1000 and fin.min() >= d.min() * (1 - 1e-5) and fin.max() <= d.max() * (1 + 1e-5)


def three_splat_scene():
    """Three records in one 20x18 frame (2x2 tiles, ragged): sorted front to back, one list per tile."""
    recs = np.zeros(3, dtype=orc.RECORD_DTYPE)
    recs["image_pos"] = [(6.0, 5.0), (11.0, 9.0), (9.0, 12.0)]
    recs["conic"] = [(0.08, 0.01, 0.06), (0.05, -0.02, 0.07), (0.04, 0.0, 0.04)]
    recs["color"] = [(0.9, 0.2, 0.1, 0.8), (0.1, 0.7, 0.3, 0.6), (0.2, 0.3, 0.9, 0.9)]
    recs["pos_xy"] = [(0.1, -0.2), (-0.3, 0.1), (0.2, 0.25)]
    recs["pos_z"] = [1.5, 2.5, 3.5]
    w, h = 20, 18
    values = np.array([0, 1, 2] * 4, dtype=np.uint32)
    bounds = np.array([[0, 3], [3, 6], [6, 9], [9, 12]], dtype=np.uint32)
    vp = np.asarray(cam.pack_camera_push_constants(cam.default_camera(aspect=w / h).get_camera_transform(),
                                                   cam.default_camera(aspect=w / h).get_camera_projection()), dtype=np.float32)
    return recs, values, bounds, w, h, vp


def restate_f64(recs, vp, w, h, Z):
    """The rules of the depth mode in float64: stop before the first splat with !(d < Z), colour/t as the default blend,
    alpha = 1 - t, depth = sum(d*alpha*t) / (1 - t)."""
    V = vp.astype(np.float64)
    rgba = np.zeros((h, w, 4))
    depth = np.full((h, w), np.inf)
    for py in range(h):
        for px in range(w):
            t, col, D = 1.0, np.zeros(3), 0.0
            for r in recs:
                if not t > 1.0 / 255.0:
                    break
                x, y, z = float(r["pos_xy"][0]), float(r["pos_xy"][1]), float(r["pos_z"])
                d = -(V[2] * x + V[6] * y + V[10] * z + V[14])
                if not d < Z[py, px]:
                    break
                ox, oy = float(r["image_pos"][0]) - px, float(r["image_pos"][1]) - py
                cx, cy, cz = (float(c) for c in r["conic"])
                alpha = float(r["color"][3]) * math.exp(-0.5 * (cx * ox * ox + cz * oy * oy) - cy * ox * oy)
                col += np.asarray(r["color"][:3], dtype=np.float64) * alpha * t
                D += d * alpha * t
                t *= 1.0 - alpha
            rgba[py, px, :3] = col
            rgba[py, px, 3] = 1.0 - t
            if 1.0 - t > 0:
                depth[py, px] = D / (1.0 - t)
    return rgba, depth


@pytest.mark.parametrize("plane", ["none", "between", "ragged"])
def test_alpha_and_depth_follow_the_rules(plane):
    recs, values, bounds, w, h, vp = three_splat_scene()
    d = splat_depths(recs, vp)
    assert d[0] < d[1] < d[2]
    Z = np.full((h, w), np.inf, dtype=np.float32)
    if plane == "between":
        Z[:] = (d[1] + d[2]) / 2            # the third splat is hidden everywhere
    elif plane == "ragged":
        Z[:, : w // 2] = (d[0] + d[1]) / 2   # left half: only the first splat; right half: hidden from the second one on
        Z[h // 2:, w // 2:] = 0.0            # lower right: nothing
    rgba, depth, staged = dref.render_depth(recs, values, bounds, w, h, vp, None if plane == "none" else Z)
    ref_rgba, ref_depth = restate_f64(recs, vp, w, h, Z)
    np.testing.assert_allclose(rgba, ref_rgba, rtol=0, atol=1e-6)
    # depth = D / (1 - t): binary32 1 - t cancels where the coverage is tiny (the float64 coverage may be 1e-30 where binary32
    # has 0 and +inf), so the depth is compared where the coverage is not small
    assert not (np.isfinite(depth) & np.isinf(ref_depth)).any()
    sure = ref_rgba[..., 3] >= 0.1
    assert sure.sum() > 50
    np.testing.assert_allclose(depth[sure], ref_depth[sure], rtol=1e-6, atol=0)
    assert staged == 12


def test_a_plane_in_front_of_everything_hides_every_splat_after_one_chunk():
    n, w, h = 30000, 200, 136
    splat60, vp, ub = make_scene(n, 4, w, h, scale_boost=1.5)
    for Z in (np.zeros((h, w), dtype=np.float32), np.full((h, w), -np.inf, dtype=np.float32)):
        fr = depth_frame(splat60, vp, ub, scene_depth=Z)
        assert not fr.rgba.any()
        assert np.isinf(fr.depth).all() and (fr.depth > 0).all()
        lengths = fr.bounds[:, 1].astype(np.int64) - fr.bounds[:, 0].astype(np.int64)
        occupied = lengths[lengths > 0]
        assert occupied.max() > 256   # some tiles have more than one chunk
        assert fr.staged == int(np.minimum(occupied, 256).sum())


def test_a_plane_between_two_slabs_shows_the_front_slab_alone():
    n_front, n_back, w, h = 3000, 4000, 176, 120
    c = cam.default_camera(aspect=w / h)
    vp = cam.pack_camera_push_constants(c.get_camera_transform(), c.get_camera_projection())
    ub = uniforms_bytes(c.global_position, 1.0, w, h, 10.0)
    front = synthetic_ply_table(n_front, 21)
    back = synthetic_ply_table(n_back, 22)
    front[:, 2] = 1.6 + 0.3 * (front[:, 2] - front[:, 2].min()) / np.ptp(front[:, 2])
    back[:, 2] = 4.0 + 1.0 * (back[:, 2] - back[:, 2].min()) / np.ptp(back[:, 2])
    both = swizzle_splats(np.concatenate([front, back]), 0.0)
    alone = both[:n_front]
    ref = orc.frame(alone, vp, uniforms(ub), quirks=False, cap=40 * n_front)
    full = orc.frame(both, vp, uniforms(ub), quirks=False, cap=40 * (n_front + n_back))
    # separated: every front splat's depth code is below every back splat's
    codes_front = full.keys[full.values < n_front] & 0xFFFF
    codes_back = full.keys[full.values >= n_front] & 0xFFFF
    assert codes_front.size and codes_back.size and codes_front.max() < codes_back.min()
    d = splat_depths(full.records, vp)
    Z = np.full((h, w), (d[full.values[full.values < n_front]].max() + d[full.values[full.values >= n_front]].min()) / 2, dtype=np.float32)
    fr = depth_frame(both, vp, ub, scene_depth=Z, quirks=False)
    np.testing.assert_array_equal(bits(fr.rgba[..., :3]), bits(ref.rgba[..., :3]))
    # and without the plane the back slab shows through
    fr_open = depth_frame(both, vp, ub, quirks=False)
    assert not np.array_equal(fr_open.rgba[..., :3], ref.rgba[..., :3])


@pytest.mark.parametrize("frame", [None, 40])
def test_splat_depth_is_the_godot_linear_depth_of_its_scene_position(frame):
    n, w, h = 4000, 160, 90
    splat60, vp, ub = make_scene(n, 8, w, h, frame=frame, model_scale=1.3)
    c = cam.default_camera(aspect=w / h) if frame is None else cam.orbit_camera(frame, aspect=w / h)
    pr = orc.project(splat60, vp, uniforms(ub))
    vis = np.unique(pr.values)
    recs = pr.records[vis]
    d = splat_depths(recs, vp).astype(np.float64)
    # Godot: the splat appears at (-x, -y, z) of its scaled position; linear depth = -(view-space z) = -basis_z . (q - origin)
    q = np.stack([-recs["pos_xy"][:, 0], -recs["pos_xy"][:, 1], recs["pos_z"]], axis=1).astype(np.float64)
    bz = c.basis[2].astype(np.float64)
    godot = -((q - c.global_position.astype(np.float64)) @ bz)
    assert (godot > 0).all()
    np.testing.assert_allclose(d, godot, rtol=2e-6, atol=1e-6)
    # and one splat alone: the depth output at its centre is its depth
    one = splat60[vis[:1]].copy()
    rgba, depth, _ = dref.render_depth(*_frame_lists(one, vp, ub), w, h, vp)
    r = pr.records[vis[0]]
    px, py = int(round(float(r["image_pos"][0]))), int(round(float(r["image_pos"][1])))
    if 0 <= px < w and 0 <= py < h and rgba[py, px, 3] > 0:
        np.testing.assert_allclose(depth[py, px], godot[0], rtol=2e-6)


def _frame_lists(splat60, vp, ub):
    fr = orc.frame(splat60, vp, uniforms(ub), cap=40 * max(1, splat60.shape[0]))
    return fr.records, fr.values, fr.bounds


# ---- composite_kernel<CONTRACT, true> on the CPU emulator against the oracle ----
#                n     seed w    h    heat kwargs
CASES = {
    "ragged_heatmap": (6000, 5, 250, 130, 1.0, dict(frame=37, scale_boost=0.5)),
    "load_in": (5000, 7, 192, 160, 0.0, dict(time=0.6, scale_boost=1.0)),
    "tiny": (40, 9, 33, 17, 0.0, dict(scale_boost=-1.0)),
}


def scene_plane(kind, w, h, d, seed):
    """none / mixed: per-pixel random depths inside the splats' range with +inf, 0 and NaN mixed in / half: the lower half of the
    frame behind a plane at the median splat depth."""
    if kind == "none":
        return None
    if kind == "half":
        Z = np.full((h, w), np.inf, dtype=np.float32)
        Z[h // 2:] = np.median(d)
        return Z
    rng = np.random.default_rng(seed)
    Z = rng.uniform(d.min(), d.max(), size=(h, w)).astype(np.float32)
    pick = rng.random((h, w))
    Z[pick < 0.1] = np.inf
    Z[(pick >= 0.1) & (pick < 0.2)] = 0.0
    Z[(pick >= 0.2) & (pick < 0.3)] = np.nan
    return Z


@pytest.mark.parametrize("variant", [SPEC, UNCONTRACTED], ids=["spec", "uncontracted"])
@pytest.mark.parametrize("plane", ["none", "mixed", "half"])
@pytest.mark.parametrize("case", list(CASES))
def test_depth_compositor_kernels_reproduce_the_oracle(case, plane, variant):
    n, seed, w, h, heat, kw = CASES[case]
    splat60, vp, ub = make_scene(n, seed, w, h, **kw)
    base = orc.frame(splat60, vp, uniforms(ub), cap=40 * n)
    Z = scene_plane(plane, w, h, splat_depths(base.records[base.values], vp), seed)
    fr = depth_frame(splat60, vp, ub, scene_depth=Z, heat=heat, contract=variant == SPEC)
    out, depth, staged = dref.emu_composite_depth(variant, fr.records, fr.values, fr.bounds, w, h, vp, Z, heat)
    np.testing.assert_array_equal(bits(out), bits(fr.rgba))
    np.testing.assert_array_equal(bits(depth), bits(fr.depth))
    assert staged == fr.staged
    if plane == "half":
        assert fr.staged <= base.staged
