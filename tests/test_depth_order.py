"""Depth-ordered frames (include/gsr.h gsr_set_depth_order) without a GPU: the order-preserving float map, the oracle's view depth, the
emulated six-pass (tile, depth word) sort against a stable uint64 argsort, the emulated DEPTH projection variants against the oracle bit
for bit, and a closed-form pair of splats that tie in the 16-bit key but not in view depth."""
import numpy as np
import pytest

from godotgaussiansplatting_b200 import camera as cam
from godotgaussiansplatting_b200.ply_file import swizzle_splats
from godotgaussiansplatting_b200.synthetic import synthetic_ply_table
from oracle import oracle as orc
from tests import depth_order_reference as dor
from tests import instance_reference as iref
from tests import ortho_reference as oref
from tests.scenes import make_scene, uniforms_bytes
from tests.test_orthographic import store_of
from tests.test_sh_degree import zero_splat_coeffs

F32, U32 = np.float32, np.uint32
W, H = 128, 96
N = 2048


def bits(a):
    return np.ascontiguousarray(a).view(U32)


def uni(ub):
    return orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8))


# ---- ord and d -------------------------------------------------------------------------------------------------------------------
def test_ord_is_monotone():
    rng = np.random.default_rng(1)
    specials = np.array([0.0, -0.0, 1e-45, -1e-45, 1e-40, -1e-40, 1.1754942e-38, -1.1754942e-38, 3.4e38, -3.4e38, 1.0, -1.0], dtype=F32)
    f = np.concatenate([specials, (rng.standard_normal(20000) * np.exp(rng.uniform(-80, 80, 20000))).astype(F32),
                        rng.uniform(-1e-38, 1e-38, 2000).astype(F32)])   # denormals
    f = f[np.isfinite(f)]
    w = dor.ord_words(f)
    o = np.argsort(w, kind="stable")
    fs = f[o]
    assert np.all(fs[1:] >= fs[:-1])                                   # unsigned order of the words is the float order
    assert np.all(np.diff(w[o].astype(np.int64)) >= 0)
    i, j = np.nonzero(f[:, None][:2000] < f[None, :2000])               # strict float order gives strict word order
    assert np.all(w[i] < w[j])
    nz, pz = dor.ord_words(np.array([-0.0, 0.0], dtype=F32))
    assert nz + 1 == pz                                                 # -0 sorts just before +0
    assert dor.ord_words(np.array([-1e-45], dtype=F32))[0] < nz


def test_oracle_depth_is_minus_view_z():
    splat60, vp, ub = make_scene(6000, 4, W, H, frame=9)
    pr = orc.project(splat60, vp, uni(ub), cap=64 * 6000)
    assert pr.visible > 1000
    d = dor.view_depth(pr.records, pr.values, vp)
    V = np.asarray(vp, dtype=F32)
    p = splat60[pr.values.astype(np.int64)].astype(F32)
    sp = [p[:, 0] * F32(1.0), p[:, 1] * F32(1.0), p[:, 2] * F32(1.0)]   # model scale 1
    view2 = ((V[2] * sp[0] + V[6] * sp[1]) + V[10] * sp[2]) + V[14] * F32(1.0)
    np.testing.assert_array_equal(bits(d), bits(-view2))
    assert np.all(d > 0)


# ---- the sort --------------------------------------------------------------------------------------------------------------------
TILE_WIDE = 512 * 8


@pytest.mark.parametrize("n", [1, 100, TILE_WIDE - 1, TILE_WIDE, TILE_WIDE + 1, 3 * TILE_WIDE + 17])
@pytest.mark.parametrize("kind", ["random", "ties", "one_tile"])
def test_emulated_sort_is_the_stable_argsort(n, kind):
    rng = np.random.default_rng(n + len(kind))
    if kind == "random":
        keys = rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(U32)
        words = rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(U32)
    elif kind == "ties":   # few tiles, few depth words: long runs of equal (tile, word) whose order must be kept
        keys = ((rng.integers(0, 3, n).astype(U32) * U32(0x1234)) << U32(16)) | rng.integers(0, 65536, n).astype(U32)
        words = (rng.integers(0, 4, n).astype(U32) * U32(0x01010101)) ^ U32(0x80000000)
    else:
        keys = (U32(777) << U32(16)) | rng.integers(0, 65536, n).astype(U32)
        words = dor.ord_words(rng.standard_normal(n).astype(F32) * F32(50))
    values = rng.permutation(n).astype(U32)
    want = dor.sort_by_depth(keys, values, words)
    got = dor.emu_sort(keys, values, words, n_max=n + 5000)
    np.testing.assert_array_equal(got[0], want[0])
    np.testing.assert_array_equal(got[1], want[1])


# ---- the projection --------------------------------------------------------------------------------------------------------------
def scene(time=10.0, n=N, seed=11, scale_boost=0.0):
    t62 = synthetic_ply_table(n, seed)
    t62[:, 9:54] += 0.02   # every coefficient non-zero
    t62[:, 55:58] += scale_boost
    splat60 = swizzle_splats(t62, 0.0)
    c = cam.orbit_camera(5, aspect=W / H)
    vp = cam.pack_camera_push_constants(c.get_camera_transform(), c.get_camera_projection())
    return splat60, vp, uniforms_bytes(c.global_position, 1.0, W, H, time)


def instances():
    from tests.test_instances import SCALED, rigid
    return [(0, 600, rigid(4)), (600, 700, SCALED), (1300, 748, rigid(6)), (100, 33, rigid(7))]


def check_projection(got, splat60, vp, ub, v=0.0, ortho=False, inst=None, cap=None):
    recs, keys, vals, words, m, vis, last, ovf = got
    pr = dor.project(splat60, vp, uni(ub), v, ortho, inst, cap)
    assert (m, vis, last) == (pr.duplicates, pr.visible, pr.last_tile)
    assert ovf == (cap is not None and pr.duplicates > cap)
    np.testing.assert_array_equal(keys, pr.keys)
    np.testing.assert_array_equal(vals, pr.values)
    ids = np.unique(pr.values)
    np.testing.assert_array_equal(bits(recs[ids].view(F32)), bits(pr.records[ids].view(F32)))
    want_words = dor.ord_words(dor.view_depth(pr.records, pr.values, vp))
    np.testing.assert_array_equal(words, want_words)   # the projection's half of the feature
    sk, sv = dor.emu_sort(keys, vals, words)            # and the sort's
    wk, wv, _ = dor.sort_by_depth(pr.keys, pr.values, want_words)
    np.testing.assert_array_equal(sk, wk)
    np.testing.assert_array_equal(sv, wv)
    return pr


def emu(splat60, bands, vp, ub, bulk_min, v=0.0, ortho=False, inst=None, store_bands=None, capacity=None):
    ranges = xf = None
    if inst is not None:
        ranges = [(f, c) for f, c, _ in inst]
        xf = [iref.inverse(x) for _, _, x in inst]
    store = store_of(splat60, store_bands or bands)
    return dor.emu_project(store, bands, vp, ub, bulk_min, splat60.shape[0], v, ortho, ranges, xf, capacity)


@pytest.mark.parametrize("time", [10.0, 0.6], ids=["static", "load_in"])
@pytest.mark.parametrize("instanced", [False, True], ids=["default", "instances"])
@pytest.mark.parametrize("bands", [1, 2, 3, 4])
def test_emulated_projection_is_the_oracle(bands, instanced, time):
    splat60, vp, ub = scene(time)
    padded = zero_splat_coeffs(splat60, bands)
    inst = instances() if instanced else None
    for bulk_min in (1, 33):
        pr = check_projection(emu(padded, bands, vp, ub, bulk_min, inst=inst), padded, vp, ub, inst=inst)
    assert pr.visible > 500


@pytest.mark.parametrize("instanced", [False, True], ids=["default", "instances"])
@pytest.mark.parametrize("mode", ["aa_0.3", "ortho", "ortho_aa_0.1"])
def test_emulated_orthographic_and_antialiased(mode, instanced):
    splat60, vp, ub = scene(seed=13)
    ortho = mode.startswith("ortho")
    v = {"aa_0.3": 0.3, "ortho_aa_0.1": 0.1}.get(mode, 0.0)
    if ortho:   # near 0.5 and a slab that reaches behind nothing: every d is positive; see the next test for negative ones
        vp, _ = oref.ortho_camera(W, H, size=2.5, near=0.5, far=4.5, frame=5)
    inst = instances() if instanced else None
    for bulk_min in (1, 33):
        pr = check_projection(emu(splat60, 4, vp, ub, bulk_min, v, ortho, inst), splat60, vp, ub, v, ortho, inst)
    assert pr.visible > 500


def test_emulated_orthographic_negative_depths():
    """An orthographic slab whose near plane is behind the camera: splats behind it have d < 0 and still sort by d."""
    splat60, _, ub = scene(seed=15)
    vp, _ = oref.ortho_camera(W, H, size=2.5, near=-4.0, far=4.5, frame=5)
    V = np.asarray(vp, dtype=np.float64)[:16].reshape(4, 4)
    eye = -np.linalg.solve(V[:3, :3].T, V[3, :3])
    splat60 = splat60.copy()
    splat60[:, 0:3] += (eye - splat60[:, 0:3].mean(axis=0)).astype(F32)   # the cloud around the camera: half of it behind
    got = emu(splat60, 4, vp, ub, 12, ortho=True)
    pr = check_projection(got, splat60, vp, ub, ortho=True)
    d = dor.view_depth(pr.records, pr.values, vp)
    assert (d < 0).sum() > 100 and (d > 0).sum() > 100


def test_emulated_big_rects_take_the_warp_wide_emit():
    splat60, vp, ub = scene(seed=16, scale_boost=1.5)
    got = emu(splat60, 4, vp, ub, 12)
    pr = check_projection(got, splat60, vp, ub)
    assert np.bincount(pr.values).max() > 32   # rects of more than 4 (and 32) tiles


def test_emulated_truncated_frame_is_the_emission_prefix():
    splat60, vp, ub = scene(seed=17)
    m = orc.project(splat60, vp, uni(ub), cap=64 * N).duplicates
    cap = m // 2 + 7
    got = emu(splat60, 4, vp, ub, 12, capacity=cap)
    check_projection(got, splat60, vp, ub, cap=cap)
    assert got[7] == 1


# ---- a closed-form case ----------------------------------------------------------------------------------------------------------
def tied_pair():
    """A perspective camera at near 0.05 and two large isotropic splats on its axis near view depth 100 whose 16-bit keys are equal
    (bins are about 0.5 units wide there): blue farther, with the lower id; red nearer."""
    c = cam.default_camera(aspect=W / H)
    assert abs(c.near - 0.05) < 1e-6
    vp = cam.pack_camera_push_constants(c.get_camera_transform(), c.get_camera_projection())
    ub = uniforms_bytes(c.global_position, 1.0, W, H, 10.0)
    V = np.asarray(vp, dtype=np.float64)[:16].reshape(4, 4)
    R, t = V[:3, :3].T, V[3, :3]
    eye = -np.linalg.solve(R, t)
    fwd = -R[2]
    s = np.zeros((2, 60), dtype=F32)
    for i, (depth, rgb) in enumerate(((100.0, (0, 0, 1)), (None, (1, 0, 0)))):
        s[i, 4] = s[i, 7] = s[i, 9] = 30.0 ** 2
        s[i, 10] = 0.95
        s[i, 12:15] = [(0.5 if ch else -0.5) / 0.28209479177387814 for ch in rgb]
    s[0, 0:3] = eye + 100.0 * fwd
    for dz in np.arange(0.02, 0.5, 0.02):   # the nearest offset that still shares the far splat's bin
        s[1, 0:3] = eye + (100.0 - dz) * fwd
        pr = orc.project(s, vp, uni(ub), cap=4096)
        k = {int(v): int(kk) & 0xFFFF for kk, v in zip(pr.keys, pr.values)}
        d = dor.view_depth(pr.records, np.array([0, 1]), vp)
        if len(k) == 2 and k[0] == k[1] and d[1] < d[0]:
            return s, vp, ub, d
    raise AssertionError("no tied offset found")


def test_tied_splats_draw_in_view_depth_order():
    s, vp, ub, d = tied_pair()
    assert 99.0 < d[1] < d[0] < 101.0
    pr = orc.project(s, vp, uni(ub), cap=4096)
    assert len(np.unique(pr.keys & U32(0xFFFF))) == 1                     # one 16-bit depth for both
    default = orc.frame(s, vp, uni(ub), cap=4096).rgba[H // 2, W // 2]
    ordered = dor.oracle_frame(s, vp, ub)["rgba"][H // 2, W // 2]
    assert default[2] > 0.8 and default[0] < 0.2, default                  # key ties keep id order: the far blue splat is on top
    assert ordered[0] > 0.8 and ordered[2] < 0.2, ordered                  # view depth: the near red one is
    got = emu(s, 4, vp, ub, 12)
    check_projection(got, s, vp, ub)
