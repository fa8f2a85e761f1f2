"""Anti-aliased trainings on the CPU (include/gsr.h gsr_set_antialiasing, gsr_upload_ply_filtered): the anti-aliased oracle against the
default oracle and a float64 restatement of the compensation, the coverage a compensated splat draws, the Python mirror of the 3D filter,
and the anti-aliased projection kernels and the filtered ingest compiled for the CPU (tests/aa_reference/aa_emu.cpp on top of
tests/kernel_emu), bit for bit."""
import numpy as np
import pytest

from godotgaussiansplatting_b200 import camera as cam
from godotgaussiansplatting_b200.ply_file import PLY_LAYOUT_3DGS, PlyFile, PlyLayout, degree_properties, narrow_table, swizzle_splats
from godotgaussiansplatting_b200.rasterizer import GaussianSplattingRasterizer
from godotgaussiansplatting_b200.synthetic import synthetic_ply_table
from oracle import oracle as orc
from tests import aa_reference as aref
from tests import ortho_reference as oref
from tests.scenes import make_scene, uniforms_bytes
from tests.test_orthographic import instances, store_of
from tests.test_sh_degree import expected_planes, sh_planes, zero_splat_coeffs

F32 = np.float32
W, H = 128, 96


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def uni(ub):
    return orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8))


def cov2d_f32(splat60, vp, width, height):
    """c2_00, c2_01, c2_11 of the perspective projection as the oracle forms them (float32, one rounding per operation, time 10 and
    model scale 1: the covariance is unscaled)."""
    V, P = vp[:16].astype(F32), vp[16:].astype(F32)
    s = splat60.astype(F32)
    sp = [s[:, 0], s[:, 1], s[:, 2]]
    view = [((V[r] * sp[0] + V[4 + r] * sp[1]) + V[8 + r] * sp[2]) + V[12 + r] * F32(1) for r in range(3)]
    z_inv = F32(1) / view[2]
    f0 = (F32(width) * F32(0.5)) * P[0] * z_inv
    f1 = (F32(height) * F32(0.5)) * P[5] * z_inv
    t0, t1 = F32(1) / P[0], F32(1) / P[5]
    clamp = lambda x, lo, hi: np.minimum(np.maximum(x, lo), hi)
    mx = clamp(view[0] * z_inv, -t0 * F32(1.3), t0 * F32(1.3))
    my = clamp(view[1] * z_inv, -t1 * F32(1.3), t1 * F32(1.3))
    j02, j12 = -f1 * mx, -f1 * my
    B0 = [V[4 * r] * f0 + V[4 * r + 2] * j02 for r in range(3)]
    B1 = [V[4 * r + 1] * f1 + V[4 * r + 2] * j12 for r in range(3)]
    c = s[:, 4:10]
    cov = [[c[:, 0], c[:, 1], c[:, 2]], [c[:, 1], c[:, 3], c[:, 4]], [c[:, 2], c[:, 4], c[:, 5]]]
    T0 = [(B0[0] * cov[k][0] + B0[1] * cov[k][1]) + B0[2] * cov[k][2] for k in range(3)]
    T1 = [(B1[0] * cov[k][0] + B1[1] * cov[k][1]) + B1[2] * cov[k][2] for k in range(3)]
    c00 = (T0[0] * B0[0] + T0[1] * B0[1]) + T0[2] * B0[2]
    c01 = (T1[0] * B0[0] + T1[1] * B0[1]) + T1[2] * B0[2]
    c11 = (T1[0] * B1[0] + T1[1] * B1[1]) + T1[2] * B1[2]
    return c00, c01, c11


# ---- the oracle ----------------------------------------------------------------------------------------------------------------
def test_aa_oracle_changes_only_opacity_and_rect():
    n = 6000
    splat60, vp, ub = make_scene(n, 4, W, H, frame=9)
    u = uni(ub)
    base = orc.project(splat60, vp, u, cap=64 * n)
    aa = aref.project(splat60, vp, u, 0.3)
    both = np.intersect1d(np.unique(base.values), np.unique(aa.values))
    assert len(both) > n // 3
    assert len(np.unique(aa.values)) <= len(np.unique(base.values))   # a smaller opacity never grows a rect
    a, b = aa.records[both], base.records[both]
    for k in ("image_pos", "conic", "pos_xy", "pos_z"):
        assert np.array_equal(bits(a[k]), bits(b[k])), k
    assert np.array_equal(bits(a["color"][:, :3]), bits(b["color"][:, :3]))
    # the opacity: splat_opacity * coef with coef restated in float64 from the oracle's own float32 determinants (the dilated det of
    # :177 and the undilated det0; both are restated here operation for operation)
    c00, c01, c11 = cov2d_f32(splat60[both], vp, W, H)
    v = F32(0.3)
    cx, cz = c00 + v, c11 + v
    det = cx * cz - c01 * c01
    assert np.array_equal(bits(b["conic"][:, 0]), bits(cz / det))   # the restated cov_2d is the oracle's
    det0 = c00 * c11 - c01 * c01
    want = b["color"][:, 3].astype(np.float64) * np.sqrt(np.maximum(2.5e-5, det0.astype(np.float64) / det))
    err = np.abs(a["color"][:, 3] - want) / np.spacing(want.astype(F32)).astype(np.float64)
    # the float32 divide, square root and product round three times (<= 1.25 ulp of coef, up to twice that in ulp of the result when
    # the two lie in different binades): most splats are within 1 ulp, none beyond 2
    assert (err <= 1.0).mean() > 0.95 and err.max() < 2.0, (np.mean(err <= 1.0), err.max())
    assert np.all(a["color"][:, 3] <= b["color"][:, 3])


def subpixel_splat(vp, sigma, opacity=0.8):
    """One isotropic white splat of `sigma` units on the orthographic camera's forward axis, 2 units in front of it."""
    V = np.asarray(vp, dtype=np.float64)[:16].reshape(4, 4)
    R, t = V[:3, :3].T, V[3, :3]
    eye = -np.linalg.solve(R, t)
    s = np.zeros((1, 60), dtype=F32)
    s[0, 0:3] = eye - 2.0 * R[2]
    s[0, 4] = s[0, 7] = s[0, 9] = sigma * sigma
    s[0, 10] = opacity
    s[0, 12:15] = 0.5 / 0.28209479177387814   # colour 1.0
    return s


@pytest.mark.parametrize("v", [0.1, 0.3])
def test_compensated_splat_draws_its_trained_coverage(v):
    """A sub-pixel splat covers o * 2 pi sqrt(det cov_2d) of the frame when its filter is compensated; drawn the reference's way it
    covers that times sqrt(det(cov_2d + 0.3) / det(cov_2d))."""
    vp, ub = oref.ortho_camera(W, H, size=4.0, near=0.5, far=10.0)
    fx, fy = F32(W) * F32(0.5) * vp[16], F32(H) * F32(0.5) * vp[21]   # px per unit: the orthographic Jacobian
    for sigma_px in (0.5, 0.7):
        sigma = sigma_px / float(fy)
        s = subpixel_splat(vp, sigma)
        sx2, sy2 = (float(fx) * sigma) ** 2, (float(fy) * sigma) ** 2
        o = float(s[0, 10])

        def coverage(variance, compensated):
            a2, b2 = sx2 + variance, sy2 + variance
            peak = o * np.sqrt(sx2 * sy2 / (a2 * b2)) if compensated else o
            r2 = 2.0 * np.log(peak * 255.0)                # alpha < 1/255 is not blended: the Mahalanobis radius kept
            return peak * 2.0 * np.pi * np.sqrt(a2 * b2) * (1.0 - np.exp(-0.5 * r2))

        # quirks off: the reference's tile-range quirk leaves the frame's last occupied tile empty, and here that is one of the splat's
        aa = aref.frame(s, vp, ub, v, ortho=True, quirks=False)["rgba"][..., 0].sum(dtype=np.float64)
        base = oref.frame(s, vp, ub, quirks=False)["rgba"][..., 0].sum(dtype=np.float64)
        ideal = o * 2.0 * np.pi * np.sqrt(sx2 * sy2)
        assert abs(aa / coverage(v, True) - 1.0) < 0.1 and abs(aa / ideal - 1.0) < 0.1, (sigma_px, aa, ideal)
        assert abs(base / coverage(0.3, False) - 1.0) < 0.1, (sigma_px, base)
        dilation = np.sqrt((sx2 + 0.3) * (sy2 + 0.3) / (sx2 * sy2))
        assert base / aa > 0.85 * dilation and dilation > 1.5


def test_eigenvalue_cull_is_unchanged():
    """The reference's cull e2 = mid - sqrt(max(0.1, mid^2 - det)) < 0 is kept: an isotropic splat whose dilated variance a + v is
    below sqrt(0.1) is not drawn.  With v = 0.3 that is a < 0.016 px^2, as in the reference; with v = 0.1 it is a < 0.216 px^2."""
    vp, ub = oref.ortho_camera(W, H, size=4.0, near=0.5, far=10.0)
    fy = float(F32(H) * F32(0.5) * vp[21])
    u = uni(ub)
    for a, drawn in ((0.20, {0.1: False, 0.3: True}), (0.23, {0.1: True, 0.3: True}), (0.01, {0.1: False, 0.3: False})):
        s = subpixel_splat(vp, np.sqrt(a) / fy)
        for v, want in drawn.items():
            assert (aref.project(s, vp, u, v, ortho=True).visible == 1) == want, (a, v)
        assert (oref.project(s, vp, u).visible == 1) == drawn[0.3]


def test_oracle_frame_functions_agree():
    splat60, vp, ub = make_scene(3000, 5, W, H, frame=3)
    for v, ortho in ((0.1, False), (2.0, False), (0.3, True)):
        if ortho:
            vp, ub = oref.ortho_camera(W, H, size=2.5, near=0.5, far=4.5, frame=3)
        a = aref.frame(splat60, vp, ub, v, ortho=ortho)
        b = aref.oracle_frame(splat60, vp, ub, v, ortho=ortho)
        assert a["visible"] > 100
        assert np.array_equal(bits(a["rgba"]), bits(b["rgba"])) and np.array_equal(a["keys"], b["keys"]) and a["staged"] == b["staged"]


# ---- the Python mirror ---------------------------------------------------------------------------------------------------------
def mip_table(n, seed=3, degree=3):
    """A Mip-Splatting-style vertex table: the trainer's properties and a trailing `filter_3D` column with positive, zero, negative and
    NaN filters and extreme scales.  Returns (table, property names)."""
    t62 = synthetic_ply_table(n, seed)
    rng = np.random.default_rng(seed)
    f = rng.uniform(0.0, 0.05, n).astype(F32)
    f[::7], f[1::11], f[2::13] = 0.0, -0.01, np.nan
    t62[3::17, 55] = 80.0      # exp(scale) beyond float32: +inf before and after the filter
    t62[4::19, 56] = -300.0    # exp(scale)^2 underflows: the filter makes the splat f wide and transparent
    t62[5::23, 57] = -40.0
    table = np.concatenate([narrow_table(t62, degree), f[:, None]], axis=1)
    return np.ascontiguousarray(table, dtype=F32), degree_properties(degree, extra=("filter_3D",))


def test_layout_finds_filter_3d():
    table, names = mip_table(8)
    lay = PlyFile.from_array(table, names).layout()
    assert lay.filter_3d == len(names) - 1
    assert PLY_LAYOUT_3DGS.filter_3d == -1 and PlyFile.from_array(table[:, :-1], names[:-1]).layout().filter_3d == -1
    assert PlyLayout(62, 3, 0, 6, 9, 54, 55, 58) == PLY_LAYOUT_3DGS


def test_swizzle_folds_the_3d_filter_in_float64():
    table, names = mip_table(500)
    lay = PlyFile.from_array(table, names).layout()
    got = swizzle_splats(table, 1.5, lay)
    plain = swizzle_splats(table, 1.5, PlyLayout(**{**lay.__dict__, "filter_3d": -1}))
    f = table[:, -1].astype(np.float64)
    off = ~(f > 0)
    assert off.sum() > 50
    assert np.array_equal(bits(got[off]), bits(plain[off]))   # f <= 0 or NaN: stored exactly as without the filter
    on = np.where(f > 0)[0]
    e = np.exp(table[on][:, lay.scale:lay.scale + 3].astype(np.float64))
    q = e * e
    g = q + (f[on] ** 2)[:, None]
    with np.errstate(over="ignore", invalid="ignore"):
        coef = np.sqrt(((q[:, 0] * q[:, 1]) * q[:, 2]) / ((g[:, 0] * g[:, 1]) * g[:, 2]))
    sig = 1.0 / (1.0 + np.exp(-table[on, lay.opacity].astype(np.float64)))
    assert np.array_equal(bits(got[on, 10]), bits((sig * coef).astype(F32)))
    # the covariance is the unfiltered one built from the scales sqrt(q + f^2)
    t = table[on].copy()
    with np.errstate(over="ignore"):
        t[:, lay.scale:lay.scale + 3] = np.log(np.sqrt(g)).astype(F32)
    ref = swizzle_splats(t, 1.5, PlyLayout(**{**lay.__dict__, "filter_3d": -1}))
    fin = np.isfinite(ref[:, 4:10]).all(axis=1) & (np.abs(ref[:, 4:10]) < 1e30).all(axis=1)
    scale = np.abs(ref[fin, 4:10]).max(axis=1, keepdims=True)   # off-diagonal entries cancel: compare against the row's magnitude
    assert np.all(np.abs(got[on][fin, 4:10] - ref[fin, 4:10]) <= 2e-5 * scale)
    assert np.all(got[on, 10][np.isfinite(coef)] <= plain[on, 10][np.isfinite(coef)])


def test_rasterizer_antialiasing_defaults():
    table, names = mip_table(64)
    c = cam.default_camera()
    assert GaussianSplattingRasterizer(PlyFile.from_array(table, names), (64, 36), None, c)._antialiasing == 0.1
    assert GaussianSplattingRasterizer(PlyFile.from_array(table, names), (64, 36), None, c, antialiasing=0.3)._antialiasing == 0.3
    plain = PlyFile.from_array(table[:, :-1], names[:-1])
    assert GaussianSplattingRasterizer(plain, (64, 36), None, c)._antialiasing == 0.0
    assert GaussianSplattingRasterizer(plain, (64, 36), None, c, antialiasing=0.3)._antialiasing == 0.3


# ---- emulated kernels against the oracle -----------------------------------------------------------------------------------------
N = 2048


def scene(time=10.0, n=N, seed=11):
    t62 = synthetic_ply_table(n, seed)
    t62[:, 9:54] += 0.02   # every coefficient non-zero
    splat60 = swizzle_splats(t62, 0.0)
    c = cam.orbit_camera(5, aspect=W / H)
    vp = cam.pack_camera_push_constants(c.get_camera_transform(), c.get_camera_projection())
    return splat60, vp, uniforms_bytes(c.global_position, 1.0, W, H, time)


def oracle_projection(splat60, vp, ub, v, ortho=False, ranges=None, xf=None):
    u = uni(ub)
    if ranges is not None:
        p = aref.project_instanced(splat60, vp, u, ranges, xf, v, ortho)
    else:
        p = aref.project(splat60, vp, u, v, ortho)
    return p.records, p.keys, p.values, p.duplicates, p.visible, p.last_tile


def assert_same_projection(got, want):
    recs, keys, vals, m, vis, last = got
    wr, wk, wv, wm, wvis, wlast = want
    assert (m, vis, last) == (wm, wvis, wlast)
    assert np.array_equal(keys, wk) and np.array_equal(vals, wv)
    ids = np.unique(wv)
    assert np.array_equal(bits(recs[ids].view(F32).reshape(len(ids), 12)), bits(wr[ids].view(F32).reshape(len(ids), 12)))


@pytest.mark.parametrize("time", [10.0, 0.6], ids=["static", "load_in"])
@pytest.mark.parametrize("bulk_min", [1, 33], ids=["bulk", "gather"])
@pytest.mark.parametrize("instanced", [False, True], ids=["default", "instances"])
@pytest.mark.parametrize("bands", [1, 2, 3, 4])
def test_emulated_projection_is_the_aa_oracle(bands, instanced, bulk_min, time):
    splat60, vp, ub = scene(time)
    ranges, xf = instances() if instanced else (None, None)
    padded = zero_splat_coeffs(splat60, bands)
    want = oracle_projection(padded, vp, ub, 0.3, False, ranges, xf)
    assert want[4] > 500
    assert_same_projection(aref.emu_project(store_of(padded, bands), bands, vp, ub, bulk_min, N, 0.3, False, ranges, xf), want)
    if bands < 4:   # a degree-3 store rendered at a lower degree
        assert_same_projection(aref.emu_project(store_of(splat60, 4), bands, vp, ub, bulk_min, N, 0.3, False, ranges, xf), want)


@pytest.mark.parametrize("instanced", [False, True], ids=["default", "instances"])
@pytest.mark.parametrize("ortho", [False, True], ids=["perspective", "orthographic"])
@pytest.mark.parametrize("v", [0.1, 0.3, 2.0])
def test_emulated_filter_variances(v, ortho, instanced):
    splat60, vp, ub = scene(seed=13)
    if ortho:
        vp, _ = oref.ortho_camera(W, H, size=2.5, near=0.5, far=4.5, frame=5)
    ranges, xf = instances() if instanced else (None, None)
    want = oracle_projection(splat60, vp, ub, v, ortho, ranges, xf)
    assert want[4] > 500
    for bulk_min in (1, 33):
        assert_same_projection(aref.emu_project(store_of(splat60, 4), 4, vp, ub, bulk_min, N, v, ortho, ranges, xf), want)


@pytest.mark.parametrize("bands", [1, 2, 3])
def test_emulated_orthographic_reduced_degrees(bands):
    splat60, _, ub = scene(time=0.6, seed=14)
    vp, _ = oref.ortho_camera(W, H, size=2.5, near=0.5, far=4.5, frame=5)
    padded = zero_splat_coeffs(splat60, bands)
    want = oracle_projection(padded, vp, ub, 0.1, True)
    assert want[4] > 500
    for store in (store_of(padded, bands), store_of(splat60, 4)):
        assert_same_projection(aref.emu_project(store, bands, vp, ub, 12, N, 0.1, True), want)


@pytest.mark.parametrize("n", [1, 31, 33, 257, 2001])
def test_emulated_projection_ragged_sizes(n):
    splat60, vp, ub = scene(n=n, seed=5)
    want = oracle_projection(splat60, vp, ub, 0.3)
    for bulk_min in (1, 12):
        assert_same_projection(aref.emu_project(store_of(splat60, 4), 4, vp, ub, bulk_min, n, 0.3), want)


# ---- emulated filtered ingest against the numpy mirror --------------------------------------------------------------------------
@pytest.mark.parametrize("degree", [0, 1, 3])
def test_emulated_filtered_ingest_is_the_mirror(degree):
    n, first, stride = 700, 3, 1024
    table, names = mip_table(n, seed=4 + degree, degree=degree)
    lay = PlyFile.from_array(table, names).layout()
    want60 = swizzle_splats(table, 2.5, lay)
    assert np.isinf(want60[3::17, 4]).all() and (want60[4::19, 10] == 0).any()
    for bands in sorted({degree + 1, 4}):
        soa = aref.emu_ply_to_soa(table, lay, 2.5, 3 + sh_planes(bands), stride, first)
        want = expected_planes(want60, bands, n)
        assert np.array_equal(bits(soa[:, first:first + n]), bits(want)), bands
        assert np.isnan(soa[:, :first]).all() and np.isnan(soa[:, first + n:]).all()
