"""Orthographic cameras on the CPU (include/gsr.h GSR_FLAG_ORTHOGRAPHIC): the orthographic oracle against an independent float64
restatement, its cull and depth key, the Python mirror's Projection::set_orthogonal and w-row packing, and the orthographic projection
kernels compiled for the CPU (tests/ortho_reference/ortho_emu.cpp on top of tests/kernel_emu) against the oracle, bit for bit."""
import numpy as np
import pytest

from godotgaussiansplatting_b200 import _lib
from godotgaussiansplatting_b200 import camera as cam
from godotgaussiansplatting_b200.ply_file import PlyFile, swizzle_splats
from godotgaussiansplatting_b200.rasterizer import GaussianSplattingRasterizer
from godotgaussiansplatting_b200.synthetic import synthetic_ply_table
from oracle import oracle as orc
from tests import instance_reference as iref
from tests import ortho_reference as oref
from tests.scenes import make_scene, uniforms_bytes
from tests.test_sh_degree import expected_planes, zero_splat_coeffs

F32 = np.float32


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def uni(ub):
    return orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8))


def view_depth(vp, p):
    """-(V p).z, the linear view depth of frame-space points p (n, 3), in float64."""
    V = np.asarray(vp, dtype=np.float64)[:16].reshape(4, 4)   # V[c][r]
    return -(p @ V[:3, 2] + V[3, 2])


def splats_on_axis(vp, depths, sigma=0.02, opacity=0.9, dc=(1.0, 0.0, 0.0)):
    """Isotropic splats on the camera's forward axis at the given view depths (splat60 rows)."""
    V = np.asarray(vp, dtype=np.float64)[:16].reshape(4, 4)
    R, t = V[:3, :3].T, V[3, :3]           # view = R p + t
    eye = -np.linalg.solve(R, t)           # the camera position in the splat frame
    fwd = -R[2]                            # the forward axis: view z decreases along it
    s = np.zeros((len(depths), 60), dtype=F32)
    s[:, 0:3] = eye[None, :] + np.asarray(depths, dtype=np.float64)[:, None] * fwd[None, :]
    s[:, 4] = s[:, 7] = s[:, 9] = sigma * sigma
    s[:, 10] = opacity
    s[:, 12:15] = dc
    return s


W, H = 128, 96


def default_ortho(size=4.0, near=0.05, far=4000.0):
    return oref.ortho_camera(W, H, size=size, near=near, far=far)


# ---- the oracle against float64 ------------------------------------------------------------------------------------------------
def test_oracle_is_orthographic_ewa_in_float64():
    n = 3000
    splat60 = swizzle_splats(synthetic_ply_table(n, 4), 0.0)
    vp, ub = oref.ortho_camera(W, H, size=2.5, near=0.5, far=4.5, frame=7)
    pr = oref.project(splat60, vp, uni(ub))
    ids = np.unique(pr.values)
    assert len(ids) > n // 2
    V = vp[:16].astype(np.float64).reshape(4, 4)
    P = vp[16:].astype(np.float64).reshape(4, 4)
    s = splat60[ids].astype(np.float64)
    view = s[:, 0:3] @ V[:3, :] + V[3]                   # rows: (V sp)^T
    clip = view @ P
    assert np.all(clip[:, 3] == 1.0) and np.all(np.abs(clip[:, 2]) <= 1.0)
    J = np.diag([W * 0.5 * P[0, 0], H * 0.5 * P[1, 1]])  # constant: no depth divide
    M = J @ V[:3, :2].T                                  # 2 x 3: rows of b^T
    c = s[:, 4:10]
    cov3 = np.stack([c[:, [0, 1, 2]], c[:, [1, 3, 4]], c[:, [2, 4, 5]]], axis=1)
    cov2 = np.einsum("ij,njk,lk->nil", M, cov3, M)
    cx, cy, cz = cov2[:, 0, 0] + 0.3, cov2[:, 0, 1], cov2[:, 1, 1] + 0.3
    det = cx * cz - cy * cy
    r = pr.records[ids]
    np.testing.assert_allclose(r["conic"][:, 0], cz / det, rtol=2e-4)
    np.testing.assert_allclose(r["conic"][:, 2], cx / det, rtol=2e-4)
    np.testing.assert_allclose(r["conic"][:, 1], -cy / det, rtol=2e-3, atol=1e-6)
    np.testing.assert_allclose(r["image_pos"][:, 0], (clip[:, 0] + 1.0) * 0.5 * (W - 1), rtol=1e-5, atol=1e-3)
    np.testing.assert_allclose(r["image_pos"][:, 1], (clip[:, 1] + 1.0) * 0.5 * (H - 1), rtol=1e-5, atol=1e-3)
    # SH: the view direction of every splat is the camera's forward axis
    f = -V[:3, 2] / np.linalg.norm(V[:3, 2])
    np.testing.assert_allclose(r["color"][:, :3], np.maximum(sh_eval64(s[:, 12:60].reshape(-1, 16, 3), f), 0.0), rtol=1e-4, atol=1e-5)


def sh_eval64(sh, d):
    """gsplat_projection.glsl:94-121 in float64 for one direction d: sh (n, 16, 3) -> (n, 3)."""
    x, y, z = d
    xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
    basis = [0.28209479177387814, -0.4886025119029199 * y, 0.4886025119029199 * z, -0.4886025119029199 * x,
             1.0925484305920792 * xy, -1.0925484305920792 * yz, 0.31539156525252005 * (2 * zz - xx - yy), -1.0925484305920792 * xz,
             0.5462742152960396 * (xx - yy), -0.5900435899266435 * y * (3 * xx - yy), 2.890611442640554 * x * yz,
             -0.4570457994644658 * y * (4 * zz - xx - yy), 0.3731763325901154 * z * (2 * zz - 3 * xx - 3 * yy),
             -0.4570457994644658 * x * (4 * zz - xx - yy), 1.445305721320277 * z * (xx - yy), -0.5900435899266435 * x * (xx - 3 * yy)]
    return 0.5 + np.einsum("k,nkc->nc", np.array(basis), sh)


def test_isotropic_splat_is_the_same_at_every_depth():
    vp, ub = default_ortho(size=4.0, near=0.05, far=100.0)
    for sigma in (0.01, 0.05, 0.2):
        s = splats_on_axis(vp, [1.0, 7.5, 60.0], sigma=sigma)
        pr = oref.project(s, vp, uni(ub))
        assert pr.visible == 3
        r = pr.records
        for k in ("conic", "image_pos"):
            assert np.array_equal(bits(r[k][0]), bits(r[k][1])) and np.array_equal(bits(r[k][0]), bits(r[k][2]))
        f = F32(W) * F32(0.5) * vp[16]   # focal = W/2 * P00, the same for y here: P11 * H/2 with size = H units of P11
        want = (np.float64(f) * sigma) ** 2 + 0.3
        np.testing.assert_allclose(r["conic"][0, 0], 1.0 / want, rtol=1e-5)
        assert len(pr.keys) == 3 * len(np.unique(pr.keys >> 16))   # the same tiles for every depth


# ---- cull and key --------------------------------------------------------------------------------------------------------------
def test_key_is_linear_and_monotone_in_view_depth():
    near, far = 0.5, 40.0
    vp, ub = default_ortho(near=near, far=far)
    d = np.linspace(near, far, 401)[1:-1]
    pr = oref.project(splats_on_axis(vp, d, sigma=0.02), vp, uni(ub))
    assert pr.visible == len(d)
    first = np.unique(pr.values, return_index=True)[1]
    key = (pr.keys[first] & 0xFFFF).astype(np.int64)
    assert np.all(np.diff(key) > 0)
    np.testing.assert_allclose(key, (d - near) / (far - near) * 65535.0, atol=2.0)


@pytest.mark.parametrize("far", [10.0, 4000.0])
def test_near_half_is_drawn_and_outside_the_slab_is_culled(far):
    near = 0.05
    vp, ub = default_ortho(near=near, far=far)
    assert oref.is_orthographic(vp)
    inside = np.array([0.06, 0.3, 1.0, 2.5, 0.49 * (near + far), 0.9 * far, 0.999 * far])
    outside = np.array([-3.0, -0.01, 0.0, 0.04, 1.01 * far, 2.0 * far])
    s = splats_on_axis(vp, np.concatenate([inside, outside]))
    u = uni(ub)
    pr = oref.project(s, vp, u)
    assert np.array_equal(np.unique(pr.values), np.arange(len(inside)))
    np.testing.assert_allclose(view_depth(vp, s[:, :3].astype(np.float64))[:len(inside)], inside, rtol=1e-4, atol=1e-4)
    # the perspective rule culls every splat nearer than (near + far) / 2 on the same matrix
    persp = orc.project(s, vp, u)
    assert not np.isin(np.arange(5), persp.values).any()
    # and the synthetic cloud in front of the default camera: nothing with the perspective rule, nearly everything orthographically
    splat60, _, _ = make_scene(20000, 2, 320, 180)
    vp2, ub2 = oref.ortho_camera(320, 180, size=4.0, near=near, far=far)
    assert orc.project(splat60, vp2, uni(ub2)).visible == 0
    assert oref.project(splat60, vp2, uni(ub2)).visible > 19000


def test_overlapping_splats_blend_front_to_back_whatever_their_ids():
    vp, ub = default_ortho(size=2.0, near=0.5, far=20.0)
    front = splats_on_axis(vp, [3.0], sigma=0.2, opacity=0.95, dc=(3.0, -2.0, -2.0))   # red
    back = splats_on_axis(vp, [3.1], sigma=0.2, opacity=0.95, dc=(-2.0, -2.0, 3.0))    # blue, 0.1 / (19.5 / 65536) bins behind
    a = oref.frame(np.concatenate([front, back]), vp, ub)
    b = oref.frame(np.concatenate([back, front]), vp, ub)
    assert np.array_equal(bits(a["rgba"]), bits(b["rgba"]))
    px = a["rgba"][H // 2, W // 2]
    assert px[0] > 0.5 and px[2] < 0.2
    # the frame function of the oracle library and the composition used by the GPU tests agree
    c = oref.oracle_frame(np.concatenate([back, front]), vp, ub)
    assert np.array_equal(bits(c["rgba"]), bits(b["rgba"])) and np.array_equal(c["keys"], b["keys"]) and c["staged"] == b["staged"]


# ---- the Python mirror ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("keep", [cam.KEEP_HEIGHT, cam.KEEP_WIDTH], ids=["keep_height", "keep_width"])
def test_orthogonal_matrix(keep):
    size, aspect, near, far = 3.5, 16.0 / 9.0, 0.05, 4000.0
    c = cam.Camera3D(near=near, far=far, projection=cam.PROJECTION_ORTHOGONAL, size=size, keep_aspect=keep)
    c.aspect = aspect
    m = c.get_camera_projection().reshape(4, 4)   # m[c][r]
    assert np.array_equal(m, cam.orthogonal(size, aspect, near, far, flip_fov=keep == cam.KEEP_WIDTH).reshape(4, 4))
    w, h = (size * aspect, size) if keep == cam.KEEP_HEIGHT else (size, size / aspect)
    np.testing.assert_allclose([m[0, 0], m[1, 1], m[2, 2], m[3, 2]], [2 / w, 2 / h, -2 / (far - near), -(far + near) / (far - near)], rtol=1e-6)
    assert np.array_equal(m[:, 3], [0, 0, 0, 1]) and m[3, 0] == 0 and m[3, 1] == 0
    off = m.copy()
    off[[0, 0, 1, 1, 2, 2], [1, 2, 0, 2, 0, 1]] = 0
    assert np.array_equal(off, m)
    assert cam.Camera3D().size == 1.0 and cam.Camera3D().keep_aspect == cam.KEEP_HEIGHT
    assert cam.Camera3D().projection == cam.PROJECTION_PERSPECTIVE


def frustum(left, right, bottom, top, near, far):
    """Godot Projection::set_frustum (float32)."""
    f = F32
    m = np.zeros((4, 4), dtype=F32)
    m[0, 0] = f(2) * f(near) / (f(right) - f(left))
    m[1, 1] = f(2) * f(near) / (f(top) - f(bottom))
    m[2, 0] = (f(right) + f(left)) / (f(right) - f(left))
    m[2, 1] = (f(top) + f(bottom)) / (f(top) - f(bottom))
    m[2, 2] = -(f(far) + f(near)) / (f(far) - f(near))
    m[2, 3] = -1
    m[3, 2] = -(f(2) * f(far) * f(near)) / (f(far) - f(near))
    return m.reshape(16)


def test_w_row_packing():
    c = cam.orbit_camera(12)
    view = c.get_camera_transform()
    for proj in (c.get_camera_projection(), cam.perspective(40.0, 1.3, 0.1, 50.0), frustum(-0.3, 0.5, -0.2, 0.4, 0.1, 100.0)):
        a = cam.pack_camera_push_constants(view, proj)
        b = cam.pack_camera_push_constants(view, proj, keep_w_row=True)
        assert a.tobytes() == b.tobytes() and not oref.is_orthographic(b)
        assert np.array_equal(a, orc.pack_camera(view, proj))
    o = cam.orthogonal(2.0, 1.5, 0.05, 4000.0)
    a, b = cam.pack_camera_push_constants(view, o), cam.pack_camera_push_constants(view, o, keep_w_row=True)
    assert not oref.is_orthographic(a) and oref.is_orthographic(b)
    assert np.array_equal(a[[19, 23, 27, 31]], [0, 0, -1, 0]) and np.array_equal(b[[19, 23, 27, 31]], [0, 0, 0, 1])
    assert np.array_equal(np.delete(a, [19, 23, 27, 31]), np.delete(b, [19, 23, 27, 31]))


@pytest.mark.parametrize("flags", [0, _lib.GSR_FLAG_ORTHOGRAPHIC])
def test_rasterizer_packs_the_w_row_of_a_flagged_context(flags):
    assert _lib.GSR_FLAG_ORTHOGRAPHIC == 0x20
    c = cam.default_camera()
    ply = PlyFile.from_array(synthetic_ply_table(8, 1))
    r = GaussianSplattingRasterizer(ply, (64, 36), None, c, flags=flags)
    assert r.update_camera_matrices()
    assert r.camera_push_constants.tobytes() == cam.pack_camera_push_constants(c.get_camera_transform(), c.get_camera_projection()).tobytes()
    c.projection, c.size = cam.PROJECTION_ORTHOGONAL, 3.0
    assert r.update_camera_matrices()
    assert oref.is_orthographic(r.camera_push_constants) == bool(flags)


# ---- emulated kernels against the oracle -----------------------------------------------------------------------------------------
N = 2048


def scene(time=10.0, far=4.5, n=N, seed=11, size=2.5):
    t62 = synthetic_ply_table(n, seed)
    t62[:, 9:54] += 0.02   # every coefficient non-zero
    splat60 = swizzle_splats(t62, 0.0)
    vp, _ = oref.ortho_camera(W, H, size=size, near=0.5, far=far, frame=5)
    c = cam.orbit_camera(5, aspect=W / H)
    return splat60, vp, uniforms_bytes(c.global_position, 1.0, W, H, time)


def store_of(splat60, bands):
    return np.ascontiguousarray(expected_planes(splat60, bands, (splat60.shape[0] + 255) // 256 * 256))


def oracle_projection(splat60, vp, ub, ranges=None, xf=None):
    u = uni(ub)
    if ranges is not None:
        p = oref.project_instanced(splat60, vp, u, ranges, xf)
    else:
        p = oref.project(splat60, vp, u)
    return p.records, p.keys, p.values, p.duplicates, p.visible, p.last_tile


def assert_same_projection(got, want):
    recs, keys, vals, m, vis, last = got
    wr, wk, wv, wm, wvis, wlast = want
    assert (m, vis, last) == (wm, wvis, wlast)
    assert np.array_equal(keys, wk) and np.array_equal(vals, wv)
    ids = np.unique(wv)
    assert np.array_equal(bits(recs[ids].view(F32).reshape(len(ids), 12)), bits(wr[ids].view(F32).reshape(len(ids), 12)))


def instances():
    from tests.test_instances import SCALED, rigid
    return [(0, 600), (600, 700), (1300, 748), (100, 33)], [iref.inverse(m) for m in (rigid(4), SCALED, rigid(6), rigid(7))]


@pytest.mark.parametrize("time", [10.0, 0.6], ids=["static", "load_in"])
@pytest.mark.parametrize("bulk_min", [1, 33], ids=["bulk", "gather"])
@pytest.mark.parametrize("instanced", [False, True], ids=["default", "instances"])
@pytest.mark.parametrize("bands", [1, 2, 3, 4])
def test_emulated_projection_is_the_ortho_oracle(bands, instanced, bulk_min, time):
    splat60, vp, ub = scene(time)
    ranges, xf = instances() if instanced else (None, None)
    padded = zero_splat_coeffs(splat60, bands)
    want = oracle_projection(padded, vp, ub, ranges, xf)
    assert want[4] > 500
    assert_same_projection(oref.emu_project(store_of(padded, bands), bands, vp, ub, bulk_min, N, ranges, xf), want)
    if bands < 4:   # a degree-3 store rendered at a lower degree
        assert_same_projection(oref.emu_project(store_of(splat60, 4), bands, vp, ub, bulk_min, N, ranges, xf), want)


@pytest.mark.parametrize("n", [1, 31, 33, 257, 2001])
def test_emulated_projection_ragged_sizes_and_default_far(n):
    splat60, vp, ub = scene(n=n, far=4000.0, seed=5)
    want = oracle_projection(splat60, vp, ub)
    for bulk_min in (1, 12):
        assert_same_projection(oref.emu_project(store_of(splat60, 4), 4, vp, ub, bulk_min, n), want)


def test_emulated_instances_one_three_eight():
    from tests.test_instances import SCALED, rigid
    splat60, vp, ub = scene(seed=8)
    for ranges, mats in (([(0, N)], [rigid(1)]), ([(0, 1000), (900, 1148), (5, 7)], [rigid(2), SCALED, rigid(3)]),
                         ([(64 * k, 200 + 13 * k) for k in range(8)], [rigid(k) if k % 3 else SCALED for k in range(8)])):
        xf = [iref.inverse(m) for m in mats]
        want = oracle_projection(splat60, vp, ub, ranges, xf)
        assert want[4] > 0
        for bulk_min in (1, 33):
            assert_same_projection(oref.emu_project(store_of(splat60, 4), 4, vp, ub, bulk_min, N, ranges, xf), want)


def test_emulated_projection_of_a_splat_at_the_camera_position():
    """The camera position lies inside a slab with near < 0; its splat has a finite view direction, so it is drawn with its colour."""
    splat60, _, ub = scene(seed=12)
    c = cam.orbit_camera(5, aspect=W / H)
    vp = cam.pack_camera_push_constants(c.get_camera_transform(), cam.orthogonal(2.5, W / H, -4.0, 4.5), keep_w_row=True)
    u = np.frombuffer(ub, dtype=F32).copy()
    s = splat60.copy()
    s[100, 0:3] = u[0:3]
    s[100, 4:10] = [0.01, 0, 0, 0.01, 0, 0.01]
    s[100, 10] = 0.8
    want = oracle_projection(s, vp, ub)
    assert 100 in want[2]
    assert np.all(np.isfinite(want[0]["color"][100])) and want[0]["color"][100, :3].max() > 0.0
    for bands in (1, 4):
        padded = zero_splat_coeffs(s, bands)
        w = oracle_projection(padded, vp, ub)
        for bulk_min in (1, 33):
            assert_same_projection(oref.emu_project(store_of(padded, bands), bands, vp, ub, bulk_min, N), w)
