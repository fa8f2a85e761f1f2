"""Splat instances (include/gsr.h gsr_set_instances) on the CPU: the composed per-instance constants against float64, the Godot transform
conversion of the Python mirror, instance_prepare_kernel + projection_kernel<true> compiled for the CPU (tests/kernel_emu) against the
instance oracle bit for bit, and the instance oracle against the default oracle frame of an explicitly transformed cloud."""
import numpy as np
import pytest

from godotgaussiansplatting_b200.rasterizer import godot_to_frame
from oracle import oracle as orc
from tests import instance_reference as iref
from tests.scenes import make_scene

F32 = np.float32


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def uniforms(ub):
    return orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8))


def rotation(axis, angle):
    axis = np.asarray(axis, dtype=np.float64)
    axis = axis / np.linalg.norm(axis)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + np.sin(angle) * K + (1 - np.cos(angle)) * (K @ K)


def to_frame(A, t):
    """(3x3 matrix form, translation) -> the 12 column-major floats of gsr_instance.to_frame."""
    return np.concatenate([np.asarray(A, dtype=np.float64).T.reshape(9), np.asarray(t, dtype=np.float64)]).astype(F32)


def rigid(seed, angle=0.5, shift=0.4):
    rng = np.random.default_rng(seed)
    return to_frame(rotation(rng.normal(size=3), rng.uniform(-angle, angle)), rng.uniform(-shift, shift, size=3))


IDENTITY = to_frame(np.eye(3), np.zeros(3))
SCALED = to_frame(rotation([0, 1, 0], 0.3) * 0.8, [0.1, -0.2, 0.3])
SHEARED = to_frame(np.array([[1.0, 0.25, 0.0], [0.0, 1.1, -0.15], [0.1, 0.0, 0.9]]), [-0.2, 0.1, 0.0])


def test_composed_constants_match_float64():
    _, vp, ub = make_scene(10, 1, 320, 200, frame=17)
    u = uniforms(ub)
    for xf12 in (rigid(1), rigid(2, 2.0, 3.0), SCALED, SHEARED):
        xf = iref.inverse(xf12)
        Vk, camk = iref.compose(vp[:16], u.camera_pos[:], xf)
        V = np.asarray(vp[:16], dtype=np.float64).reshape(4, 4).T
        M = np.eye(4)
        M[:3, :3] = xf[:9].astype(np.float64).reshape(3, 3).T
        M[:3, 3] = xf[9:12]
        Vk64 = (V @ M).T.reshape(16)
        Mi = np.linalg.inv(M)
        cam64 = Mi[:3, :3] @ np.asarray(u.camera_pos[:], dtype=np.float64) + Mi[:3, 3]
        scale = np.abs(V).max() * (np.abs(M).max() + 1)
        np.testing.assert_allclose(Vk, Vk64, rtol=0, atol=8 * np.finfo(F32).eps * scale)
        np.testing.assert_allclose(camk, cam64, rtol=0, atol=16 * np.finfo(F32).eps * (np.abs(cam64).max() + np.abs(M).max() * 4))


@pytest.mark.parametrize("basis", ["identity", "y_up"])
def test_godot_conversion(basis):
    bo = np.eye(3, dtype=F32) if basis == "identity" else np.array([[1, 0, 0], [0, 0, 1], [0, -1, 0]], dtype=F32)
    ident = godot_to_frame(np.hstack([np.eye(3), np.zeros((3, 1))]), bo)
    assert np.array_equal(ident, np.hstack([np.eye(3), np.zeros((3, 1))]).astype(F32))
    R = rotation([0.3, 1.0, -0.2], 0.7)
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, [1.5, -0.25, 2.0]
    Ti = np.linalg.inv(T)
    M, Mi = godot_to_frame(T, bo).astype(np.float64), godot_to_frame(Ti, bo).astype(np.float64)
    H, Hi = np.vstack([M, [0, 0, 0, 1]]), np.vstack([Mi, [0, 0, 0, 1]])
    np.testing.assert_allclose(H @ Hi, np.eye(4), atol=1e-6)
    # the conversion agrees with the frame-space convention of uniforms / get_splat_position: p_frame = F B p_godot
    F = np.diag([-1.0, -1.0, 1.0])
    B = bo.T.astype(np.float64)
    p = np.array([0.3, -1.2, 0.8])
    np.testing.assert_allclose(M[:, :3] @ (F @ B @ p) + M[:, 3], F @ B @ (R @ p + T[:3, 3]), atol=1e-6)


# ---- the emulated kernels against the instance oracle --------------------------------------------------------------------------
N, W, H = 2048, 128, 96   # N is a multiple of 256: a range may end exactly at the end of the planes


def cases():
    n8 = N // 8
    return {
        "one": [(0, N, rigid(3))],
        "three": [(0, 600, rigid(4)), (600, 700, SCALED), (1300, 748, SHEARED)],
        "eight": [(k * n8, n8, rigid(10 + k)) for k in range(8)],
        "overlap_repeat": [(0, 900, IDENTITY), (500, 900, rigid(5)), (0, 900, rigid(6)), (0, 900, rigid(7))],
        "ragged": [(100 * i + 3, c, rigid(20 + i)) for i, c in enumerate((1, 31, 32, 33, 257, 0))],
        "tail": [(N - 301, 301, rigid(8)), (N - 33, 33, SCALED), (1, 64, IDENTITY)],   # unaligned first, ending at max_splats
    }


@pytest.mark.parametrize("time", [10.0, 0.6], ids=["static", "load_in"])
@pytest.mark.parametrize("case", list(cases()))
def test_emulated_kernels_are_the_instance_oracle(case, time):
    splat60, vp, ub = make_scene(N, 9, W, H, frame=31, time=time, scale_boost=0.5)
    inst = cases()[case]
    ranges = [(f, c) for f, c, _ in inst]
    xf = np.stack([iref.inverse(x) for _, _, x in inst])
    ref = iref.project(splat60, vp, uniforms(ub), ranges, xf)
    got, consts, overflow = iref.emu_project(splat60, N, vp, ub, ranges, xf)
    assert not overflow
    for k in range(len(inst)):
        Vk, camk = iref.compose(vp[:16], uniforms(ub).camera_pos[:], xf[k])
        np.testing.assert_array_equal(bits(consts[k, :16]), bits(Vk))
        np.testing.assert_array_equal(bits(consts[k, 16:19]), bits(camk))
        np.testing.assert_array_equal(bits(consts[k, 19:31]), bits(xf[k, :12]))
    assert got.drawn == ref.drawn
    assert (got.duplicates, got.visible, got.last_tile) == (ref.duplicates, ref.visible, ref.last_tile)
    assert ref.visible > 0
    np.testing.assert_array_equal(got.keys, ref.keys)
    np.testing.assert_array_equal(got.values, ref.values)
    ids = np.unique(ref.values)
    np.testing.assert_array_equal(bits(got.records[ids].view(np.float32)), bits(ref.records[ids].view(np.float32)))


def test_all_empty_instances_draw_nothing():
    splat60, vp, ub = make_scene(256, 2, 64, 48)
    xf = np.stack([iref.inverse(IDENTITY)] * 2)
    got, _, _ = iref.emu_project(splat60, 256, vp, ub, [(0, 0), (256, 0)], xf)
    assert (got.drawn, got.duplicates, got.visible, got.last_tile) == (0, 0, 0, -1)


# ---- physical check: a rigid instance is the transformed cloud -----------------------------------------------------------------
def transformed_cloud(splat60, A, t):
    """Positions A p + t, covariances A S A^T; SH untouched (the caller keeps only the view-independent DC band)."""
    s = np.array(splat60, dtype=np.float64)
    s[:, 0:3] = s[:, 0:3] @ A.T + t
    S = np.empty((s.shape[0], 3, 3))
    S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2] = (s[:, 4 + i] for i in range(6))
    S[:, 1, 0], S[:, 2, 0], S[:, 2, 1] = S[:, 0, 1], S[:, 0, 2], S[:, 1, 2]
    S = A @ S @ A.T
    s[:, 4], s[:, 5], s[:, 6], s[:, 7], s[:, 8], s[:, 9] = S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]
    return s.astype(F32)


def test_rigid_instance_is_the_transformed_cloud():
    n, w, h = 6000, 200, 150
    splat60, vp, ub = make_scene(n, 4, w, h, frame=12, scale_boost=0.3)
    splat60 = splat60.copy()
    splat60[:, 15:] = 0.0   # DC colour only: the SH view direction does not matter
    A, t = rotation([0.2, 1.0, 0.1], 0.6), np.array([0.3, -0.1, 0.2])
    xf = iref.inverse(to_frame(A, t))[None]
    got = iref.frame(splat60, vp, uniforms(ub), [(0, n)], xf)
    ref = orc.frame(transformed_cloud(splat60, xf[0, :9].astype(np.float64).reshape(3, 3).T, xf[0, 9:12].astype(np.float64)), vp,
                    uniforms(ub), cap=64 * n)
    assert got.proj.visible > 0.5 * n
    err = np.abs(got.rgba - ref.rgba).max(axis=2)
    agree = float((err <= 1e-3).mean())
    # measured: 100 % of the pixels agree within 1e-3 (largest difference 4.6e-6); only rounding separates the two frames
    assert agree >= 0.999, agree
