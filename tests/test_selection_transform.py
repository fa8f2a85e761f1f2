"""Selection transform edits without a GPU (include/gsr.h "Splat transform edits"): the emulated transform_selection_kernel bit for bit
against the numpy rule of tests/transform_reference fed the library's own matrices, the library's float64 SH band matrices against their
defining property and an independent derivation, the frame-space composition of the Python mirror, the export of the edited cloud
(store_to_table) through the emulated ingest, and PlyFile.save."""
import ctypes as C

import numpy as np
import pytest

from godotgaussiansplatting_b200.ply_file import PlyFile, default_properties, degree_properties
from godotgaussiansplatting_b200.rasterizer import compose_frame_edit, godot_to_frame, pack_mask, store_to_table
from godotgaussiansplatting_b200.synthetic import synthetic_ply_table
from tests import transform_reference as tref

F32, U32 = np.float32, np.uint32
N = 300            # max_splats: not a multiple of 32
STRIDE = 512       # plane_stride: max_splats rounded up to 256


def rot(axis, deg):
    a = np.deg2rad(deg)
    c, s = np.cos(a), np.sin(a)
    i, j = [(1, 2), (2, 0), (0, 1)][axis]
    R = np.eye(3)
    R[i, i], R[i, j], R[j, i], R[j, j] = c, -s, s, c
    return R


def ts12(L, t):
    return np.concatenate([np.asarray(L, dtype=np.float64).T.reshape(9), np.asarray(t, dtype=np.float64)]).astype(F32)


RIGID = rot(0, 31) @ rot(1, -47) @ rot(2, 12)
TRANSFORMS = {
    "identity": (np.eye(3), [0, 0, 0]),
    "rigid": (RIGID, [0.3, -1.2, 2.5]),
    "uniform": (1.7 * rot(2, 65), [0.0, 0.5, 0.0]),
    "nonuniform": (RIGID @ np.diag([2.0, 0.5, 1.3]), [1.0, 0.0, -0.25]),
    "reflection": (np.diag([-1.0, 1.0, 1.0]) @ RIGID, [0.0, 0.0, 0.1]),
    "rot90": (np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]]) @ np.array([[1.0, 0, 0], [0, 0, -1.0], [0, 1.0, 0]]), [2, 0, 0]),
}


def random_store(bands, half, seed=0, n=N, stride=STRIDE):
    """A store with arbitrary finite values and a few specials: +-0, NaN and inf in positions and coefficients, and a coefficient large
    enough that its rotated value saturates the binary16 range."""
    rng = np.random.default_rng(seed)
    P = tref.sh_planes(bands, half)
    st = np.zeros((3 + P, stride, 4), dtype=F32)
    st[0, :n, :3] = rng.normal(size=(n, 3))
    st[0, :n, 3] = rng.random(n)
    st[1, :n] = rng.normal(size=(n, 4))
    st[2, :n, :2] = rng.normal(size=(n, 2))
    st[2, :n, 2] = rng.random(n)
    nv = 3 * bands * bands
    c = rng.normal(size=(n, nv)).astype(F32)
    st[0, 3, 0], st[0, 4, 1], st[0, 5, 2], st[0, 6, 0] = -0.0, np.nan, np.inf, -np.inf
    c[7, :], c[8, 3:] = -0.0, 0.0
    if nv > 3:
        c[9, 3], c[10, 4], c[11, 5] = np.nan, np.inf, -np.inf
        c[12, 3:] = 60000.0   # the rotated coefficient of a non-identity transform passes 65504
        c[13, 3:] = -60000.0
    if half:
        h = tref.sh_half(c).astype(U32)
        h = np.concatenate([h, np.zeros((n, 8 * P - nv), dtype=U32)], axis=1)
        st[3:, :n] = (h[:, 0::2] | (h[:, 1::2] << U32(16))).reshape(n, P, 4).transpose(1, 0, 2).view(F32)
    else:
        c = np.concatenate([c, np.zeros((n, 4 * P - nv), dtype=F32)], axis=1)
        st[3:, :n] = c.reshape(n, P, 4).transpose(1, 0, 2)
    return st


def selection(kind, seed=1):
    rng = np.random.default_rng(seed)
    hid = rng.random(N) < 0.2
    if kind == "random":
        sel = rng.random(N) < 0.5
    elif kind == "range":
        sel = np.zeros(N, bool)
        sel[37:250] = True
    elif kind == "all":
        sel = np.ones(N, bool)
        hid[:] = False
    else:
        sel = np.zeros(N, bool)
    return sel & ~hid


# ---- the kernel against the rule -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("transform", list(TRANSFORMS))
@pytest.mark.parametrize("snapshot", [False, True])
@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("bands", [1, 2, 3, 4])
def test_kernel_is_the_rule(bands, half, snapshot, transform):
    L, t = TRANSFORMS[transform]
    m95 = tref.matrices(ts12(L, t))
    store = random_store(bands, half, seed=bands)
    src = random_store(bands, half, seed=50 + bands) if snapshot else None
    for kind in ("random", "range", "all", "none"):
        sel = selection(kind, seed=bands + 3)
        got = tref.emu_transform(store, bands, half, pack_mask(sel, N), m95, src)
        want = tref.oracle(store, bands, half, sel, m95, src)
        tref.assert_store_equal(got, want, half, f"{kind}")
        untouched = ~np.concatenate([sel, np.zeros(STRIDE - N, bool)])
        np.testing.assert_array_equal(got[:, untouched].view(U32), store[:, untouched].view(U32))   # unselected, hidden, padding
    if half and bands > 1 and transform == "rigid":
        sel = np.ones(N, bool)
        out = tref.oracle(store, bands, half, sel, m95, src)
        words = out[3:, 12:14].view(U32)
        assert ((words & 0x7FFF) == 0x7BFF).any() or ((words >> 16 & 0x7FFF) == 0x7BFF).any()   # +-65504 reached


def test_identity_keeps_every_finite_non_zero_word():
    # (-0 and inf do not survive x * 1 + y * 0: the rule's IEEE operations give +0 and NaN)
    for bands in (1, 2, 3, 4):
        for half in (False, True):
            store = random_store(bands, half, seed=7)
            store[:, 0:20] = store[:, 100:120]   # no specials
            m95 = tref.matrices(ts12(np.eye(3), [0, 0, 0]))
            got = tref.emu_transform(store, bands, half, pack_mask(np.ones(N, bool), N), m95)
            np.testing.assert_array_equal(got.view(U32), store.view(U32))


def test_singular_and_non_finite_are_refused():
    assert tref.matrices(ts12(np.diag([1.0, 0.0, 1.0]), [0, 0, 0])) is None
    assert tref.matrices(ts12(np.ones((3, 3)), [0, 0, 0])) is None
    assert tref.matrices(ts12(np.diag([1e30, 1e30, 1e30]), [0, 0, 0])) is not None   # det 1e90 is finite in float64


# ---- the SH band matrices ----------------------------------------------------------------------------------------------------
def random_q(rng, proper):
    Q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    if (np.linalg.det(Q) > 0) != proper:
        Q[:, 0] *= -1.0
    return Q


@pytest.mark.parametrize("proper", [True, False])
def test_band_matrices_have_the_defining_property(proper):
    rng = np.random.default_rng(11 if proper else 12)
    for _ in range(5):
        Q = random_q(rng, proper)
        np.testing.assert_allclose(tref.lib_polar(Q), Q, atol=1e-14)
        d = rng.normal(size=(100, 3))
        for l in (1, 2, 3):
            M = tref.lib_band_matrix(Q, l)
            np.testing.assert_allclose(tref.sh_poly(l, d @ Q), tref.sh_poly(l, d) @ M.T, atol=1e-12 * (1 + np.abs(d).max() ** l))
            np.testing.assert_allclose(M @ M.T, np.eye(2 * l + 1), atol=1e-12)


def test_band_matrices_compose():
    rng = np.random.default_rng(13)
    for proper in (True, False):
        Q1, Q2 = random_q(rng, proper), random_q(rng, True)
        for l in (1, 2, 3):
            # P((Q1 Q2)^T d) = P(Q2^T Q1^T d) = M(Q2) M(Q1) P(d)
            np.testing.assert_allclose(tref.lib_band_matrix(Q1 @ Q2, l), tref.lib_band_matrix(Q2, l) @ tref.lib_band_matrix(Q1, l), atol=1e-12)


def test_polar_factor_is_the_svd_one():
    rng = np.random.default_rng(14)
    for _ in range(20):
        L = rng.normal(size=(3, 3)) * rng.uniform(0.01, 100.0, size=3)
        np.testing.assert_allclose(tref.lib_polar(L), tref.polar(L), atol=1e-12)


def test_identity_gives_exactly_i():
    _, Ms = tref.unpack(tref.matrices(ts12(np.eye(3), [0, 0, 0])))
    for l in (1, 2, 3):
        np.testing.assert_array_equal(Ms[l].view(U32), np.eye(2 * l + 1, dtype=F32).view(U32))   # +0 off the diagonal


@pytest.mark.parametrize("transform", list(TRANSFORMS))
def test_rounded_matrices_within_one_ulp_of_numpy(transform):
    L, t = TRANSFORMS[transform]
    ts = ts12(L, t)
    _, Ms = tref.unpack(tref.matrices(ts))
    Lf, _ = tref.to_source_matrix(ts)
    Q = tref.polar(Lf)
    for l in (1, 2, 3):
        M = tref.band_matrix(Q, l)
        M = np.where(np.abs(M) < 1e-9, 0.0, M)
        ref = M.astype(F32)
        ulp = np.abs(np.spacing(ref))
        assert (np.abs(Ms[l].astype(np.float64) - ref.astype(np.float64)) <= ulp).all(), (l, Ms[l] - ref)


# ---- frame-space composition (GaussianSplattingRasterizer.transform_selection) ------------------------------------------------
def test_frame_edit_composes_through_an_instance():
    rng = np.random.default_rng(15)
    A, tk = rot(1, 33) @ np.diag([1.5, 1.5, 1.5]), np.array([0.4, -2.0, 1.0])
    bo = np.array([[1, 0, 0], [0, 0, 1], [0, -1, 0]], dtype=np.float32)   # a PLY up-axis flip
    G = np.eye(4)
    G[:3, :3], G[:3, 3] = rot(2, -20) @ rot(0, 70), [0.5, 0.25, -3.0]
    B_u = godot_to_frame(G, bo).astype(np.float64)
    for ms in (1.0, 0.25):
        m = compose_frame_edit(B_u, A, tk, ms).astype(np.float64)
        x = rng.normal(size=(50, 3))
        moved = (x @ m[:, :3].T + m[:, 3]) * ms @ A.T + tk        # to_frame . to_source
        want = ((x * ms) @ A.T + tk) @ B_u[:, :3].T + B_u[:, 3]   # B . to_frame
        np.testing.assert_allclose(moved, want, rtol=1e-5, atol=1e-5)


# ---- export of the edited cloud ------------------------------------------------------------------------------------------------
def emu_ingest(table62, stride):
    t = np.ascontiguousarray(table62, dtype=F32)
    soa = np.zeros((15, stride, 4), dtype=F32)
    assert tref.emu().emu_ply_to_soa(C.c_void_p(t.ctypes.data), 62, t.shape[0], C.c_float(0.0), C.c_void_p(soa.ctypes.data), stride, 0) == 0
    return soa


def test_kept_table_round_trip():
    tref.emu().emu_ply_to_soa.argtypes = [C.c_void_p, C.c_uint, C.c_ulonglong, C.c_float, C.c_void_p, C.c_ulonglong, C.c_ulonglong]
    table = synthetic_ply_table(N, 21)
    table[:, 55:58] += np.random.default_rng(3).normal(size=(N, 3)).astype(F32)   # anisotropic scales
    store = emu_ingest(table, STRIDE)
    hidden = np.random.default_rng(4).random(N) < 0.25
    out = store_to_table(store, N, 4, False, hidden)
    assert out.shape == (int((~hidden).sum()), 62)
    assert list(degree_properties(3)) == default_properties(62)
    np.testing.assert_array_equal(out[:, 3:6], 0.0)   # normals
    again = emu_ingest(out, STRIDE)
    keep = np.flatnonzero(~hidden)
    k = keep.size
    a, b = store[:, keep], again[:, :k]
    np.testing.assert_array_equal(b[0].view(U32), a[0].view(U32))          # positions (and creation time 0)
    np.testing.assert_array_equal(b[3:].view(U32), a[3:].view(U32))        # DC and SH
    ulp = np.spacing(a[2, :, 2])
    assert (np.abs(b[2, :, 2] - a[2, :, 2]) <= ulp).all()                  # opacity within 1 ulp

    def sigma(s):
        S = np.empty((s.shape[1], 3, 3))
        S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1] = s[1, :, 0], s[1, :, 1], s[1, :, 2], s[1, :, 3]
        S[:, 1, 2], S[:, 2, 2] = s[2, :, 0], s[2, :, 1]
        S[:, 1, 0], S[:, 2, 0], S[:, 2, 1] = S[:, 0, 1], S[:, 0, 2], S[:, 1, 2]
        return S
    Sa, Sb = sigma(a), sigma(b)
    lmax = np.abs(np.linalg.eigvalsh(Sa)).max(axis=1)
    err = np.abs(Sb - Sa).max(axis=(1, 2)) / lmax
    assert err.max() <= 1e-5, err.max()


def test_kept_table_of_a_half_store_widens():
    bands = 3
    store = random_store(bands, True, seed=5)
    store[0, :N, 3] = 0.0
    store[1, :N] = [1.0, 0.1, 0.0, 2.0]
    store[2, :N, :3] = [0.2, 0.5, 0.5]
    out = store_to_table(store, N, bands, True)
    assert out.shape == (N, len(degree_properties(2)))
    c = np.ascontiguousarray(store[3:, :N].transpose(1, 0, 2)).view(U32).reshape(N, -1)
    h = np.stack([c & 0xFFFF, c >> 16], axis=2).reshape(N, -1).astype(np.uint16).view(np.float16).astype(F32)
    np.testing.assert_array_equal(out[:, 6:9], h[:, 0:3])
    np.testing.assert_array_equal(out[:, 9:9 + 24], h[:, 3:27].reshape(N, 8, 3).transpose(0, 2, 1).reshape(N, 24))
    np.testing.assert_allclose(out[:, 33], 0.0, atol=1e-6)   # logit(0.5)


def test_ply_save_round_trip(tmp_path):
    table = synthetic_ply_table(77, 8)
    table[5, 7] = np.nan
    ply = PlyFile.from_array(table, default_properties(62))
    path = str(tmp_path / "edited.ply")
    ply.save(path)
    back = PlyFile(path)
    assert back.size == 77 and back.properties == ply.properties
    np.testing.assert_array_equal(back.vertices.view(U32), ply.vertices.view(U32))
