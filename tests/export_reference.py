"""Reference implementation of splat export (include/gsr.h "Splat export") for the tests.

TEST INFRASTRUCTURE.  Three parts:
  1. stores in the layout of GSR_BUF_SPLATS ((planes, plane_stride, 4) float32) built from 60-float splat structs, and the special
     covariances real clouds are full of;
  2. the rule: which splats are exported, and the checks of a row table against store_to_table (the float64 numpy export) and against
     the decomposition's bars;
  3. the CPU kernel emulator of export_count_kernel and export_ply_kernel (tests/export_reference/export_emu.cpp), with several CTAs
     running at once.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from godotgaussiansplatting_b200.ply_file import degree_properties
from godotgaussiansplatting_b200.rasterizer import pack_mask, store_to_table
from tests import cutout_reference as cr
from tests.transform_reference import sh_half, sh_planes

F32, U32 = np.float32, np.uint32
HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "export_reference")
QNAN = 0x7FC00000
_emu = None


def row_floats(degree: int) -> int:
    return 17 + 3 * ((degree + 1) ** 2 - 1)


# ---- stores ---------------------------------------------------------------------------------------------------------------------
def store_from_structs(s60, bands: int, half: bool, stride: int) -> np.ndarray:
    """60-float splat structs (n <= stride) -> a store of `bands` bands (float32 or binary16 SH), slots past n zero."""
    s60 = np.asarray(s60, dtype=F32)
    n, K = s60.shape[0], bands * bands
    P = sh_planes(bands, half)
    store = np.zeros((3 + P, stride, 4), dtype=F32)
    store[0:3, :n] = s60[:, 0:12].reshape(n, 3, 4).transpose(1, 0, 2)
    vals = s60[:, 12:12 + 3 * K]
    if half:
        h = np.zeros((n, 8 * P), dtype=np.uint16)
        h[:, :3 * K] = sh_half(vals)
        words = h[:, 0::2].astype(U32) | (h[:, 1::2].astype(U32) << 16)
        store[3:, :n] = words.view(F32).reshape(n, P, 4).transpose(1, 0, 2)
    else:
        f = np.zeros((n, 4 * P), dtype=F32)
        f[:, :3 * K] = vals
        store[3:, :n] = f.reshape(n, P, 4).transpose(1, 0, 2)
    return store


def sh_values(store, n: int, bands: int, half: bool) -> np.ndarray:
    """(n, 3K) float32: the stored SH values of the first n splats, binary16 widened."""
    K, P = bands * bands, sh_planes(bands, half)
    raw = np.ascontiguousarray(np.asarray(store, dtype=F32)[3:3 + P, :n].transpose(1, 0, 2)).reshape(n, 4 * P)
    if half:
        w = raw.view(U32)
        raw = np.stack([w & 0xFFFF, w >> 16], axis=2).reshape(n, 8 * P).astype(np.uint16).view(np.float16).astype(F32)
    return raw[:, :3 * K]


def set_covariance(store, s, S):
    """Write the symmetric 3x3 S (float64) into slot s as the six float32 covariance words."""
    S = np.asarray(S, dtype=np.float64)
    store[1, s] = [S[0, 0], S[0, 1], S[0, 2], S[1, 1]]
    store[2, s, 0:2] = [S[1, 2], S[2, 2]]


def rotation(axis, angle):
    a = np.asarray(axis, dtype=np.float64)
    a = a / np.linalg.norm(a)
    K = np.array([[0.0, -a[2], a[1]], [a[2], 0.0, -a[0]], [-a[1], a[0], 0.0]])
    return np.eye(3) + np.sin(angle) * K + (1.0 - np.cos(angle)) * K @ K


def special_covariances(rng):
    """(name, S or six raw words) of the cases the decomposition must survive."""
    out = []
    for k in range(3):
        out.append(("isotropic", np.eye(3) * 10.0 ** rng.uniform(-6, 0)))
    R = rotation(rng.normal(size=3), 1.1)
    out.append(("repeated_pair", R @ np.diag([1e-3, 1e-3, 4e-2]) @ R.T))
    out.append(("repeated_pair_low", R @ np.diag([5e-2, 2e-4, 2e-4]) @ R.T))
    out.append(("needle", R @ np.diag([1e-12, 1e-12, 1.0]) * 1e-2 @ R.T))
    out.append(("disc", R @ np.diag([1e-14, 1e-2, 1e-2]) @ R.T))
    out.append(("needle_axis", np.diag([4.0, 4e-12, 4e-12])))
    out.append(("zero", np.zeros((3, 3))))
    out.append(("slightly_negative", R @ np.diag([-1e-10, 3e-3, 1e-2]) @ R.T))
    for axis in ((1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 0), (1, -1, 1)):
        R180 = rotation(axis, np.pi)
        out.append(("rot180", R180 @ np.diag([1e-3, 4e-3, 9e-3]) @ R180.T))
    out.append(("diagonal_desc", np.diag([9e-2, 4e-2, 1e-2])))
    for bad in (np.nan, np.inf, -np.inf):
        out.append(("nonfinite", bad))
    return out


def put_special(store, s, S):
    """Slot s gets the special covariance S (a float: every word finite except word s % 6)."""
    if np.isscalar(S):
        set_covariance(store, s, np.eye(3) * 1e-3)
        w = [(1, 0), (1, 1), (1, 2), (1, 3), (2, 0), (2, 1)][s % 6]
        store[w[0], s, w[1]] = S
    else:
        set_covariance(store, s, S)


# ---- the rule -------------------------------------------------------------------------------------------------------------------
def exported(store, n: int, hidden, selected, selected_only: bool) -> np.ndarray:
    """The exported store indices, ascending: [0, n), plane-0 x, y, z not NaN, in scope (hidden None: the masks are not in use)."""
    p0 = np.asarray(store, dtype=F32)[0, :n, :3]
    ok = ~np.isnan(p0).any(axis=1)
    if hidden is None:
        scope = np.zeros(n, dtype=bool) if selected_only else np.ones(n, dtype=bool)
    else:
        scope = np.asarray(selected, dtype=bool)[:n] if selected_only else ~np.asarray(hidden, dtype=bool)[:n]
    return np.flatnonzero(ok & scope)


def narrow(table, from_degree: int, degree: int) -> np.ndarray:
    """A degree_properties(from_degree) table -> the table of degree_properties(degree): f_rest keeps the first (degree+1)^2 - 1
    coefficients of each channel (f_rest is channel-major, so the names do not carry over between degrees)."""
    t = np.asarray(table)
    ks, kd = (from_degree + 1) ** 2 - 1, (degree + 1) ** 2 - 1
    rest = t[:, 9:9 + 3 * ks].reshape(t.shape[0], 3, ks)[:, :, :kd].reshape(t.shape[0], 3 * kd)
    return np.ascontiguousarray(np.concatenate([t[:, :9], rest, t[:, 9 + 3 * ks:]], axis=1))


def finite_covariance(store, idx) -> np.ndarray:
    s = np.asarray(store, dtype=F32)
    w = np.concatenate([s[1, idx], s[2, idx, :2]], axis=1)
    return np.isfinite(w).all(axis=1)


def covariances(store, idx) -> np.ndarray:
    s = np.asarray(store, dtype=F32)
    p1, p2 = s[1, idx].astype(np.float64), s[2, idx].astype(np.float64)
    S = np.empty((len(idx), 3, 3))
    S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2] = p1[:, 0], p1[:, 1], p1[:, 2], p1[:, 3], p2[:, 0], p2[:, 1]
    S[:, 1, 0], S[:, 2, 0], S[:, 2, 1] = S[:, 0, 1], S[:, 0, 2], S[:, 1, 2]
    return S


def quat_matrix(q) -> np.ndarray:
    q = np.asarray(q, dtype=np.float64)
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], axis=1),
                     np.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], axis=1),
                     np.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], axis=1)], axis=1)


def ulp_distance(a, b) -> np.ndarray:
    """|a - b| in float32 ulps (ordered bit patterns)."""
    def key(x):
        u = np.asarray(x, dtype=F32).view(np.int32).astype(np.int64)
        return np.where(u < 0, -(u & 0x7FFFFFFF), u)
    return np.abs(key(a) - key(b))


def check_rows(rows, store, n: int, bands: int, half: bool, hidden, selected, selected_only: bool, degree: int):
    """Every clause of the rule for a table of exported rows: count and order, then the fields."""
    idx = exported(store, n, hidden, selected, selected_only)
    rows = np.asarray(rows, dtype=F32)
    assert rows.shape == (idx.size, row_floats(degree)), (rows.shape, idx.size)
    if idx.size == 0:
        return idx
    names = degree_properties(degree)
    col = {nm: i for i, nm in enumerate(names)}
    s = np.asarray(store, dtype=F32)
    ok = finite_covariance(store, idx)
    # positions, normals, f_dc, f_rest bit for bit, opacity within 1 ulp: against store_to_table (restricted to degree d)
    fin = idx[ok]
    if fin.size:
        keep = np.zeros(n, dtype=bool)
        keep[fin] = True
        ref = narrow(store_to_table(store, n, bands, half, ~keep), bands - 1, degree)
        got = rows[ok]
        sc = col["scale_0"]
        np.testing.assert_array_equal(got[:, :col["opacity"]].view(U32), ref[:, :col["opacity"]].view(U32))
        assert ulp_distance(got[:, col["opacity"]], ref[:, col["opacity"]]).max() <= 1
        assert np.array_equal(got[:, col["opacity"]] == 0.0, ref[:, col["opacity"]] == 0.0)
        # scales and rotations
        S = covariances(store, fin)
        lam = np.linalg.eigvalsh(S)
        lmax = np.maximum(np.abs(lam).max(axis=1), np.finfo(np.float64).tiny)
        e = np.exp(2.0 * got[:, sc:sc + 3].astype(np.float64))
        assert (np.abs(e - lam) <= 1e-6 * lmax[:, None] + 1e-300).all(), np.abs(e - lam).max(axis=1) / lmax
        q = got[:, col["rot_0"]:col["rot_0"] + 4].astype(np.float64)
        assert (np.abs(np.linalg.norm(q, axis=1) - 1.0) <= 2.0 ** -22).all()
        assert (q[:, 0] >= 0.0).all()
        R = quat_matrix(q)
        rebuilt = R @ (e[:, :, None] * np.transpose(R, (0, 2, 1)))
        assert (np.abs(rebuilt - S).max(axis=(1, 2)) <= 1e-6 * lmax + 1e-300).all(), (np.abs(rebuilt - S).max(axis=(1, 2)) / lmax).max()
    bad = rows[~ok]
    if bad.size:
        np.testing.assert_array_equal(bad[:, col["scale_0"]:col["scale_0"] + 3].view(U32), np.full((bad.shape[0], 3), QNAN, dtype=U32))
        np.testing.assert_array_equal(bad[:, col["rot_0"]:col["rot_0"] + 4], np.tile(np.array([1, 0, 0, 0], dtype=F32), (bad.shape[0], 1)))
        # the other fields still follow the rule
        np.testing.assert_array_equal(bad[:, 0:3].view(U32), s[0, idx[~ok], :3].view(U32))
    return idx


# ---- the CPU kernel emulator ----------------------------------------------------------------------------------------------------
def emu():
    global _emu
    if _emu is None:
        out_dir = HERE if os.access(HERE, os.W_OK) else tempfile.mkdtemp(prefix="gsr_export_emu_")
        out = os.path.join(out_dir, "libexport_emu.so")
        deps = [os.path.join(HERE, "export_emu.cpp")] + cr._EMU_DEPS[1:] + [os.path.join(cr.CSRC, "selection.cu")]
        if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(d) for d in deps):
            tmp = f"{out}.{os.getpid()}.tmp"
            subprocess.run([os.environ.get("ORC_CXX", "/usr/bin/g++")] + cr._EMU_FLAGS + ["-I", cr.CUDA_INC, deps[0], "-o", tmp], check=True)
            os.replace(tmp, out)
        L = C.CDLL(out)
        vp, ull = C.c_void_p, C.c_ulonglong
        L.emu_export_ply.argtypes = [C.c_int, C.c_int, vp, ull, ull, vp, vp, C.c_int, C.c_int, vp, ull, C.c_uint, C.c_uint]
        L.emu_export_ply.restype = C.c_longlong
        _emu = L
    return _emu


def emu_export(store, bands, half, hidden, selected, n, selected_only, degree, ctas=4, slow=0, count_only=False):
    """The emulated kernels: the rows (or, count_only, the count).  hidden None: the masks are not in use."""
    s = np.ascontiguousarray(store, dtype=F32)
    m = s.shape[1]
    hw = None if hidden is None else pack_mask(hidden, len(hidden))
    sw = None if hidden is None else pack_mask(selected, len(selected))
    ptr = (lambda a: None if a is None else a.ctypes.data)
    L = emu()
    count = L.emu_export_ply(bands, int(half), s.ctypes.data, m, n, ptr(hw), ptr(sw), int(selected_only), degree, None, 0, ctas, slow)
    assert count >= 0
    if count_only:
        return int(count)
    rows = np.full((count, row_floats(degree)), np.nan, dtype=F32)
    if count:
        got = L.emu_export_ply(bands, int(half), s.ctypes.data, m, n, ptr(hw), ptr(sw), int(selected_only), degree, rows.ctypes.data, count,
                               ctas, slow)
        assert got == count, got
    return rows
