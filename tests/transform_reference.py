"""Reference implementation of the selection transform (include/gsr.h "Splat transform edits") for the tests.

TEST INFRASTRUCTURE.  Three parts:
  1. the rule in numpy float32, one rounding per operation in the order of include/gsr.h, fed the library's own 95 constants (the
     emulator's edit_transform_matrices, or GSR_BUF_EDIT_TRANSFORM on the GPU);
  2. an independent float64 derivation of the SH band matrices (numpy's SVD for the polar factor, a least-squares fit on random
     directions), to check the library's;
  3. the CPU kernel emulator of transform_selection_kernel and of the host's matrix code (tests/transform_reference/transform_emu.cpp).
Stores are (planes, plane_stride, 4) float32 arrays in the layout of GSR_BUF_SPLATS.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from tests import cutout_reference as cr

F32, U32 = np.float32, np.uint32
HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "transform_reference")
OFFSET = {1: 12, 2: 21, 3: 46}   # M~_l in the 95 floats
SH_C = dict(c1=0.4886025119029199, c20=1.0925484305920792, c22=0.31539156525252005, c24=0.5462742152960396, c30=0.5900435899266435,
            c31=2.890611442640554, c32=0.4570457994644658, c33=0.3731763325901154, c35=1.445305721320277)
_emu = None


# ---- the SH band matrices --------------------------------------------------------------------------------------------------
def sh_poly(l, d):
    """P_l(d) for (n, 3) float64 directions: the polynomials that multiply coefficients l^2 .. l^2 + 2l in projection.cu's sh_color."""
    d = np.asarray(d, dtype=np.float64)
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    xx, yy, zz = x * x, y * y, z * z
    k = SH_C
    if l == 1:
        cols = [-k["c1"] * y, k["c1"] * z, -k["c1"] * x]
    elif l == 2:
        cols = [k["c20"] * x * y, -k["c20"] * y * z, k["c22"] * (2 * zz - xx - yy), -k["c20"] * x * z, k["c24"] * (xx - yy)]
    else:
        cols = [-k["c30"] * y * (3 * xx - yy), k["c31"] * x * y * z, -k["c32"] * y * (4 * zz - xx - yy), k["c33"] * z * (2 * zz - 3 * xx - 3 * yy),
                -k["c32"] * x * (4 * zz - xx - yy), k["c35"] * z * (xx - yy), -k["c30"] * x * (xx - 3 * yy)]
    return np.stack(cols, axis=1)


def polar(L):
    """The orthogonal polar factor U V^T of a 3x3 matrix (numpy's SVD)."""
    U, _, Vt = np.linalg.svd(np.asarray(L, dtype=np.float64))
    return U @ Vt


def band_matrix(Q, l, seed=0):
    """M_l with P_l(Q^T d) = M_l P_l(d), by least squares on 256 random directions."""
    d = np.random.default_rng(seed).normal(size=(256, 3))
    Pd, Pq = sh_poly(l, d), sh_poly(l, d @ np.asarray(Q, dtype=np.float64))   # row d Q = (Q^T d)^T
    Mt, *_ = np.linalg.lstsq(Pd, Pq, rcond=None)
    return Mt.T


def to_source_matrix(ts12):
    """[L | t] column-major 12 floats -> (L 3x3 float64, t 3 float64)."""
    m = np.asarray(ts12, dtype=np.float64).reshape(4, 3).T
    return m[:, :3], m[:, 3]


def unpack(m95):
    """The 95 floats -> (to_source 12, {l: M~_l}) as float32."""
    m = np.asarray(m95, dtype=F32)
    return m[:12], {l: m[OFFSET[l]:OFFSET[l] + (2 * l + 1) ** 2].reshape(2 * l + 1, 2 * l + 1) for l in (1, 2, 3)}


# ---- the rule in numpy float32 ---------------------------------------------------------------------------------------------
def sh_planes(bands, half):
    k3 = 3 * bands * bands
    return (k3 + 7) // 8 if half else (k3 + 3) // 4


def sh_half(c):
    """The upload's binary16 rounding: nearest even, +-65504 saturation, NaN stays NaN -> uint16 bits."""
    c = np.asarray(c, dtype=F32)
    with np.errstate(invalid="ignore"):
        c = np.where(np.abs(c) > F32(65504), np.copysign(F32(65504), c), c).astype(F32)
    return c.astype(np.float16).view(np.uint16)


def oracle(store, bands, half, selected, m95, src=None):
    """The store after gsr_transform_selection: selected = bool over [0, n) (n <= plane_stride), src = the planes read (None: store)."""
    store = np.asarray(store, dtype=F32)
    s = store if src is None else np.asarray(src, dtype=F32)
    out = store.copy()
    idx = np.flatnonzero(np.asarray(selected, dtype=bool))
    L, Ms = unpack(m95)
    out[:, idx] = s[:, idx]
    p0, p1, p2 = s[0, idx], s[1, idx], s[2, idx]
    S = [[p1[:, 0], p1[:, 1], p1[:, 2]], [p1[:, 1], p1[:, 3], p2[:, 0]], [p1[:, 2], p2[:, 0], p2[:, 1]]]
    with np.errstate(all="ignore"):
        for r in range(3):
            out[0, idx, r] = ((L[r] * p0[:, 0] + L[3 + r] * p0[:, 1]) + L[6 + r] * p0[:, 2]) + L[9 + r]
        G = [[(L[r] * S[0][c] + L[3 + r] * S[1][c]) + L[6 + r] * S[2][c] for c in range(3)] for r in range(3)]
        E = {(r, c): (G[r][0] * L[c] + G[r][1] * L[3 + c]) + G[r][2] * L[6 + c] for r in range(3) for c in range(r, 3)}
        out[1, idx] = np.stack([E[0, 0], E[0, 1], E[0, 2], E[1, 1]], axis=1)
        out[2, idx, 0], out[2, idx, 1] = E[1, 2], E[2, 2]
        P, nv = sh_planes(bands, half), 3 * bands * bands
        raw = np.ascontiguousarray(s[3:3 + P, idx].transpose(1, 0, 2)).view(U32).reshape(idx.size, 4 * P)
        if half:
            halves = np.stack([raw & U32(0xFFFF), raw >> U32(16)], axis=2).reshape(idx.size, 8 * P).astype(np.uint16)
            c = halves.view(np.float16).astype(F32)
        else:
            c = raw.view(F32).copy()
        for l in range(1, bands):
            n, k0, M = 2 * l + 1, l * l, Ms[l]
            new = c.copy()
            for ch in range(3):
                for j in range(n):
                    acc = c[:, 3 * k0 + ch] * M[0, j]
                    for i in range(1, n):
                        acc = acc + c[:, 3 * (k0 + i) + ch] * M[i, j]
                    new[:, 3 * (k0 + j) + ch] = acc
            c = new
        if half:
            h = sh_half(c).astype(U32)
            h[:, :3] = halves[:, :3]   # DC as stored
            h[:, nv:] = 0
            words = h[:, 0::2] | (h[:, 1::2] << U32(16))
        else:
            words = c.view(U32).copy()
            words[:, nv:] = 0
        out[3:3 + P, idx] = words.reshape(idx.size, P, 4).transpose(1, 0, 2).view(F32)
    return out


def _half_nan(h):
    return (h & 0x7C00) == 0x7C00 and (h & 0x3FF) != 0


def assert_store_equal(got, want, half, msg=""):
    """Bit for bit, except that a NaN may be any NaN (payloads differ between GPU, CPU and numpy): float words in planes 0-2 and float
    SH planes, binary16 halves in half SH planes."""
    g, w = np.ascontiguousarray(got, dtype=F32).view(U32), np.ascontiguousarray(want, dtype=F32).view(U32)
    assert g.shape == w.shape, (g.shape, w.shape)
    diff = np.argwhere(g != w)
    for p, s, k in diff:
        a, b = int(g[p, s, k]), int(w[p, s, k])
        if half and p >= 3:
            ok = all(_half_nan((a >> sh) & 0xFFFF) and _half_nan((b >> sh) & 0xFFFF) for sh in (0, 16) if ((a ^ b) >> sh) & 0xFFFF)
        else:
            ok = np.isnan(np.uint32(a).view(F32)) and np.isnan(np.uint32(b).view(F32))
        assert ok, f"{msg} plane {p} splat {s} word {k}: got {a:#010x}, want {b:#010x}"


# ---- the CPU kernel emulator -------------------------------------------------------------------------------------------------
def emu():
    global _emu
    if _emu is None:
        out_dir = HERE if os.access(HERE, os.W_OK) else tempfile.mkdtemp(prefix="gsr_transform_emu_")
        out = os.path.join(out_dir, "libtransform_emu.so")
        deps = [os.path.join(HERE, "transform_emu.cpp")] + cr._EMU_DEPS[1:] + [os.path.join(cr.CSRC, "selection.cu")]
        if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(d) for d in deps):
            tmp = f"{out}.{os.getpid()}.tmp"
            subprocess.run([os.environ.get("ORC_CXX", "/usr/bin/g++")] + cr._EMU_FLAGS + ["-I", cr.CUDA_INC, deps[0], "-o", tmp], check=True)
            os.replace(tmp, out)
        L = C.CDLL(out)
        vp = C.c_void_p
        L.emu_edit_matrices.argtypes = [vp, vp]
        L.emu_transform_selection.argtypes = [C.c_int, C.c_int, vp, vp, C.c_ulonglong, vp, C.c_uint, vp]
        L.emu_polar.argtypes = [vp, vp]
        L.emu_band_matrix.argtypes = [vp, C.c_int, vp]
        _emu = L
    return _emu


def lib_polar(L):
    """The library's float64 polar factor of a 3x3 matrix."""
    a = np.ascontiguousarray(L, dtype=np.float64)
    q = np.zeros((3, 3))
    emu().emu_polar(a.ctypes.data, q.ctypes.data)
    return q


def lib_band_matrix(Q, l):
    """The library's float64 M_l(Q)."""
    a = np.ascontiguousarray(Q, dtype=np.float64)
    m = np.zeros((2 * l + 1, 2 * l + 1))
    emu().emu_band_matrix(a.ctypes.data, l, m.ctypes.data)
    return m


def matrices(ts12):
    """The library's 95 floats for to_source (None for a singular L)."""
    t = np.ascontiguousarray(ts12, dtype=F32)
    out = np.zeros(95, dtype=F32)
    return out if emu().emu_edit_matrices(t.ctypes.data, out.ctypes.data) == 0 else None


def emu_transform(store, bands, half, selected_words, m95, src=None):
    """transform_selection_kernel on a copy of the store; selected_words = the packed mask (uint32)."""
    dst = np.ascontiguousarray(store, dtype=F32).copy()
    s = dst if src is None else np.ascontiguousarray(src, dtype=F32)
    words = np.ascontiguousarray(selected_words, dtype=U32)
    m = np.ascontiguousarray(m95, dtype=F32)
    assert emu().emu_transform_selection(bands, int(half), dst.ctypes.data, s.ctypes.data, dst.shape[1], words.ctypes.data, words.size,
                                         m.ctypes.data) == 0
    return dst
