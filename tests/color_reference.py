"""Reference implementation of the selection colour edit (include/gsr.h "Splat colour edits") for the tests.

TEST INFRASTRUCTURE.  Three parts:
  1. the rule in numpy float32, one rounding per operation in the order of include/gsr.h, fed 41 constants: the library's own (the
     emulator's edit_color_constants, or GSR_BUF_EDIT_COLOR on the GPU) or those of the independent float64 derivation below;
  2. that derivation in numpy float64, to check the library's constants;
  3. the CPU kernel emulator of recolor_selection_kernel and edit_color_constants (tests/color_reference/color_emu.cpp).
Stores are (planes, plane_stride, 4) float32 arrays in the layout of GSR_BUF_SPLATS.  The binary16 rounding and the store comparison are
those of tests/transform_reference.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from godotgaussiansplatting_b200 import _lib
from tests import cutout_reference as cr
from tests.transform_reference import assert_store_equal, sh_half, sh_planes  # noqa: F401  (re-exported for the tests)

F32, U32 = np.float32, np.uint32
HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "color_reference")
SH_C0 = float(F32(0.28209479177387814))   # the projection's float SH_C0, widened
_emu = None


def edit_struct(matrix34=None, band_scale=(1.0, 1.0, 1.0), opacity_scale=1.0, opacity_offset=0.0) -> _lib.GsrColorEdit:
    """A gsr_color_edit from a row-major (3, 4) [A | b] (None: the identity)."""
    m = np.hstack([np.eye(3), np.zeros((3, 1))]) if matrix34 is None else np.asarray(matrix34, dtype=np.float64)
    e = _lib.GsrColorEdit()
    e.matrix[:] = [float(v) for v in np.concatenate([m[:, :3].T.reshape(9), m[:, 3]]).astype(F32)]
    e.band_scale[:] = [float(F32(v)) for v in band_scale]
    e.opacity_scale, e.opacity_offset = float(F32(opacity_scale)), float(F32(opacity_offset))
    return e


def affine(e):
    """(A, b) of an edit as float64 (exact: from its float fields)."""
    m = np.array(e.matrix[:], dtype=np.float64)
    return m[:9].reshape(3, 3).T.copy(), m[9:].copy()


# ---- the constants ------------------------------------------------------------------------------------------------------------
def constants_numpy(e):
    """The 41 constants derived independently in numpy float64, each rounded to float32 once."""
    A, b = affine(e)
    d = ((((A[:, 0] * 0.5 + A[:, 1] * 0.5) + A[:, 2] * 0.5) + b) - 0.5) / SH_C0
    N = [float(s) * A for s in e.band_scale[:]]
    return np.concatenate([A.reshape(9), d] + [n.reshape(9) for n in N] + [[e.opacity_scale, e.opacity_offset]]).astype(F32)


def unpack(k41):
    k = np.asarray(k41, dtype=F32)
    return k[0:9].reshape(3, 3), k[9:12], {l: k[12 + 9 * (l - 1):21 + 9 * (l - 1)].reshape(3, 3) for l in (1, 2, 3)}, k[39], k[40]


def band_of(k):
    return 0 if k == 0 else 1 if k < 4 else 2 if k < 9 else 3


# ---- the rule in numpy float32 ---------------------------------------------------------------------------------------------
def oracle(store, bands, half, selected, k41, src=None):
    """The store after gsr_recolor_selection: selected = bool over [0, n) (n <= plane_stride), src = the planes read (None: store)."""
    store = np.asarray(store, dtype=F32)
    s = store if src is None else np.asarray(src, dtype=F32)
    out = store.copy()
    idx = np.flatnonzero(np.asarray(selected, dtype=bool))
    A, d, N, sc, t = unpack(k41)
    out[:, idx] = s[:, idx]
    with np.errstate(all="ignore"):
        u = (s[2, idx, 2] * sc) + t
        out[2, idx, 2] = np.where(u > F32(1), F32(1), np.where(u > F32(0), u, F32(0)))
        P, nv = sh_planes(bands, half), 3 * bands * bands
        raw = np.ascontiguousarray(s[3:3 + P, idx].transpose(1, 0, 2)).view(U32).reshape(idx.size, 4 * P)
        if half:
            c = np.stack([raw & U32(0xFFFF), raw >> U32(16)], axis=2).reshape(idx.size, 8 * P).astype(np.uint16).view(np.float16).astype(F32)
        else:
            c = raw.view(F32).copy()
        new = c.copy()
        for k in range(bands * bands):
            M = A if k == 0 else N[band_of(k)]
            r, g, b = c[:, 3 * k], c[:, 3 * k + 1], c[:, 3 * k + 2]
            for i in range(3):
                v = (M[i, 0] * r + M[i, 1] * g) + M[i, 2] * b
                new[:, 3 * k + i] = v + d[i] if k == 0 else v
        if half:
            h = sh_half(new).astype(U32)
            h[:, nv:] = 0
            words = h[:, 0::2] | (h[:, 1::2] << U32(16))
        else:
            words = new.view(U32).copy()
            words[:, nv:] = 0
        out[3:3 + P, idx] = words.reshape(idx.size, P, 4).transpose(1, 0, 2).view(F32)
    return out


# ---- the CPU kernel emulator -------------------------------------------------------------------------------------------------
def emu():
    global _emu
    if _emu is None:
        out_dir = HERE if os.access(HERE, os.W_OK) else tempfile.mkdtemp(prefix="gsr_color_emu_")
        out = os.path.join(out_dir, "libcolor_emu.so")
        deps = [os.path.join(HERE, "color_emu.cpp")] + cr._EMU_DEPS[1:] + [os.path.join(cr.CSRC, "selection.cu")]
        if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(d) for d in deps):
            tmp = f"{out}.{os.getpid()}.tmp"
            subprocess.run([os.environ.get("ORC_CXX", "/usr/bin/g++")] + cr._EMU_FLAGS + ["-I", cr.CUDA_INC, deps[0], "-o", tmp], check=True)
            os.replace(tmp, out)
        L = C.CDLL(out)
        vp = C.c_void_p
        L.emu_color_constants.argtypes = [C.POINTER(_lib.GsrColorEdit), vp]
        L.emu_recolor_selection.argtypes = [C.c_int, C.c_int, vp, vp, C.c_ulonglong, vp, C.c_uint, vp]
        L.emu_ply_to_soa.argtypes = [vp, C.c_uint, C.c_ulonglong, C.c_float, vp, C.c_ulonglong, C.c_ulonglong]
        _emu = L
    return _emu


def constants(e):
    """The library's 41 constants of an edit."""
    out = np.zeros(41, dtype=F32)
    emu().emu_color_constants(C.byref(e), out.ctypes.data)
    return out


def emu_recolor(store, bands, half, selected_words, k41, src=None):
    """recolor_selection_kernel on a copy of the store; selected_words = the packed mask (uint32)."""
    dst = np.ascontiguousarray(store, dtype=F32).copy()
    s = dst if src is None else np.ascontiguousarray(src, dtype=F32)
    words = np.ascontiguousarray(selected_words, dtype=U32)
    k = np.ascontiguousarray(k41, dtype=F32)
    assert emu().emu_recolor_selection(bands, int(half), dst.ctypes.data, s.ctypes.data, dst.shape[1], words.ctypes.data, words.size,
                                       k.ctypes.data) == 0
    return dst
