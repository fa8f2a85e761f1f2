"""Reference implementation of splat delete and duplicate (include/gsr.h "Splat delete and duplicate") for the tests.

TEST INFRASTRUCTURE.  Two parts:
  1. the rule in numpy: stores are (planes, plane_stride, 4) float32 arrays in the layout of GSR_BUF_SPLATS, masks bool arrays over
     max_splats; every word moves bit for bit, so the comparison is on the uint32 words;
  2. the CPU kernel emulator of compact_store_kernel and its follow-up kernels (tests/delete_reference/delete_emu.cpp), with several
     CTAs running at once.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from godotgaussiansplatting_b200.rasterizer import delete_remap, pack_mask, unpack_mask  # noqa: F401  (re-exported for the tests)
from tests import cutout_reference as cr

F32, U32 = np.float32, np.uint32
HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "delete_reference")
QNAN = 0x7FC00000
_emu = None


def vacant(store, lo, hi):
    """Slots [lo, hi) of a store made vacant in place: plane-0 x, y, z the quiet NaN, every other word +0."""
    w = store.view(U32)
    w[:, lo:hi] = 0
    w[0, lo:hi, :3] = QNAN


def vacate_slots(store, slots):
    """The slots of a bool mask (over the first slots of the store) made vacant in place, as a delete leaves them."""
    idx = np.flatnonzero(np.asarray(slots, dtype=bool))
    w = store.view(U32)
    w[:, idx] = 0
    w[0, idx, :3] = QNAN


# ---- the rule ---------------------------------------------------------------------------------------------------------------
def delete_rule(store, hidden, selected, n):
    """(store, hidden, selected, k) after gsr_delete_hidden of the cloud [0, n)."""
    out = np.ascontiguousarray(store, dtype=F32).copy()
    hid, sel = np.asarray(hidden, dtype=bool), np.asarray(selected, dtype=bool)
    kept = np.flatnonzero(~hid[:n])
    k = kept.size
    out[:, :k] = np.asarray(store, dtype=F32)[:, kept]
    vacant(out, k, n)
    new_sel = np.zeros_like(sel)
    new_sel[:k] = sel[kept]
    return out, np.zeros_like(hid), new_sel, k


def duplicate_rule(store, hidden, selected, n):
    """(store, hidden, selected, S) after gsr_duplicate_selection of the cloud [0, n) (the caller checks n + S <= max_splats)."""
    out = np.ascontiguousarray(store, dtype=F32).copy()
    hid, sel = np.asarray(hidden, dtype=bool).copy(), np.asarray(selected, dtype=bool)
    src = np.flatnonzero(sel[:n])
    S = src.size
    out[:, n:n + S] = np.asarray(store, dtype=F32)[:, src]
    new_sel = np.zeros_like(sel)
    new_sel[n:n + S] = True
    hid[n:n + S] = False
    return out, hid, new_sel, S


# ---- the CPU kernel emulator -------------------------------------------------------------------------------------------------
def emu():
    global _emu
    if _emu is None:
        out_dir = HERE if os.access(HERE, os.W_OK) else tempfile.mkdtemp(prefix="gsr_delete_emu_")
        out = os.path.join(out_dir, "libdelete_emu.so")
        deps = [os.path.join(HERE, "delete_emu.cpp")] + cr._EMU_DEPS[1:] + [os.path.join(cr.CSRC, "selection.cu")]
        if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(d) for d in deps):
            tmp = f"{out}.{os.getpid()}.tmp"
            subprocess.run([os.environ.get("ORC_CXX", "/usr/bin/g++")] + cr._EMU_FLAGS + ["-I", cr.CUDA_INC, deps[0], "-o", tmp], check=True)
            os.replace(tmp, out)
        L = C.CDLL(out)
        vp, ull = C.c_void_p, C.c_ulonglong
        L.emu_delete_hidden.argtypes = [C.c_int, C.c_int, vp, ull, ull, vp, vp, vp, C.c_uint, C.c_uint, C.c_uint]
        L.emu_delete_hidden.restype = C.c_longlong
        L.emu_duplicate_selection.argtypes = [C.c_int, C.c_int, vp, ull, ull, ull, vp, vp, C.c_uint, C.c_uint]
        L.emu_duplicate_selection.restype = C.c_longlong
        _emu = L
    return _emu


def emu_delete(store, bands, half, hidden, selected, n, ctas=4, slow=0):
    """The emulated kernels on copies: (store, hidden, selected, k).  slow > 0: the first CTA of every wave waits `slow` scheduler
    rounds between its first look-back and its loads (delete_emu.cpp g_slow)."""
    m = len(hidden)
    dst = np.ascontiguousarray(store, dtype=F32).copy()
    hw, sw = pack_mask(hidden, m).copy(), pack_mask(selected, m).copy()
    scratch = np.zeros_like(hw)
    k = emu().emu_delete_hidden(bands, int(half), dst.ctypes.data, dst.shape[1], n, hw.ctypes.data, sw.ctypes.data, scratch.ctypes.data,
                                hw.size, ctas, slow)
    assert k >= 0 and not scratch.any()
    return dst, unpack_mask(hw, m), unpack_mask(sw, m), int(k)


def emu_duplicate(store, bands, half, hidden, selected, n, max_splats, ctas=4):
    """The emulated kernels on copies: (store, hidden, selected, S), S = -2 - S' when the S' copies do not fit."""
    m = len(hidden)
    dst = np.ascontiguousarray(store, dtype=F32).copy()
    hw, sw = pack_mask(hidden, m).copy(), pack_mask(selected, m).copy()
    S = emu().emu_duplicate_selection(bands, int(half), dst.ctypes.data, dst.shape[1], n, max_splats, hw.ctypes.data, sw.ctypes.data, hw.size,
                                      ctas)
    assert S != -1
    return dst, unpack_mask(hw, m), unpack_mask(sw, m), int(S)
