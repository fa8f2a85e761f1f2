"""Reference implementation of splat property selection (include/gsr.h "Splat property selection") for the tests.

TEST INFRASTRUCTURE.  Two parts:
  1. the rule in numpy float32, one rounding per operation in the order of include/gsr.h: stores are (planes, plane_stride, 4) float32
     arrays in the layout of GSR_BUF_SPLATS, masks bool arrays over max_splats; the histogram bins by np.searchsorted on the rule;
  2. the CPU kernel emulator of select_where_kernel and splat_histogram_kernel (tests/property_reference/property_emu.cpp), the histogram
     with several CTAs running at once.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from godotgaussiansplatting_b200 import _lib
from godotgaussiansplatting_b200.rasterizer import pack_mask, unpack_mask
from tests import cutout_reference as cr
from tests import selection_reference as sref

F32, U32 = np.float32, np.uint32
HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "property_reference")
OPACITY, SIZE, VOLUME, ISOTROPY, COLOR = range(5)
PROPS = [OPACITY, SIZE, VOLUME, ISOTROPY, COLOR]
SH_C0 = F32(0.28209479177387814)
_emu = None


# ---- the rule ---------------------------------------------------------------------------------------------------------------
def dc_of(store, half):
    """f_r, f_g, f_b of every slot: plane 3 x, y, z, or half slots 0..2 of plane 3 widened."""
    p3 = np.asarray(store, dtype=F32)[3]
    if not half:
        return p3[:, 0], p3[:, 1], p3[:, 2]
    w = p3.view(U32)
    h = lambda u: (u & 0xFFFF).astype(np.uint16).view(np.float16).astype(F32)
    return h(w[:, 0]), h(w[:, 0] >> 16), h(w[:, 1])


def values(store, half, prop, rgb=(0.0, 0.0, 0.0)):
    """The property of every slot of the store (float32)."""
    s = np.asarray(store, dtype=F32)
    with np.errstate(all="ignore"):
        if prop == OPACITY:
            return s[2, :, 2].copy()
        if prop == COLOR:
            d2 = None
            for i, f in enumerate(dc_of(s, half)):
                d = (F32(0.5) + f * SH_C0) - F32(rgb[i])
                d2 = d * d if d2 is None else d2 + d * d
            return d2
        S00, S01, S02, S11 = (s[1, :, k] for k in range(4))
        S12, S22 = s[2, :, 0], s[2, :, 1]
        t = (S00 + S11) + S22
        if prop == SIZE:
            return t
        det = ((S00 * ((S11 * S22) - (S12 * S12))) - (S01 * ((S01 * S22) - (S12 * S02)))) + (S02 * ((S01 * S12) - (S11 * S02)))
        if prop == VOLUME:
            return det
        return (F32(27.0) * det) / ((t * t) * t)


def tested(store, first, count):
    """The splats of [first, first + count) (count already bounded by the cloud) whose plane-0 x, y, z are not NaN."""
    m = np.asarray(store).shape[1]
    idx = np.arange(m)
    ok = (idx >= first) & (idx < first + count)
    return ok & ~np.isnan(np.asarray(store, dtype=F32)[0, :, :3]).any(axis=1)


def where_inside(store, half, first, count, filters):
    """inside of gsr_select_where: filters = [(property, lo, hi, rgb)]."""
    inside = tested(store, first, count)
    for prop, lo, hi, rgb in filters:
        v = values(store, half, prop, rgb)
        with np.errstate(invalid="ignore"):
            inside &= (F32(lo) <= v) & (v <= F32(hi))
    return inside


def where_rule(store, half, hidden, selected, first, count, filters, op):
    """The selected mask after gsr_select_where (the mask arrays cover the store's slots [0, max_splats))."""
    m = len(hidden)
    inside = where_inside(store, half, first, count, filters)[:m]
    return sref.combine(op, np.asarray(selected, dtype=bool), inside, np.asarray(hidden, dtype=bool))


def ord_key(v):
    """gsr_set_depth_order's ord of float32 values."""
    b = np.ascontiguousarray(v, dtype=F32).view(U32)
    return np.where(b >> 31 != 0, ~b, b | U32(0x80000000)).astype(U32)


def histogram_rule(store, half, hidden, selected, first, count, prop, rgb, edges, selected_only):
    """(counts[bins + 3], (min, max)) of gsr_splat_histogram; hidden None: the masks are not in use."""
    m = np.asarray(store).shape[1]
    keep = tested(store, first, count)
    if hidden is not None:
        h = np.zeros(m, dtype=bool)
        h[:len(hidden)] = hidden
        keep &= ~h
        if selected_only:
            s = np.zeros(m, dtype=bool)
            s[:len(selected)] = selected
            keep &= s
    elif selected_only:
        keep[:] = False
    v = values(store, half, prop, rgb)[keep]
    e = np.asarray(edges, dtype=F32)
    B = e.size - 1
    nan = np.isnan(v)
    w = v[~nan]
    below, above = w < e[0], w > e[B]
    mid = w[~below & ~above]
    i = np.minimum(np.searchsorted(e, mid, side="right") - 1, B - 1)   # e_i <= v < e_{i+1}; v == e_B in the last bin
    counts = np.zeros(B + 3, dtype=np.uint64)
    counts[:B] = np.bincount(i, minlength=B)
    counts[B], counts[B + 1], counts[B + 2] = below.sum(), above.sum(), nan.sum()
    if w.size == 0:
        return counts, (np.inf, -np.inf)
    k = ord_key(w)
    return counts, (float(w[np.argmin(k)]), float(w[np.argmax(k)]))


# ---- the CPU kernel emulator -------------------------------------------------------------------------------------------------
def emu():
    global _emu
    if _emu is None:
        out_dir = HERE if os.access(HERE, os.W_OK) else tempfile.mkdtemp(prefix="gsr_property_emu_")
        out = os.path.join(out_dir, "libproperty_emu.so")
        deps = [os.path.join(HERE, "property_emu.cpp"), os.path.abspath(__file__)] + cr._EMU_DEPS[1:] + [os.path.join(cr.CSRC, "selection.cu")]
        if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(d) for d in deps):
            tmp = f"{out}.{os.getpid()}.tmp"
            subprocess.run([os.environ.get("ORC_CXX", "/usr/bin/g++")] + cr._EMU_FLAGS + ["-I", cr.CUDA_INC, deps[0], "-o", tmp], check=True)
            os.replace(tmp, out)
        L = C.CDLL(out)
        vp, ull, u = C.c_void_p, C.c_ulonglong, C.c_uint
        L.emu_select_where.argtypes = [C.c_int, vp, ull, vp, vp, u, u, ull, ull, vp, u]
        L.emu_splat_histogram.argtypes = [C.c_int, vp, ull, ull, ull, vp, vp, u, vp, vp, u, vp, vp, u, u]
        _emu = L
    return _emu


def filter_array(filters):
    arr = (_lib.GsrSplatFilter * max(1, len(filters)))()
    for k, (prop, lo, hi, rgb) in enumerate(filters):
        arr[k].property, arr[k].lo, arr[k].hi = int(prop), float(lo), float(hi)
        arr[k].rgb[:] = [float(x) for x in rgb]
    return arr


def emu_where(store, half, hidden, selected, first, count, filters, op):
    """The emulated kernel on copies of the masks: the selected mask after it."""
    m = len(hidden)
    st = np.ascontiguousarray(store, dtype=F32)
    hw, sw = pack_mask(hidden, m), pack_mask(selected, m).copy()
    fa = filter_array(filters)
    rc = emu().emu_select_where(int(half), st.ctypes.data, st.shape[1], sw.ctypes.data, hw.ctypes.data, hw.size, op, first, count,
                                C.addressof(fa), len(filters))
    assert rc == 0
    return unpack_mask(sw, m)


def emu_histogram(store, half, hidden, selected, first, count, prop, rgb, edges, selected_only, blocks=1, ctas=1):
    """The emulated kernel (blocks CTAs, ctas of them at once): (counts, (min, max)) as gsr_splat_histogram returns them."""
    st = np.ascontiguousarray(store, dtype=F32)
    e = np.ascontiguousarray(edges, dtype=F32)
    B = e.size - 1
    counts = np.zeros(B + 3, dtype=np.uint64)
    keys = np.array([-2 ** 31, -2 ** 31], dtype=np.int32)   # HistArgs.keys: max of s(~ord) and of s(ord), s = the signed key
    hw = sw = None
    if hidden is not None:
        m = len(hidden)
        hw, sw = pack_mask(hidden, m), pack_mask(selected, m)
    f = filter_array([(prop, 0.0, 0.0, rgb)])
    rc = emu().emu_splat_histogram(int(half), st.ctypes.data, st.shape[1], first, count, None if hw is None else hw.ctypes.data,
                                   None if sw is None else sw.ctypes.data, int(selected_only), C.addressof(f), e.ctypes.data, B,
                                   counts.ctypes.data, keys.ctypes.data, blocks, ctas)
    assert rc == 0
    if keys[1] == -2 ** 31:
        return counts, (np.inf, -np.inf)
    k = keys.view(U32) ^ U32(0x80000000)
    lo, hi = int(~k[0] & 0xFFFFFFFF), int(k[1])
    back = lambda o: float(np.array([o ^ 0x80000000 if o >> 31 else ~o & 0xFFFFFFFF], dtype=U32).view(F32)[0])   # ord back to the float
    return counts, (back(lo), back(hi))
