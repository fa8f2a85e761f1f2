"""Reference implementations of splat contribution (include/gsr.h gsr_set_splat_contribution) for the tests.

TEST INFRASTRUCTURE.
  * contribution_oracle.c -- the per-pixel walk of the ID oracle (tests/id_reference/id_oracle.c) accumulated into the four fields,
    compiled together with tests/depth_reference/depth_oracle.c and oracle/gsr_oracle.c, which it extends without changing them;
  * slot_of -- the source slot of every drawn id of an instance layout (the mapping of splat_sources);
  * contribution_emu.cpp -- composite_contrib_kernel<CONTRACT> and the contribution variants of select_where_kernel and
    splat_histogram_kernel compiled for the CPU on top of tests/kernel_emu and tests/property_reference/property_emu.cpp;
  * prop_values / where_inside / histogram_rule -- the property rules in numpy, the stored-word properties from
    tests/property_reference.
The libraries are written next to their sources, or to a temporary directory when the tree is read-only.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from godotgaussiansplatting_b200 import _lib
from godotgaussiansplatting_b200.rasterizer import CONTRIBUTION_DTYPE, pack_mask, unpack_mask
from oracle import oracle as orc
from tests import cutout_reference as cr
from tests import depth_reference as dref
from tests import id_reference as idr
from tests import instance_reference as iref
from tests import property_reference as pref
from tests import selection_reference as sref

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "contribution_reference")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32, U32 = np.float32, np.uint32
CONTRIBUTION, PEAK, VIEWS, PIXELS = (_lib.GSR_PROP_CONTRIBUTION, _lib.GSR_PROP_PEAK_CONTRIBUTION, _lib.GSR_PROP_VIEWS,
                                      _lib.GSR_PROP_CONTRIBUTING_PIXELS)
CONTRIB_PROPS = [CONTRIBUTION, PEAK, VIEWS, PIXELS]

_ORACLE_DEPS = [os.path.join(HERE, "contribution_oracle.c"), os.path.join(ROOT, "tests", "depth_reference", "depth_oracle.c"),
                os.path.join(ROOT, "oracle", "gsr_oracle.c"), os.path.abspath(__file__)]
_EMU_DEPS = [os.path.join(HERE, "contribution_emu.cpp"), os.path.abspath(__file__),
             os.path.join(ROOT, "tests", "property_reference", "property_emu.cpp"), os.path.join(cr.CSRC, "selection.cu")] + cr._EMU_DEPS[1:]

_oracle = None
_emu = None


def _out_dir() -> str:
    if os.access(HERE, os.W_OK):
        return HERE
    d = os.path.join(tempfile.gettempdir(), f"gsr_contribution_reference_{os.getuid()}")
    os.makedirs(d, exist_ok=True)
    return d


def oracle_lib():
    global _oracle
    if _oracle is None:
        cc = os.environ.get("ORC_CC", "/usr/bin/gcc")
        out = os.path.join(_out_dir(), "libcontribution_oracle.so")
        if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(d) for d in _ORACLE_DEPS):
            tmp = f"{out}.{os.getpid()}.tmp"
            subprocess.run([cc] + dref._ORC_FLAGS + [_ORACLE_DEPS[0], "-o", tmp, "-lm"], check=True)
            os.replace(tmp, out)
        L = C.CDLL(out)
        L.cto_set_blend_contraction.argtypes = [C.c_int]
        vp = C.c_void_p
        L.cto_accumulate.argtypes = [vp, vp, vp, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp, C.c_int64]
        _oracle = L
    return _oracle


def emu_lib():
    global _emu
    if _emu is None:
        cxx = os.environ.get("ORC_CXX", "/usr/bin/g++")
        out = os.path.join(_out_dir(), "libcontribution_emu.so")
        if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(d) for d in _EMU_DEPS):
            tmp = f"{out}.{os.getpid()}.tmp"
            subprocess.run([cxx] + cr._EMU_FLAGS + ["-I", cr.CUDA_INC, _EMU_DEPS[0], "-o", tmp], check=True)
            os.replace(tmp, out)
        L = C.CDLL(out)
        vp, ull, u = C.c_void_p, C.c_ulonglong, C.c_uint
        L.emu_composite_contrib.restype = C.c_int
        L.emu_composite_contrib.argtypes = [C.c_int, vp, vp, vp, vp, vp, vp, vp, C.c_int, C.c_int, vp, vp, vp, vp, C.c_uint32, C.c_int,
                                            C.c_int, C.POINTER(ull)]
        L.emu_select_where_contrib.argtypes = [C.c_int, vp, ull, vp, vp, u, u, ull, ull, vp, u, vp]
        L.emu_splat_histogram_contrib.argtypes = [C.c_int, vp, ull, ull, ull, vp, vp, u, vp, vp, u, vp, vp, u, u, vp]
        _emu = L
    return _emu


# ---- the buffer --------------------------------------------------------------------------------------------------------------
def zeros(slots):
    """A zeroed contribution buffer of `slots` records (numpy, CONTRIBUTION_DTYPE)."""
    return np.zeros(slots, dtype=CONTRIBUTION_DTYPE)


def fields(buf):
    """(weight, pixels, peak bits, views) of a buffer: the four fields the rule defines (last_frame is the library's)."""
    b = np.asarray(buf).view(CONTRIBUTION_DTYPE)
    return b["weight"].copy(), b["pixels"].copy(), b["peak"].view(U32).copy(), b["views"].copy()


def assert_same(got, want):
    for name, g, w in zip(("weight", "pixels", "peak", "views"), fields(got), fields(want)):
        np.testing.assert_array_equal(g, w, err_msg=name)


def slot_of(ranges, drawn):
    """The source slot of every drawn id [0, drawn) of an instance layout ((first, count) per instance); padding ids map to 2^32 - 1."""
    w0, _ = iref.layout(ranges)
    out = np.full(drawn, 0xFFFFFFFF, dtype=U32)
    for k, (first, count) in enumerate(ranges):
        out[32 * w0[k]:32 * w0[k] + int(count)] = np.arange(int(first), int(first) + int(count), dtype=np.int64).astype(U32)
    return out


def instance_tables(ranges):
    """(warp_inst, desc) of an instance layout, as the library's device tables."""
    w0, _ = iref.layout(ranges)
    desc = np.zeros(len(ranges), dtype=[("first", "<u8"), ("count", "<u4"), ("warp0", "<u4")])
    for k, (first, count) in enumerate(ranges):
        desc[k] = (int(first), int(count), w0[k])
    return idr.warp_instances(ranges), desc


# ---- the oracle and the emulated kernel ----------------------------------------------------------------------------------------
def accumulate(buf, records, sorted_values, bounds, width, height, vp32, scene_depth=None, contract=True, ranges=None):
    """The oracle: adds one frame to `buf` (a CONTRIBUTION_DTYPE array over the slots) in place."""
    recs = np.ascontiguousarray(records)
    assert recs.dtype == orc.RECORD_DTYPE
    v = np.ascontiguousarray(sorted_values, dtype=U32)
    if v.size == 0:
        v = np.zeros(1, dtype=U32)
    b = np.ascontiguousarray(bounds, dtype=U32)
    vp = np.ascontiguousarray(vp32, dtype=F32).reshape(32)
    z = dref._scene_depth(scene_depth, width, height)
    n = len(buf)
    so = None if ranges is None else slot_of(ranges, len(recs))
    w, p, pk, vw = (np.ascontiguousarray(buf[f]) for f in ("weight", "pixels", "peak", "views"))
    seen = np.zeros(n, dtype=np.uint8)
    L = oracle_lib()
    L.cto_set_blend_contraction(int(bool(contract)))
    ptr = lambda a: None if a is None else a.ctypes.data
    try:
        L.cto_accumulate(recs.ctypes.data, v.ctypes.data, b.ctypes.data, int(width), int(height), vp.ctypes.data, ptr(z), ptr(so),
                         w.ctypes.data, p.ctypes.data, pk.ctypes.data, vw.ctypes.data, seen.ctypes.data, n)
    finally:
        L.cto_set_blend_contraction(1)
    buf["weight"], buf["pixels"], buf["peak"], buf["views"] = w, p, pk, vw
    return buf


def emu_composite_contrib(variant, buf, records, values, bounds, width, height, vp32, scene_depth=None, ranges=None, epoch=1, ctas=3,
                          overflow=False, frames=None):
    """composite_contrib_kernel<variant == 0> on the CPU emulator, adding one frame to `buf` in place.  frames: a uint32[1] counter or
    None.  Returns (rgba, depth, staged)."""
    out = np.zeros((height, width, 4), dtype=F32)
    depth = np.zeros((height, width), dtype=F32)
    vals = np.concatenate([np.asarray(values, dtype=U32), np.zeros(512, dtype=U32)])
    recs, bnds = np.ascontiguousarray(records), np.ascontiguousarray(bounds, dtype=U32)
    vp = np.ascontiguousarray(vp32, dtype=F32).reshape(32)
    z = dref._scene_depth(scene_depth, width, height)
    wi = desc = None
    if ranges is not None:
        wi, desc = instance_tables(ranges)
    assert buf.flags.c_contiguous and buf.dtype == CONTRIBUTION_DTYPE
    staged = C.c_ulonglong(0)
    ptr = lambda a: None if a is None else a.ctypes.data
    rc = emu_lib().emu_composite_contrib(int(variant), recs.ctypes.data, vals.ctypes.data, bnds.ctypes.data, out.ctypes.data,
                                         depth.ctypes.data, ptr(z), vp.ctypes.data, int(width), int(height), ptr(wi), ptr(desc),
                                         buf.ctypes.data, ptr(frames), int(epoch), int(ctas), int(bool(overflow)), C.byref(staged))
    assert rc == 0, "not every tile was rendered"
    return out, depth, int(staged.value)


# ---- the property rules ------------------------------------------------------------------------------------------------------
def prop_values(store, half, prop, rgb, buf):
    """A property of every slot: the contribution properties from the buffer, the others by tests/property_reference."""
    if prop not in CONTRIB_PROPS:
        return pref.values(store, half, prop, rgb)
    b = np.asarray(buf).view(CONTRIBUTION_DTYPE)
    m = np.asarray(store).shape[1]
    if prop == CONTRIBUTION:
        v = b["weight"].astype(F32) * F32(2.0 ** -24)   # round to nearest, then an exact scale
    elif prop == PEAK:
        v = b["peak"].copy()
    elif prop == VIEWS:
        v = b["views"].astype(F32)
    else:
        v = b["pixels"].astype(F32)
    out = np.zeros(m, dtype=F32)
    out[:len(v)] = v[:m]
    return out


def where_rule(store, half, hidden, selected, first, count, filters, op, buf):
    inside = pref.tested(store, first, count)
    for prop, lo, hi, rgb in filters:
        v = prop_values(store, half, prop, rgb, buf)
        with np.errstate(invalid="ignore"):
            inside &= (F32(lo) <= v) & (v <= F32(hi))
    m = len(hidden)
    return sref.combine(op, np.asarray(selected, dtype=bool), inside[:m], np.asarray(hidden, dtype=bool))


def histogram_rule(store, half, hidden, selected, first, count, prop, edges, buf):
    """(counts[bins + 3], (min, max)) of gsr_splat_histogram over the kept splats (hidden None: the masks are not in use)."""
    keep = pref.tested(store, first, count)
    if hidden is not None:
        keep[:len(hidden)] &= ~np.asarray(hidden, dtype=bool)
    v = prop_values(store, half, prop, (0.0, 0.0, 0.0), buf)[keep]
    e = np.asarray(edges, dtype=F32)
    B = e.size - 1
    nan = np.isnan(v)
    w = v[~nan]
    below, above = w < e[0], w > e[B]
    mid = w[~below & ~above]
    i = np.minimum(np.searchsorted(e, mid, side="right") - 1, B - 1)
    counts = np.zeros(B + 3, dtype=np.uint64)
    counts[:B] = np.bincount(i, minlength=B)
    counts[B], counts[B + 1], counts[B + 2] = below.sum(), above.sum(), nan.sum()
    if w.size == 0:
        return counts, (np.inf, -np.inf)
    k = pref.ord_key(w)
    return counts, (float(w[np.argmin(k)]), float(w[np.argmax(k)]))


def emu_where(store, half, hidden, selected, first, count, filters, op, buf):
    m = len(hidden)
    st = np.ascontiguousarray(store, dtype=F32)
    hw, sw = pack_mask(hidden, m), pack_mask(selected, m).copy()
    fa = pref.filter_array(filters)
    b = np.ascontiguousarray(buf)
    rc = emu_lib().emu_select_where_contrib(int(half), st.ctypes.data, st.shape[1], sw.ctypes.data, hw.ctypes.data, hw.size, op, first,
                                            count, C.addressof(fa), len(filters), b.ctypes.data)
    assert rc == 0
    return unpack_mask(sw, m)


def emu_histogram(store, half, hidden, first, count, prop, edges, buf, blocks=3, ctas=2):
    st = np.ascontiguousarray(store, dtype=F32)
    e = np.ascontiguousarray(edges, dtype=F32)
    B = e.size - 1
    counts = np.zeros(B + 3, dtype=np.uint64)
    keys = np.array([-2 ** 31, -2 ** 31], dtype=np.int32)
    hw = sw = None
    if hidden is not None:
        m = len(hidden)
        hw, sw = pack_mask(hidden, m), pack_mask(np.zeros(m, dtype=bool), m)
    f = pref.filter_array([(prop, 0.0, 0.0, (0.0, 0.0, 0.0))])
    b = np.ascontiguousarray(buf)
    rc = emu_lib().emu_splat_histogram_contrib(int(half), st.ctypes.data, st.shape[1], first, count, None if hw is None else hw.ctypes.data,
                                               None if sw is None else sw.ctypes.data, 0, C.addressof(f), e.ctypes.data, B,
                                               counts.ctypes.data, keys.ctypes.data, blocks, ctas, b.ctypes.data)
    assert rc == 0
    if keys[1] == -2 ** 31:
        return counts, (np.inf, -np.inf)
    k = keys.view(U32) ^ U32(0x80000000)
    lo, hi = int(~k[0] & 0xFFFFFFFF), int(k[1])
    back = lambda o: float(np.array([o ^ 0x80000000 if o >> 31 else ~o & 0xFFFFFFFF], dtype=U32).view(F32)[0])
    return counts, (back(lo), back(hi))
