"""Reference implementation of cutout frames (include/gsr.h gsr_set_cutouts) for the tests.

TEST INFRASTRUCTURE.  The oracle is composed from the unchanged oracle/ and the other references, like tests/depth_order_reference.py:
  1. the cut mask of every drawn id in numpy float32 with the library's operations and order: u[r] = ((C[r] x + C[3+r] y) + C[6+r] z)
     + C[9+r] on the source position sp = position * model_scale (GSR_CUTOUT_SOURCE) or the record's frame-space position (sp without
     instances, A sp + t with them: GSR_CUTOUT_FRAME);
  2. project with the frame's reference (oracle.project, tests/ortho_reference, tests/aa_reference, tests/instance_reference) at
     unlimited capacity and drop every pair whose value is cut -- the pairs stay in emission order, since the kernel's scan keeps
     drawn-id order;
  3. the counters from the remaining pairs: V = distinct values, M = pairs, last tile = max(key >> 16) (a rect's last tile is its
     largest pair tile); a static-capacity frame truncates to `cap` after the filter;
  4. the sort (the depth-order one for mode 1), oracle.boundaries, then oracle.render or tests/depth_reference.render_depth.
The emulated kernels (cutout_emu.cpp: projection_kernel<.., CUT = true> on tests/kernel_emu) are built on first use next to their sources,
or in a temporary directory when the tree is read-only.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from oracle import oracle as orc
from tests import depth_order_reference as dor
from tests import depth_reference as dref
from tests import instance_reference as iref

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cutout_reference")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "godotgaussiansplatting_b200", "csrc")
CUDA_INC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
_EMU_DEPS = [os.path.join(HERE, "cutout_emu.cpp"), os.path.abspath(__file__), os.path.join(ROOT, "include", "gsr.h")] + [
    os.path.join(ROOT, "tests", "kernel_emu", f) for f in ("kernel_emu.cpp", "cuda_shim.h")] + [
    os.path.join(ROOT, "oracle", "glsl_cpu", "glsl_emu.hpp")] + [
    os.path.join(CSRC, f) for f in ("compositor.cu", "ranges.cu", "radix_sort.cu", "projection.cu", "ingest.cu", "present.cu", "group.cu",
                                    "common.cuh")]
_EMU_FLAGS = ["-std=gnu++17", "-O1", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-w"]

F32 = np.float32
U32 = np.uint32
BOX, ELLIPSOID = 0, 1
KEEP, REMOVE = 0, 1
FRAME, SOURCE = 0, 1
MAX_CUTOUTS = 16
_emu = None

# CutoutArgs (csrc/common.cuh): the set split by action, KEEP volumes first
VOLUME_DTYPE = np.dtype([("m", "<f4", (12,)), ("kind", "<i4")])
ARGS_DTYPE = np.dtype([("n_keep", "<u4"), ("n_remove", "<u4"), ("vol", VOLUME_DTYPE, (MAX_CUTOUTS,))])


def _out_dir() -> str:
    if os.access(HERE, os.W_OK):
        return HERE
    d = os.path.join(tempfile.gettempdir(), f"gsr_cutout_reference_{os.getuid()}")
    os.makedirs(d, exist_ok=True)
    return d


def emu_lib():
    global _emu
    if _emu is None:
        out = os.path.join(_out_dir(), "libcutout_emu.so")
        if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(d) for d in _EMU_DEPS):
            cxx = os.environ.get("ORC_CXX", "/usr/bin/g++")
            tmp = f"{out}.{os.getpid()}.tmp"   # concurrent test processes each build their own copy and swap it in whole
            subprocess.run([cxx] + _EMU_FLAGS + ["-I", CUDA_INC, _EMU_DEPS[0], "-o", tmp], check=True)
            os.replace(tmp, out)
        L = C.CDLL(out)
        vp, uint = C.c_void_p, C.c_uint
        L.emu_cutout_args_bytes.restype = uint
        L.emu_cutout_projection.restype = C.c_longlong
        L.emu_cutout_projection.argtypes = [C.c_int, C.c_int, C.c_int, C.c_float, vp, C.c_ulonglong, uint, vp, vp, C.c_int, vp, vp, vp, vp,
                                            uint, C.POINTER(uint), C.POINTER(C.c_int), C.POINTER(uint), vp, vp, vp, vp]
        assert L.emu_cutout_args_bytes() == ARGS_DTYPE.itemsize
        _emu = L
    return _emu


# ---- volumes -----------------------------------------------------------------------------------------------------------------
def volume(to_local, shape=BOX, action=KEEP, space=FRAME):
    """One gsr_cutout: to_local as a (3, 4) matrix [A | t] (or its 12 column-major floats)."""
    m = np.asarray(to_local, dtype=F32)
    c12 = m.T.reshape(12) if m.shape == (3, 4) else m.reshape(12)
    return (c12.astype(F32), int(shape), int(action), int(space))


def box(centre, half, shape=BOX, action=KEEP, space=FRAME):
    """An axis-aligned box (or the ellipsoid inscribed in it) with the given centre and half extents, as a to_local volume."""
    c = np.asarray(centre, dtype=np.float64)
    h = np.asarray(half, dtype=np.float64) * np.ones(3)
    A = np.diag(1.0 / h)
    return volume(np.concatenate([A, (-A @ c)[:, None]], axis=1), shape, action, space)


def cutout_args(vols) -> np.ndarray:
    """The CutoutArgs that gsr_set_cutouts builds from `vols`: KEEP volumes first, each list in the given order."""
    a = np.zeros(1, dtype=ARGS_DTYPE)[0]
    j = 0
    for act in (KEEP, REMOVE):
        for c12, shape, action, space in vols:
            if action != act:
                continue
            a["vol"][j]["m"] = c12
            a["vol"][j]["kind"] = shape | (space << 1)
            j += 1
            if act == KEEP:
                a["n_keep"] += 1
            else:
                a["n_remove"] += 1
    return a


def inside(c12, shape, p) -> np.ndarray:
    """Is every (n, 3) float32 position p inside the unit shape of a volume?  One rounding per operation, IEEE comparisons."""
    Cm = np.asarray(c12, dtype=F32).reshape(12)
    p = np.asarray(p, dtype=F32).reshape(-1, 3)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    with np.errstate(all="ignore"):
        u = [((Cm[r] * x + Cm[3 + r] * y) + Cm[6 + r] * z) + Cm[9 + r] for r in range(3)]
        if shape == ELLIPSOID:
            return ((u[0] * u[0] + u[1] * u[1]) + u[2] * u[2]) <= F32(1.0)
        return (np.abs(u[0]) <= F32(1.0)) & (np.abs(u[1]) <= F32(1.0)) & (np.abs(u[2]) <= F32(1.0))


def drawn_mask(vols, sp, fp) -> np.ndarray:
    """The rule of gsr_set_cutouts for source positions sp and frame-space positions fp ((n, 3) float32): True = drawn."""
    n = np.asarray(sp).reshape(-1, 3).shape[0]
    in_keep, in_remove = np.zeros(n, dtype=bool), np.zeros(n, dtype=bool)
    for c12, shape, action, space in vols:
        hit = inside(c12, shape, sp if space == SOURCE else fp)
        if action == KEEP:
            in_keep |= hit
        else:
            in_remove |= hit
    if not any(v[2] == KEEP for v in vols):
        in_keep[:] = True
    return in_keep & ~in_remove


def positions(splat60, model_scale=1.0, inst=None):
    """(sp, fp) of every drawn id: without instances the splats' sp twice; with instances [(first, count, to_frame12)] the drawn-id
    layout of gsr_set_instances (padding ids get NaN, which no volume contains)."""
    s = np.ascontiguousarray(splat60, dtype=F32).reshape(-1, 60)
    sp_all = s[:, 0:3] * F32(model_scale)
    if inst is None:
        return sp_all, sp_all
    ranges = [(f, c) for f, c, _ in inst]
    w0, D = iref.layout(ranges)
    sp = np.full((D, 3), np.nan, dtype=F32)
    fp = np.full((D, 3), np.nan, dtype=F32)
    for k, (first, count, x) in enumerate(inst):
        ids = 32 * w0[k] + np.arange(count)
        sp[ids] = sp_all[first:first + count]
        fp[ids] = iref.frame_position(iref.inverse(x), sp_all[first:first + count])
    return sp, fp


# ---- the oracle --------------------------------------------------------------------------------------------------------------
def oracle_frame(splat60, vp32, ub, vols, v=0.0, ortho=False, heat=0.0, contract=True, inst=None, scene_depth=None, depth=False,
                 quirks=True, cap=None, depth_order=False):
    """A whole cutout frame (steps 1-4).  inst = [(first, count, to_frame12)]; cap truncates the pairs like GSR_FLAG_STATIC_CAPACITY;
    depth_order sorts like GSR_DEPTH_ORDER_VIEW_DEPTH.  Returns a dict of every stage; `unsorted_keys` / `unsorted_values` are the
    pairs in emission order, `mask` the drawn mask per id."""
    u = orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8))
    W, H = u.dims[0], u.dims[1]
    pr = dor.project(splat60, vp32, u, v, ortho, inst)
    sp, fp = positions(splat60, u.model_scale, inst)
    mask = drawn_mask(vols, sp, fp)
    sel = mask[pr.values.astype(np.int64)]
    keys, values = pr.keys[sel].astype(U32), pr.values[sel].astype(U32)
    m, visible = int(keys.size), int(np.unique(values).size)
    last = int((keys >> U32(16)).max()) if m else -1
    if cap is not None:
        keys, values = keys[:cap], values[:cap]
    if depth_order:
        k, vals, _ = dor.sort_by_depth(keys, values, dor.ord_words(dor.view_depth(pr.records, values, vp32)))
    else:
        k, vals = orc.sort_pairs(keys, values)
    T = ((W + 15) // 16) * ((H + 15) // 16)
    b = orc.boundaries(k, T, quirks=quirks)
    dep = None
    if depth or scene_depth is not None:
        rgba, dep, staged = dref.render_depth(pr.records, vals, b, W, H, vp32, scene_depth, heat, contract)
    else:
        orc.set_blend_contraction(contract)
        try:
            rgba, staged, _ = orc.render(pr.records, vals, b, W, H, heat)
        finally:
            orc.set_blend_contraction(True)
    return dict(rgba=rgba, records=pr.records, keys=k, values=vals, unsorted_keys=keys, unsorted_values=values, bounds=b, visible=visible,
                m=m, last_tile=last, staged=staged, depth=dep, mask=mask, overflow=cap is not None and m > cap)


# ---- the emulated kernels ----------------------------------------------------------------------------------------------------
def emu_project(store, bands, vp, ub, bulk_min, num_splats, vols=None, v=0.0, ortho=False, ranges=None, xf=None, capacity=None,
                depth=False):
    """projection_kernel<ranges is not None, bands, ortho, v > 0, depth, vols is not None> over `store` on the CPU.  Returns (records,
    keys, values, depth words or None, M, V, last tile, overflow) with the pairs in emission order."""
    stride = store.shape[1]
    inst = ranges is not None
    frame_c = desc = warp_inst = None
    n = int(num_splats)
    if inst:
        w0, D = iref.layout(ranges)
        u = orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8))
        frame_c = np.zeros((len(ranges), 32), dtype=F32)
        for k in range(len(ranges)):
            Vk, camk = iref.compose(vp[:16], u.camera_pos[:], xf[k])
            frame_c[k, :16], frame_c[k, 16:19], frame_c[k, 19:31] = Vk, camk, xf[k][:12]
        warp_inst = np.full(((D + 255) // 256) * 8 + 1, 0xFFFFFFFF, dtype=U32)
        for k, (_, c) in enumerate(ranges):
            warp_inst[w0[k]:w0[k] + (c + 31) // 32] = k
        desc = np.zeros(max(len(ranges), 1), dtype=np.dtype([("first", "<u8"), ("count", "<u4"), ("warp0", "<u4")]))
        for k, (f, c) in enumerate(ranges):
            desc[k] = (f, c, w0[k])
        n = D
    cap = int(capacity if capacity is not None else 64 * max(n, 1))
    recs = np.zeros(max(n, 1), dtype=orc.RECORD_DTYPE)
    keys = np.zeros(max(cap, 1), dtype=U32)
    vals = np.zeros(max(cap, 1), dtype=U32)
    words = np.zeros(max(cap, 1), dtype=U32) if depth else None
    args = None if vols is None else np.array([cutout_args(vols)], dtype=ARGS_DTYPE)
    vis, last, ovf = C.c_uint(0), C.c_int(-1), C.c_uint(0)
    vp32 = np.ascontiguousarray(vp, dtype=F32)
    ubuf = np.frombuffer(ub, dtype=np.uint8).copy()
    m = emu_lib().emu_cutout_projection(int(inst), int(bands), int(bool(ortho)), float(v), store.ctypes.data, stride, n, vp32.ctypes.data,
                                        ubuf.ctypes.data, int(bulk_min), recs.ctypes.data, keys.ctypes.data, vals.ctypes.data,
                                        None if words is None else words.ctypes.data, cap, C.byref(vis), C.byref(last), C.byref(ovf),
                                        None if frame_c is None else frame_c.ctypes.data, None if desc is None else desc.ctypes.data,
                                        None if warp_inst is None else warp_inst.ctypes.data, None if args is None else args.ctypes.data)
    assert m >= 0
    mm = min(int(m), cap)
    return (recs[:n], keys[:mm].copy(), vals[:mm].copy(), None if words is None else words[:mm].copy(), int(m), int(vis.value),
            int(last.value), int(ovf.value))
