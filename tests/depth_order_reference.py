"""Reference implementation of depth-ordered frames (include/gsr.h gsr_set_depth_order) for the tests.

TEST INFRASTRUCTURE.  The oracle is composed from the unchanged oracle/ and the other references, like tests/instance_reference.py:
  1. project with oracle.project, or tests/ortho_reference, tests/aa_reference or tests/instance_reference as the frame needs: records
     and the pairs in emission order;
  2. d per pair from its record's position with numpy float32 operations in the library's order,
     d = -(((V[2] x + V[6] y) + V[10] z) + V[14] * 1);
  3. a stable sort by (key >> 16) << 32 | ord(d) as uint64;
  4. oracle.boundaries, then oracle.render -- or tests/depth_reference.render_depth for depth compositing.
The emulated kernels (depth_order_emu.cpp: projection_kernel<.., DEPTH = true> and the six-pass sort on tests/kernel_emu) are built on
first use next to their sources, or in a temporary directory when the tree is read-only.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from oracle import oracle as orc
from tests import aa_reference as aref
from tests import depth_reference as dref
from tests import instance_reference as iref
from tests import ortho_reference as oref

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "depth_order_reference")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "godotgaussiansplatting_b200", "csrc")
CUDA_INC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
_EMU_DEPS = [os.path.join(HERE, "depth_order_emu.cpp"), os.path.abspath(__file__), os.path.join(ROOT, "include", "gsr.h")] + [
    os.path.join(ROOT, "tests", "kernel_emu", f) for f in ("kernel_emu.cpp", "cuda_shim.h")] + [
    os.path.join(ROOT, "oracle", "glsl_cpu", "glsl_emu.hpp")] + [
    os.path.join(CSRC, f) for f in ("compositor.cu", "ranges.cu", "radix_sort.cu", "projection.cu", "ingest.cu", "present.cu", "group.cu",
                                    "common.cuh")]
_EMU_FLAGS = ["-std=gnu++17", "-O1", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-w"]

F32 = np.float32
U32 = np.uint32
_emu = None


def _out_dir() -> str:
    if os.access(HERE, os.W_OK):
        return HERE
    d = os.path.join(tempfile.gettempdir(), f"gsr_depth_order_reference_{os.getuid()}")
    os.makedirs(d, exist_ok=True)
    return d


def emu_lib():
    global _emu
    if _emu is None:
        out = os.path.join(_out_dir(), "libdepth_order_emu.so")
        if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(d) for d in _EMU_DEPS):
            cxx = os.environ.get("ORC_CXX", "/usr/bin/g++")
            tmp = f"{out}.{os.getpid()}.tmp"   # concurrent test processes each build their own copy and swap it in whole
            subprocess.run([cxx] + _EMU_FLAGS + ["-I", CUDA_INC, _EMU_DEPS[0], "-o", tmp], check=True)
            os.replace(tmp, out)
        L = C.CDLL(out)
        vp, uint = C.c_void_p, C.c_uint
        L.emu_depth_projection.restype = C.c_longlong
        L.emu_depth_projection.argtypes = [C.c_int, C.c_int, C.c_int, C.c_float, vp, C.c_ulonglong, uint, vp, vp, C.c_int, vp, vp, vp, vp, uint,
                                           C.POINTER(uint), C.POINTER(C.c_int), C.POINTER(uint), vp, vp, vp]
        L.emu_depth_sort.argtypes = [vp, vp, vp, C.c_uint32, C.c_uint32, C.c_int]
        _emu = L
    return _emu


# ---- the oracle --------------------------------------------------------------------------------------------------------------
def ord_words(d) -> np.ndarray:
    """ord(f) = bits(f) ^ (sign ? 0xFFFFFFFF : 0x80000000): unsigned order = float order for every finite f, -0 just before +0."""
    b = np.ascontiguousarray(d, dtype=F32).view(U32)
    return b ^ np.where(b >> U32(31), U32(0xFFFFFFFF), U32(0x80000000)).astype(U32)


def view_depth(records, values, vp32) -> np.ndarray:
    """d of every pair: -(((V2 x + V6 y) + V10 z) + V14 * 1) in float32 from the record's position (the compositor's d)."""
    V = np.asarray(vp32, dtype=F32).reshape(32)
    r = records[np.asarray(values, dtype=np.int64)]
    x, y, z = r["pos_xy"][:, 0].astype(F32), r["pos_xy"][:, 1].astype(F32), r["pos_z"].astype(F32)
    with np.errstate(all="ignore"):
        return -(((V[2] * x + V[6] * y) + V[10] * z) + V[14] * F32(1.0))


def sort_by_depth(keys, values, words):
    """Stable sort by (key >> 16) << 32 | word.  Returns (keys, values, words) in the sorted order."""
    keys, values, words = (np.asarray(a, dtype=U32) for a in (keys, values, words))
    o = np.argsort(((keys >> U32(16)).astype(np.uint64) << np.uint64(32)) | words.astype(np.uint64), kind="stable")
    return keys[o], values[o], words[o]


def project(splat60, vp32, u, v=0.0, ortho=False, inst=None, cap=None):
    """Step 1: records and the pairs in emission order (orc.Projection or iref.InstanceProjection)."""
    if inst is not None:
        ranges = [(f, n) for f, n, _ in inst]
        xf = np.stack([iref.inverse(x) for _, _, x in inst])
        if v > 0:
            return aref.project_instanced(splat60, vp32, u, ranges, xf, v, ortho)
        if ortho:
            return oref.project_instanced(splat60, vp32, u, ranges, xf)
        return iref.project(splat60, vp32, u, ranges, xf)
    n = np.asarray(splat60).reshape(-1, 60).shape[0]
    cap = int(cap if cap is not None else 64 * max(n, 1))
    if v > 0:
        return aref.project(splat60, vp32, u, v, ortho, cap=cap)
    if ortho:
        return oref.project(splat60, vp32, u, cap=cap)
    return orc.project(splat60, vp32, u, cap=cap)


def oracle_frame(splat60, vp32, ub, v=0.0, ortho=False, heat=0.0, contract=True, inst=None, scene_depth=None, depth=False, quirks=True,
                 cap=None):
    """A whole depth-ordered frame (steps 1-4).  inst = [(first, count, to_frame12)]; cap truncates the pairs like
    GSR_FLAG_STATIC_CAPACITY.  Returns a dict of every stage, `words` = the sorted depth words, `unsorted_words` = emission order."""
    u = orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8))
    W, H = u.dims[0], u.dims[1]
    pr = project(splat60, vp32, u, v, ortho, inst, cap)
    words = ord_words(view_depth(pr.records, pr.values, vp32))
    k, vals, w = sort_by_depth(pr.keys, pr.values, words)
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
    return dict(rgba=rgba, records=pr.records, keys=k, values=vals, words=w, unsorted_words=words, bounds=b, visible=pr.visible,
                m=pr.duplicates, last_tile=pr.last_tile, staged=staged, depth=dep)


# ---- the emulated kernels ----------------------------------------------------------------------------------------------------
def emu_project(store, bands, vp, ub, bulk_min, num_splats, v=0.0, ortho=False, ranges=None, xf=None, capacity=None):
    """projection_kernel<ranges is not None, bands, ortho, v > 0, true> over `store` (soa_planes(store bands) x stride float4) on the
    CPU.  Returns (records, keys, values, depth words, M, V, last tile, overflow) with the pairs in emission order."""
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
    words = np.zeros(max(cap, 1), dtype=U32)
    vis, last, ovf = C.c_uint(0), C.c_int(-1), C.c_uint(0)
    vp32 = np.ascontiguousarray(vp, dtype=F32)
    ubuf = np.frombuffer(ub, dtype=np.uint8).copy()
    m = emu_lib().emu_depth_projection(int(inst), int(bands), int(bool(ortho)), float(v), store.ctypes.data, stride, n, vp32.ctypes.data,
                                       ubuf.ctypes.data, int(bulk_min), recs.ctypes.data, keys.ctypes.data, vals.ctypes.data, words.ctypes.data,
                                       cap, C.byref(vis), C.byref(last), C.byref(ovf), None if frame_c is None else frame_c.ctypes.data,
                                       None if desc is None else desc.ctypes.data, None if warp_inst is None else warp_inst.ctypes.data)
    assert m >= 0
    mm = min(int(m), cap)
    return recs[:n], keys[:mm].copy(), vals[:mm].copy(), words[:mm].copy(), int(m), int(vis.value), int(last.value), int(ovf.value)


def emu_sort(keys, values, words, n_max=None, hist_grid=3):
    """sort_pairs_depth_device on the CPU: (keys, values) sorted by (key >> 16, word), stable.  (The words themselves are only carried
    by the four wide passes: the library never reads them after the sort.)"""
    n = len(keys)
    n_max = int(n_max if n_max is not None else max(n, 1))
    k = np.zeros(n_max, dtype=U32); k[:n] = keys
    v = np.zeros(n_max, dtype=U32); v[:n] = values
    w = np.zeros(n_max, dtype=U32); w[:n] = words
    assert emu_lib().emu_depth_sort(k.ctypes.data, v.ctypes.data, w.ctypes.data, n, n_max, int(hist_grid)) == 0
    return k[:n].copy(), v[:n].copy()
