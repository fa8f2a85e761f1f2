"""Reference implementations of splat IDs (include/gsr.h gsr_set_splat_ids) for the tests.

TEST INFRASTRUCTURE.
  * id_oracle.c -- the per-pixel (best, id) walk added to the depth-compositing blend, compiled together with
    tests/depth_reference/depth_oracle.c and oracle/gsr_oracle.c, which it extends without changing them;
  * warp_instances / with_instances -- k = the instance of the drawn warp v >> 5 of an instance layout;
  * sources -- the source splat of every drawn id (the rule GaussianSplattingRasterizer.splat_sources follows);
  * id_emu.cpp -- composite_ids_kernel<CONTRACT, MOTION> compiled for the CPU on top of tests/kernel_emu.
The libraries are written next to their sources, or to a temporary directory when the tree is read-only.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from oracle import oracle as orc
from tests import depth_reference as dref
from tests import instance_reference as iref

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "id_reference")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "godotgaussiansplatting_b200", "csrc")
CUDA_INC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
F32, U32 = np.float32, np.uint32
NO_ID = 0xFFFFFFFF

_ORACLE_DEPS = [os.path.join(HERE, "id_oracle.c"), os.path.join(ROOT, "tests", "depth_reference", "depth_oracle.c"),
                os.path.join(ROOT, "oracle", "gsr_oracle.c"), os.path.abspath(__file__)]
_EMU_DEPS = [os.path.join(HERE, "id_emu.cpp"), os.path.abspath(__file__)] + [
    os.path.join(ROOT, "tests", "kernel_emu", f) for f in ("kernel_emu.cpp", "cuda_shim.h")] + [
    os.path.join(ROOT, "oracle", "glsl_cpu", "glsl_emu.hpp")] + [
    os.path.join(CSRC, f) for f in ("compositor.cu", "ranges.cu", "radix_sort.cu", "projection.cu", "ingest.cu", "present.cu", "group.cu",
                                    "common.cuh")]

_oracle = None
_emu = None


def _out_dir() -> str:
    if os.access(HERE, os.W_OK):
        return HERE
    d = os.path.join(tempfile.gettempdir(), f"gsr_id_reference_{os.getuid()}")
    os.makedirs(d, exist_ok=True)
    return d


def _build(name: str, deps: list[str], cmd) -> str:
    out = os.path.join(_out_dir(), name)
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(d) for d in deps):
        subprocess.run(cmd(out), check=True)
    return out


def oracle_lib():
    global _oracle
    if _oracle is None:
        cc = os.environ.get("ORC_CC", "/usr/bin/gcc")
        so = _build("libid_oracle.so", _ORACLE_DEPS, lambda out: [cc] + dref._ORC_FLAGS + [_ORACLE_DEPS[0], "-o", out, "-lm"])
        L = C.CDLL(so)
        L.ido_set_blend_contraction.argtypes = [C.c_int]
        vp = C.c_void_p
        L.ido_render_ids.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_float, vp, vp, vp, vp, vp, C.POINTER(C.c_int64)]
        _oracle = L
    return _oracle


def emu_lib():
    global _emu
    if _emu is None:
        cxx = os.environ.get("ORC_CXX", "/usr/bin/g++")
        so = _build("libid_emu.so", _EMU_DEPS, lambda out: [cxx] + dref._EMU_FLAGS + ["-I", CUDA_INC, _EMU_DEPS[0], "-o", out])
        L = C.CDLL(so)
        vp = C.c_void_p
        L.emu_composite_ids.restype = C.c_int
        L.emu_composite_ids.argtypes = [C.c_int, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, C.c_int, C.c_int, C.c_float, vp, vp, vp,
                                        vp, C.c_float, C.POINTER(C.c_ulonglong)]
        _emu = L
    return _emu


# ---- instances -----------------------------------------------------------------------------------------------------------------
def warp_instances(ranges):
    """The instance of every drawn warp of an instance layout (NO_ID past the last one), as the library's warp table."""
    w0, D = iref.layout(ranges)
    warps = np.full(D // 32 + 8, NO_ID, dtype=U32)
    for k, (_, count) in enumerate(ranges):
        warps[w0[k]:w0[k] + (int(count) + 31) // 32] = k
    return warps


def with_instances(v, ranges=None):
    """(H, W) drawn ids -> (H, W, 2) (v, k): k = the instance of warp v >> 5, NO_ID without instances and where v is NO_ID."""
    v = np.asarray(v, dtype=U32)
    k = np.full(v.shape, NO_ID, dtype=U32)
    if ranges is not None:
        hit = v != NO_ID
        k[hit] = warp_instances(ranges)[v[hit] >> 5]
    return np.stack([v, k], axis=-1)


def sources(ids, ranges=None):
    """The source splat of every pixel of an (H, W, 2) ID array: first_k + (v - 32 w_k), or v without instances; NO_ID stays NO_ID."""
    ids = np.asarray(ids, dtype=U32)
    v, k = ids[..., 0].astype(np.int64), ids[..., 1]
    out = np.full(v.shape, NO_ID, dtype=np.int64)
    hit = ids[..., 0] != NO_ID
    if ranges is None:
        out[hit] = v[hit]
        return out
    w0, _ = iref.layout(ranges)
    first = np.array([int(f) for f, _ in ranges], dtype=np.int64)
    base = np.array(w0, dtype=np.int64) * 32
    kk = k[hit].astype(np.int64)
    out[hit] = first[kk] + (v[hit] - base[kk])
    return out


# ---- the per-pixel oracle and the emulated kernel ------------------------------------------------------------------------------
def render_ids(records, sorted_values, bounds, width, height, vp32, scene_depth=None, heatmap=0.0, contract=True, ranges=None):
    """The oracle on the full frame.  ranges: the instance layout ((first, count) per instance) or None.
    Returns (rgba, depth, ids[H, W, 2] uint32, staged)."""
    recs = np.ascontiguousarray(records)
    assert recs.dtype == orc.RECORD_DTYPE
    v = np.ascontiguousarray(sorted_values, dtype=U32)
    if v.size == 0:
        v = np.zeros(1, dtype=U32)
    b = np.ascontiguousarray(bounds, dtype=U32)
    vp = np.ascontiguousarray(vp32, dtype=F32).reshape(32)
    z = dref._scene_depth(scene_depth, width, height)
    out = np.zeros((height, width, 4), dtype=F32)
    depth = np.zeros((height, width), dtype=F32)
    ids = np.zeros((height, width), dtype=U32)
    staged = C.c_int64(0)
    L = oracle_lib()
    L.ido_set_blend_contraction(int(bool(contract)))
    try:
        L.ido_render_ids(recs.ctypes.data, v.ctypes.data, b.ctypes.data, int(width), int(height), float(heatmap), vp.ctypes.data,
                         None if z is None else z.ctypes.data, out.ctypes.data, depth.ctypes.data, ids.ctypes.data, C.byref(staged))
    finally:
        L.ido_set_blend_contraction(1)
    return out, depth, with_instances(ids, ranges), int(staged.value)


def emu_composite_ids(variant, records, values, bounds, width, height, vp32, scene_depth=None, heatmap=0.0, ranges=None, motion=None):
    """composite_ids_kernel<variant == 0, motion is not None> on the CPU emulator.  ranges: the instance layout or None.
    motion: None, or (prev_vp32, instances) with instances as in tests/motion_reference.emu_composite_motion.
    Returns (rgba, depth, motion or None, ids, staged)."""
    out = np.zeros((height, width, 4), dtype=F32)
    depth = np.zeros((height, width), dtype=F32)
    mo = np.full((height, width, 2), np.nan, dtype=F32)
    ids = np.full((height, width, 2), 0xDEADBEEF, dtype=U32)
    vals = np.concatenate([np.asarray(values, dtype=U32), np.zeros(512, dtype=U32)])
    recs, bnds = np.ascontiguousarray(records), np.ascontiguousarray(bounds, dtype=U32)
    vp = np.ascontiguousarray(vp32, dtype=F32).reshape(32)
    z = dref._scene_depth(scene_depth, width, height)
    wi = None if ranges is None else warp_instances(ranges)
    pvp = desc = pxf = plane0 = None
    ms = 1.0
    if motion is not None:
        pvp = np.ascontiguousarray(motion[0], dtype=F32).reshape(32)
        assert (motion[1] is None) == (ranges is None), "the motion and ID variants share the warp table"
        if motion[1] is not None:
            splat60, max_splats, mranges, prev_xf, ms = motion[1]
            assert ranges is not None and [tuple(map(int, r)) for r in mranges] == [tuple(map(int, r)) for r in ranges]
            soa, _ = iref.soa_planes(splat60, max_splats)
            plane0 = np.ascontiguousarray(soa[0])
            w0, _ = iref.layout(ranges)
            desc = np.zeros(len(ranges), dtype=[("first", "<u8"), ("count", "<u4"), ("warp0", "<u4")])
            for k, (first, count) in enumerate(ranges):
                desc[k] = (int(first), int(count), w0[k])
            pxf = np.ascontiguousarray(prev_xf, dtype=F32).reshape(-1, 12)
    staged = C.c_ulonglong(0)
    ptr = lambda a: None if a is None else a.ctypes.data
    rc = emu_lib().emu_composite_ids(int(variant), int(motion is not None), recs.ctypes.data, vals.ctypes.data, bnds.ctypes.data,
                                     out.ctypes.data, depth.ctypes.data, mo.ctypes.data, ids.ctypes.data, ptr(z), vp.ctypes.data, ptr(pvp),
                                     int(width), int(height), float(heatmap), ptr(wi), ptr(desc), ptr(pxf), ptr(plane0), float(ms),
                                     C.byref(staged))
    assert rc == 0, "not every tile was rendered"
    return out, depth, (mo if motion is not None else None), ids, int(staged.value)
