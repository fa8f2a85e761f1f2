"""Reference implementations of motion vectors (include/gsr.h gsr_set_motion_vectors) for the tests.

TEST INFRASTRUCTURE.
  * splat_motion -- the per-splat motion m of every record id, in numpy float32 (plain operations only, one rounding each);
  * motion_oracle.c -- the per-pixel accumulation (it needs fmaf), compiled together with tests/depth_reference/depth_oracle.c and
    oracle/gsr_oracle.c, which it extends without changing them;
  * motion_emu.cpp -- composite_kernel<CONTRACT, true, true> compiled for the CPU on top of tests/kernel_emu.
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

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "motion_reference")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "godotgaussiansplatting_b200", "csrc")
CUDA_INC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
F32 = np.float32

_ORACLE_DEPS = [os.path.join(HERE, "motion_oracle.c"), os.path.join(ROOT, "tests", "depth_reference", "depth_oracle.c"),
                os.path.join(ROOT, "oracle", "gsr_oracle.c"), os.path.abspath(__file__)]
_EMU_DEPS = [os.path.join(HERE, "motion_emu.cpp"), os.path.abspath(__file__)] + [
    os.path.join(ROOT, "tests", "kernel_emu", f) for f in ("kernel_emu.cpp", "cuda_shim.h")] + [
    os.path.join(ROOT, "oracle", "glsl_cpu", "glsl_emu.hpp")] + [
    os.path.join(CSRC, f) for f in ("compositor.cu", "ranges.cu", "radix_sort.cu", "projection.cu", "ingest.cu", "present.cu", "group.cu",
                                    "common.cuh")]

_oracle = None
_emu = None


def _out_dir() -> str:
    if os.access(HERE, os.W_OK):
        return HERE
    d = os.path.join(tempfile.gettempdir(), f"gsr_motion_reference_{os.getuid()}")
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
        so = _build("libmotion_oracle.so", _ORACLE_DEPS, lambda out: [cc] + dref._ORC_FLAGS + [_ORACLE_DEPS[0], "-o", out, "-lm"])
        L = C.CDLL(so)
        L.mvo_set_blend_contraction.argtypes = [C.c_int]
        vp = C.c_void_p
        L.mvo_render_motion.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_float, vp, vp, vp, vp, vp, vp, C.POINTER(C.c_int64)]
        _oracle = L
    return _oracle


def emu_lib():
    global _emu
    if _emu is None:
        cxx = os.environ.get("ORC_CXX", "/usr/bin/g++")
        so = _build("libmotion_emu.so", _EMU_DEPS, lambda out: [cxx] + dref._EMU_FLAGS + ["-I", CUDA_INC, _EMU_DEPS[0], "-o", out])
        L = C.CDLL(so)
        vp = C.c_void_p
        L.emu_composite_motion.restype = C.c_int
        L.emu_composite_motion.argtypes = [C.c_int, vp, vp, vp, vp, vp, vp, vp, vp, vp, C.c_int, C.c_int, C.c_float, vp, vp, vp, vp,
                                           C.c_float, C.POINTER(C.c_ulonglong)]
        _emu = L
    return _emu


# ---- the per-splat motion ---------------------------------------------------------------------------------------------------
def pix(M32, q0, q1, q2, width, height):
    """pix(M, q) of include/gsr.h: the projection's image_pos operations without the load-in term.  Returns (x, y, clip3)."""
    M = np.asarray(M32, dtype=F32).reshape(32)
    V, P = M[:16], M[16:]
    view = [((V[r] * q0 + V[4 + r] * q1) + V[8 + r] * q2) + V[12 + r] * F32(1.0) for r in range(4)]
    clip = {r: ((P[r] * view[0] + P[4 + r] * view[1]) + P[8 + r] * view[2]) + P[12 + r] * view[3] for r in (0, 1, 3)}
    with np.errstate(all="ignore"):
        x = ((clip[0] / clip[3] + F32(1.0)) * F32(0.5)) * F32(width - 1)
        y = ((clip[1] / clip[3] + F32(1.0)) * F32(0.5)) * F32(height - 1)
    return x.astype(F32), y.astype(F32), clip[3].astype(F32)


def splat_motion(records, vp32, prev_vp32, width, height, prev_pos=None):
    """m of every record id, (N, 2) float32: pix(M', p') - pix(M, p), (0, 0) unless clip3' > 0 and both components are finite.
    prev_pos: (N, 3) float32 p' (None: p' = p)."""
    p0 = np.ascontiguousarray(records["pos_xy"][:, 0], dtype=F32)
    p1 = np.ascontiguousarray(records["pos_xy"][:, 1], dtype=F32)
    p2 = np.ascontiguousarray(records["pos_z"], dtype=F32)
    if prev_pos is None:
        q0, q1, q2 = p0, p1, p2
    else:
        q0, q1, q2 = (np.ascontiguousarray(prev_pos[:, i], dtype=F32) for i in range(3))
    x, y, _ = pix(vp32, p0, p1, p2, width, height)
    xp, yp, wp = pix(prev_vp32, q0, q1, q2, width, height)
    with np.errstate(all="ignore"):
        mx, my = (xp - x).astype(F32), (yp - y).astype(F32)
    ok = (wp > 0) & np.isfinite(mx) & np.isfinite(my)
    m = np.zeros((len(p0), 2), dtype=F32)
    m[ok, 0], m[ok, 1] = mx[ok], my[ok]
    return m


def instance_prev_positions(splat60, ranges, prev_to_frame, model_scale, drawn):
    """p' of every drawn id of an instance layout: A'_k * (plane 0 of source splat s) * model_scale, float32, the record's operations.
    prev_to_frame: (n, 12) previous [A | t] per instance."""
    s = np.ascontiguousarray(splat60, dtype=F32).reshape(-1, 60)
    w0, _ = iref.layout(ranges)
    out = np.zeros((max(drawn, 1), 3), dtype=F32)
    ms = F32(model_scale)
    for k, (first, count) in enumerate(ranges):
        first, count = int(first), int(count)
        if count == 0:
            continue
        sp = s[first:first + count, 0:3] * ms
        xf = np.concatenate([np.asarray(prev_to_frame[k], dtype=F32).reshape(12), np.zeros(12, dtype=F32)])
        out[32 * w0[k]:32 * w0[k] + count] = iref.frame_position(xf, sp)
    return out[:drawn]


# ---- the per-pixel oracle and the emulated kernel ---------------------------------------------------------------------------
def render_motion(records, sorted_values, bounds, width, height, vp32, motion, scene_depth=None, heatmap=0.0, contract=True):
    """The oracle on the full frame.  motion: (N, 2) float32 per record id (splat_motion).  Returns (rgba, depth, motion[H, W, 2], staged)."""
    recs = np.ascontiguousarray(records)
    assert recs.dtype == orc.RECORD_DTYPE
    v = np.ascontiguousarray(sorted_values, dtype=np.uint32)
    if v.size == 0:
        v = np.zeros(1, dtype=np.uint32)
    b = np.ascontiguousarray(bounds, dtype=np.uint32)
    vp = np.ascontiguousarray(vp32, dtype=F32).reshape(32)
    m = np.ascontiguousarray(motion, dtype=F32)
    z = dref._scene_depth(scene_depth, width, height)
    out = np.zeros((height, width, 4), dtype=F32)
    depth = np.zeros((height, width), dtype=F32)
    mo = np.zeros((height, width, 2), dtype=F32)
    staged = C.c_int64(0)
    L = oracle_lib()
    L.mvo_set_blend_contraction(int(bool(contract)))
    try:
        L.mvo_render_motion(recs.ctypes.data, v.ctypes.data, b.ctypes.data, int(width), int(height), float(heatmap), vp.ctypes.data,
                            None if z is None else z.ctypes.data, m.ctypes.data, out.ctypes.data, depth.ctypes.data, mo.ctypes.data,
                            C.byref(staged))
    finally:
        L.mvo_set_blend_contraction(1)
    return out, depth, mo, int(staged.value)


def emu_composite_motion(variant, records, values, bounds, width, height, vp32, prev_vp32, scene_depth=None, heatmap=0.0,
                         instances=None):
    """composite_kernel<variant == 0, true, true> on the CPU emulator.  instances: None, or (splat60, max_splats, ranges, prev_to_frame
    (n, 12), model_scale).  Returns (rgba, depth, motion, staged)."""
    out = np.zeros((height, width, 4), dtype=F32)
    depth = np.zeros((height, width), dtype=F32)
    mo = np.full((height, width, 2), np.nan, dtype=F32)
    vals = np.concatenate([np.asarray(values, dtype=np.uint32), np.zeros(512, dtype=np.uint32)])
    recs, bnds = np.ascontiguousarray(records), np.ascontiguousarray(bounds, dtype=np.uint32)
    vp = np.ascontiguousarray(vp32, dtype=F32).reshape(32)
    pvp = np.ascontiguousarray(prev_vp32, dtype=F32).reshape(32)
    z = dref._scene_depth(scene_depth, width, height)
    keep = []
    wi = desc = pxf = plane0 = None
    ms = 1.0
    if instances is not None:
        splat60, max_splats, ranges, prev_xf, ms = instances
        soa, _ = iref.soa_planes(splat60, max_splats)
        plane0 = np.ascontiguousarray(soa[0])
        w0, D = iref.layout(ranges)
        warps = np.full(D // 32 + 8, 0xFFFFFFFF, dtype=np.uint32)
        d = np.zeros(len(ranges), dtype=[("first", "<u8"), ("count", "<u4"), ("warp0", "<u4")])
        for k, (first, count) in enumerate(ranges):
            nw = (int(count) + 31) // 32
            warps[w0[k]:w0[k] + nw] = k
            d[k] = (int(first), int(count), w0[k])
        pxf = np.ascontiguousarray(prev_xf, dtype=F32).reshape(-1, 12)
        keep = [plane0, warps, d, pxf]
        wi, desc = warps, d
    staged = C.c_ulonglong(0)
    ptr = lambda a: None if a is None else a.ctypes.data
    rc = emu_lib().emu_composite_motion(int(variant), recs.ctypes.data, vals.ctypes.data, bnds.ctypes.data, out.ctypes.data,
                                        depth.ctypes.data, mo.ctypes.data, ptr(z), vp.ctypes.data, pvp.ctypes.data, int(width), int(height),
                                        float(heatmap), ptr(wi), ptr(desc), ptr(pxf), ptr(plane0), float(ms), C.byref(staged))
    del keep
    assert rc == 0, "not every tile was rendered"
    return out, depth, mo, int(staged.value)
