"""Reference implementation of splat instances (include/gsr.h gsr_set_instances) for the tests.

TEST INFRASTRUCTURE.  The instance oracle is built from the unchanged oracle/ (one projection per instance with that instance's
composed view matrix and camera position, then the default sort, tile ranges and compositor), plus:
  * instance_emu.cpp -- instance_prepare_kernel + projection_kernel<true> compiled for the CPU on top of tests/kernel_emu, built on
    first use next to its source, or in a temporary directory when the tree is read-only.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile
from dataclasses import dataclass

import numpy as np

from oracle import oracle as orc
from tests import depth_reference as dref

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "instance_reference")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "godotgaussiansplatting_b200", "csrc")
CUDA_INC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")

_EMU_DEPS = [os.path.join(HERE, "instance_emu.cpp"), os.path.abspath(__file__)] + [
    os.path.join(ROOT, "tests", "kernel_emu", f) for f in ("kernel_emu.cpp", "cuda_shim.h")] + [
    os.path.join(ROOT, "oracle", "glsl_cpu", "glsl_emu.hpp")] + [
    os.path.join(CSRC, f) for f in ("compositor.cu", "ranges.cu", "radix_sort.cu", "projection.cu", "ingest.cu", "present.cu", "group.cu",
                                    "common.cuh")]
_EMU_FLAGS = ["-std=gnu++17", "-O1", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-w"]
_emu = None

F32 = np.float32


def _out_dir() -> str:
    if os.access(HERE, os.W_OK):
        return HERE
    d = os.path.join(tempfile.gettempdir(), f"gsr_instance_reference_{os.getuid()}")
    os.makedirs(d, exist_ok=True)
    return d


def emu_lib():
    global _emu
    if _emu is None:
        out = os.path.join(_out_dir(), "libinstance_emu.so")
        if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(d) for d in _EMU_DEPS):
            cxx = os.environ.get("ORC_CXX", "/usr/bin/g++")
            subprocess.run([cxx] + _EMU_FLAGS + ["-I", CUDA_INC, _EMU_DEPS[0], "-o", out], check=True)
        L = C.CDLL(out)
        L.emu_projection_instanced.restype = C.c_longlong
        L.emu_projection_instanced.argtypes = [C.c_void_p, C.c_ulonglong, C.c_void_p, C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p,
                                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint, C.POINTER(C.c_uint), C.POINTER(C.c_int),
                                               C.POINTER(C.c_uint), C.c_void_p]
        _emu = L
    return _emu


# ---- transforms ------------------------------------------------------------------------------------------------------------
def inverse(to_frame12) -> np.ndarray:
    """[A | t] (12 floats, column-major) -> the 24 floats of GSR_BUF_INSTANCES: A|t, then [A^-1 | -A^-1 t] in float64 rounded to float."""
    m = np.asarray(to_frame12, dtype=np.float32).reshape(12)
    A = m[:9].astype(np.float64).reshape(3, 3).T      # matrix form: column c = a_c
    t = m[9:].astype(np.float64)
    B = np.linalg.inv(A)
    u = -(B @ t)
    return np.concatenate([m, B.T.reshape(9).astype(F32), u.astype(F32)]).astype(F32)


def compose(V16, cam3, xf24):
    """The per-frame constants of one instance (include/gsr.h; instance_prepare_kernel): V_k (16) and cam_k (3), float32, one
    rounding per operation, structurally zero terms skipped."""
    V = np.asarray(V16, dtype=F32).reshape(16)
    x = np.asarray(xf24, dtype=F32).reshape(24)
    A = [x[3 * c:3 * c + 3] for c in range(3)]
    t, B, u = x[9:12], [x[12 + 3 * c:15 + 3 * c] for c in range(3)], x[21:24]
    cam = np.asarray(cam3, dtype=F32).reshape(3)
    Vk = np.zeros(16, dtype=F32)
    for c in range(3):
        for r in range(4):
            Vk[4 * c + r] = (V[r] * A[c][0] + V[4 + r] * A[c][1]) + V[8 + r] * A[c][2]
    for r in range(4):
        Vk[12 + r] = ((V[r] * t[0] + V[4 + r] * t[1]) + V[8 + r] * t[2]) + V[12 + r]
    camk = np.array([((B[0][r] * cam[0] + B[1][r] * cam[1]) + B[2][r] * cam[2]) + u[r] for r in range(3)], dtype=F32)
    return Vk, camk


def frame_position(xf24, sp):
    """w[r] = ((A[0][r] sp0 + A[1][r] sp1) + A[2][r] sp2) + t[r] for an (n, 3) float32 array sp."""
    x = np.asarray(xf24, dtype=F32).reshape(24)
    sp = np.asarray(sp, dtype=F32)
    return np.stack([((x[r] * sp[:, 0] + x[3 + r] * sp[:, 1]) + x[6 + r] * sp[:, 2]) + x[9 + r] for r in range(3)], axis=1).astype(F32)


def layout(ranges):
    """First drawn warp of every instance and D."""
    w0, w = [], 0
    for _, count in ranges:
        w0.append(w)
        w += (int(count) + 31) // 32
    return w0, 32 * w


# ---- the oracle ------------------------------------------------------------------------------------------------------------
@dataclass
class InstanceProjection:
    records: np.ndarray   # (D,) RECORD_DTYPE at drawn ids (ids that emitted nothing are zero)
    keys: np.ndarray      # emission order
    values: np.ndarray
    visible: int
    duplicates: int
    last_tile: int
    drawn: int


def project(splat60, vp32, uniforms, ranges, xf):
    """Steps 1-3 of the instance oracle: compose, project each range with orc.project, move values and records to drawn ids
    (records with frame-space positions); pairs concatenated in instance order.  xf: (n, 24) float32 (GSR_BUF_INSTANCES)."""
    splat60 = np.ascontiguousarray(splat60, dtype=F32).reshape(-1, 60)
    vp32 = np.asarray(vp32, dtype=F32).reshape(32)
    w0, D = layout(ranges)
    recs = np.zeros(D, dtype=orc.RECORD_DTYPE)
    keys, vals = [], []
    vis, m, last = 0, 0, -1
    for k, (first, count) in enumerate(ranges):
        first, count = int(first), int(count)
        if count == 0:
            continue
        Vk, camk = compose(vp32[:16], uniforms.camera_pos[:], xf[k])
        u = orc.make_uniforms(camk, uniforms.model_scale, uniforms.dims[0], uniforms.dims[1], uniforms.time)
        u.camera_pos[:] = [float(c) for c in camk]
        pr = orc.project(splat60[first:first + count], np.concatenate([Vk, vp32[16:]]), u, cap=64 * count + 1024)
        assert pr.duplicates <= 64 * count + 1024
        emitted = np.unique(pr.values)
        r = pr.records[emitted].copy()
        sp = np.stack([r["pos_xy"][:, 0], r["pos_xy"][:, 1], r["pos_z"]], axis=1)
        w = frame_position(xf[k], sp)
        r["pos_xy"] = w[:, :2]
        r["pos_z"] = w[:, 2]
        recs[32 * w0[k] + emitted] = r
        keys.append(pr.keys)
        vals.append(pr.values.astype(np.uint32) + np.uint32(32 * w0[k]))
        vis += pr.visible
        m += pr.duplicates
        last = max(last, pr.last_tile)
    cat = lambda xs: np.concatenate(xs).astype(np.uint32) if xs else np.zeros(0, dtype=np.uint32)
    return InstanceProjection(recs, cat(keys), cat(vals), vis, m, last, D)


@dataclass
class InstanceFrame:
    rgba: np.ndarray
    proj: InstanceProjection
    keys: np.ndarray      # sorted
    values: np.ndarray
    bounds: np.ndarray
    staged: int
    depth: np.ndarray | None = None


def frame(splat60, vp32, uniforms, ranges, xf, heatmap=0.0, quirks=True, scene_depth=None, depth=False, contract=True):
    """The instance oracle's whole frame (step 4: sort, tile ranges, compositor or the depth-compositing oracle)."""
    pr = project(splat60, vp32, uniforms, ranges, xf)
    W, H = uniforms.dims[0], uniforms.dims[1]
    T = ((W + 15) // 16) * ((H + 15) // 16)
    k, v = orc.sort_pairs(pr.keys, pr.values)
    b = orc.boundaries(k, T, quirks=quirks)
    if depth or scene_depth is not None:
        rgba, dep, staged = dref.render_depth(pr.records, v, b, W, H, vp32, scene_depth, heatmap, contract)
        return InstanceFrame(rgba, pr, k, v, b, staged, dep)
    orc.set_blend_contraction(contract)
    try:
        rgba, staged, _ = orc.render(pr.records, v, b, W, H, heatmap)
    finally:
        orc.set_blend_contraction(True)
    return InstanceFrame(rgba, pr, k, v, b, staged)


# ---- the emulated kernels --------------------------------------------------------------------------------------------------
def soa_planes(splat60, max_splats):
    """The library's SoA layout: 15 planes of plane_stride float4 (max_splats rounded up to 256), zero beyond the uploaded splats."""
    s = np.ascontiguousarray(splat60, dtype=F32).reshape(-1, 60)
    stride = (int(max_splats) + 255) & ~255
    soa = np.zeros((15, stride, 4), dtype=F32)
    soa[:, :s.shape[0], :] = s.reshape(-1, 15, 4).transpose(1, 0, 2)
    return soa, stride


def emu_project(splat60, max_splats, vp32, uniforms_bytes, ranges, xf, capacity=None):
    """instance_prepare_kernel + projection_kernel<true> on the CPU.  Returns (InstanceProjection with keys/values in emission order,
    the (n, 32) constants the prepare kernel wrote, overflow)."""
    soa, stride = soa_planes(splat60, max_splats)
    n = len(ranges)
    _, D = layout(ranges)
    cap = int(capacity if capacity is not None else 64 * max(D, 1))
    rng = np.array([[int(f), int(c)] for f, c in ranges], dtype=np.uint64).reshape(-1)
    x = np.ascontiguousarray(xf, dtype=F32).reshape(-1)
    recs = np.zeros(max(D, 1), dtype=orc.RECORD_DTYPE)
    keys = np.zeros(max(cap, 1), dtype=np.uint32)
    vals = np.zeros(max(cap, 1), dtype=np.uint32)
    consts = np.zeros((max(n, 1), 32), dtype=F32)
    vp = np.ascontiguousarray(vp32, dtype=F32).reshape(32)
    ub = np.frombuffer(bytes(uniforms_bytes), dtype=np.uint8).copy()
    vis, last, ovf = C.c_uint(0), C.c_int(-1), C.c_uint(0)
    m = emu_lib().emu_projection_instanced(soa.ctypes.data, stride, vp.ctypes.data, ub.ctypes.data, n, x.ctypes.data if n else None,
                                           rng.ctypes.data if n else None, recs.ctypes.data, keys.ctypes.data, vals.ctypes.data, cap,
                                           C.byref(vis), C.byref(last), C.byref(ovf), consts.ctypes.data)
    assert m >= 0
    mm = min(int(m), cap)
    return InstanceProjection(recs[:D], keys[:mm].copy(), vals[:mm].copy(), int(vis.value), int(m), int(last.value), D), consts[:n], bool(ovf.value)
