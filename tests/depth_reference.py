"""Reference implementations of depth compositing (include/gsr.h gsr_set_depth_compositing) for the tests.

TEST INFRASTRUCTURE.  Two small shared libraries, built on first use from tests/depth_reference/:
  * depth_oracle.c -- the CPU oracle of the mode, compiled together with oracle/gsr_oracle.c (same exp, records and contraction
    switch as the oracle's default frame);
  * depth_emu.cpp  -- composite_kernel<CONTRACT, true> compiled for the CPU on top of tests/kernel_emu.
They are written next to their sources, or to a temporary directory when the tree is read-only.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from oracle import oracle as orc

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "depth_reference")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "godotgaussiansplatting_b200", "csrc")
CUDA_INC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")

_ORACLE_DEPS = [os.path.join(HERE, "depth_oracle.c"), os.path.join(ROOT, "oracle", "gsr_oracle.c"), os.path.abspath(__file__)]
_EMU_DEPS = [os.path.join(HERE, "depth_emu.cpp"), os.path.abspath(__file__)] + [
    os.path.join(ROOT, "tests", "kernel_emu", f) for f in ("kernel_emu.cpp", "cuda_shim.h")] + [
    os.path.join(ROOT, "oracle", "glsl_cpu", "glsl_emu.hpp")] + [
    os.path.join(CSRC, f) for f in ("compositor.cu", "ranges.cu", "radix_sort.cu", "projection.cu", "ingest.cu", "present.cu", "group.cu",
                                    "common.cuh")]


def _out_dir() -> str:
    if os.access(HERE, os.W_OK):
        return HERE
    d = os.path.join(tempfile.gettempdir(), f"gsr_depth_reference_{os.getuid()}")
    os.makedirs(d, exist_ok=True)
    return d


def _build(name: str, deps: list[str], cmd) -> str:
    out = os.path.join(_out_dir(), name)
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(d) for d in deps):
        subprocess.run(cmd(out), check=True)
    return out


# the oracle's build flags (oracle/Makefile): no implicit contraction, fmaf() only where the source writes it
_ORC_FLAGS = ["-O3", "-march=x86-64-v3", "-mfma", "-ffp-contract=off", "-fno-fast-math", "-fopenmp", "-fPIC", "-std=gnu11", "-shared"]
# the kernel emulator's build flags (tests/kernel_emu/build.py)
_EMU_FLAGS = ["-std=gnu++17", "-O1", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-w"]

_oracle = None
_emu = None


def oracle_lib():
    global _oracle
    if _oracle is None:
        cc = os.environ.get("ORC_CC", "/usr/bin/gcc")
        so = _build("libdepth_oracle.so", _ORACLE_DEPS, lambda out: [cc] + _ORC_FLAGS + [_ORACLE_DEPS[0], "-o", out, "-lm"])
        L = C.CDLL(so)
        fp = C.POINTER(C.c_float)
        L.dco_set_blend_contraction.argtypes = [C.c_int]
        L.dco_render_depth.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, fp, C.c_void_p, fp, fp,
                                       C.POINTER(C.c_int64)]
        _oracle = L
    return _oracle


def emu_lib():
    global _emu
    if _emu is None:
        cxx = os.environ.get("ORC_CXX", "/usr/bin/g++")
        so = _build("libdepth_emu.so", _EMU_DEPS, lambda out: [cxx] + _EMU_FLAGS + ["-I", CUDA_INC, _EMU_DEPS[0], "-o", out])
        L = C.CDLL(so)
        L.emu_composite_depth.restype = C.c_int
        L.emu_composite_depth.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_int, C.c_int, C.c_float, C.POINTER(C.c_ulonglong)]
        _emu = L
    return _emu


def _f(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _scene_depth(scene_depth, width, height):
    if scene_depth is None:
        return None
    z = np.ascontiguousarray(scene_depth, dtype=np.float32)
    assert z.shape == (height, width), z.shape
    return z


def render_depth(records, sorted_values, bounds, width, height, vp32, scene_depth=None, heatmap=0.0, contract=True):
    """The oracle of the mode on the full frame.  vp32: the 32-float view_proj whose view row gives each splat's view depth;
    scene_depth: None (nothing occludes) or (H, W) float32 linear depth.  contract: the gsr spec (True) or the uncontracted blend.
    Returns (rgba[H,W,4] float32 with premultiplied rgb and alpha = coverage, depth[H,W] float32, staged C)."""
    recs = np.ascontiguousarray(records)
    assert recs.dtype == orc.RECORD_DTYPE
    v = np.ascontiguousarray(sorted_values, dtype=np.uint32)
    if v.size == 0:
        v = np.zeros(1, dtype=np.uint32)
    b = np.ascontiguousarray(bounds, dtype=np.uint32)
    vp = np.ascontiguousarray(vp32, dtype=np.float32).reshape(32)
    z = _scene_depth(scene_depth, width, height)
    out = np.zeros((height, width, 4), dtype=np.float32)
    depth = np.zeros((height, width), dtype=np.float32)
    staged = C.c_int64(0)
    L = oracle_lib()
    L.dco_set_blend_contraction(int(bool(contract)))
    try:
        L.dco_render_depth(recs.ctypes.data, v.ctypes.data, b.ctypes.data, int(width), int(height), float(heatmap), _f(vp),
                           None if z is None else z.ctypes.data, _f(out), _f(depth), C.byref(staged))
    finally:
        L.dco_set_blend_contraction(1)
    return out, depth, int(staged.value)


def frame_depth(splat60, vp32, uniforms, heatmap=0.0, quirks=True, cap=None, scene_depth=None, contract=True):
    """oracle.frame (projection, sort, tile ranges) with the tile lists rendered by render_depth: the returned Frame's rgba and staged
    are the mode's, and it gains `depth`."""
    fr = orc.frame(splat60, vp32, uniforms, heatmap=heatmap, quirks=quirks, cap=cap)
    assert not fr.overflow, "the depth oracle renders frames that fit their capacity"
    W, H = uniforms.dims[0], uniforms.dims[1]
    fr.rgba, fr.depth, fr.staged = render_depth(fr.records, fr.values, fr.bounds, W, H, vp32, scene_depth, heatmap, contract)
    return fr


def emu_composite_depth(variant, records, values, bounds, width, height, vp32, scene_depth=None, heatmap=0.0):
    """composite_kernel<variant == 0, true> on the CPU emulator (one persistent block, natural order).  Returns (rgba, depth, staged)."""
    out = np.zeros((height, width, 4), dtype=np.float32)
    depth = np.zeros((height, width), dtype=np.float32)
    vals = np.concatenate([np.asarray(values, dtype=np.uint32), np.zeros(512, dtype=np.uint32)])   # the kernels never read past a range
    recs, bnds = np.ascontiguousarray(records), np.ascontiguousarray(bounds, dtype=np.uint32)
    vp = np.ascontiguousarray(vp32, dtype=np.float32).reshape(32)
    z = _scene_depth(scene_depth, width, height)
    staged = C.c_ulonglong(0)
    rc = emu_lib().emu_composite_depth(int(variant), recs.ctypes.data, vals.ctypes.data, bnds.ctypes.data, out.ctypes.data, depth.ctypes.data,
                                       None if z is None else z.ctypes.data, vp.ctypes.data, int(width), int(height), float(heatmap),
                                       C.byref(staged))
    assert rc == 0, "not every tile was rendered"
    return out, depth, int(staged.value)
