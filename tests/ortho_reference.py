"""Reference implementations of orthographic frames (include/gsr.h GSR_FLAG_ORTHOGRAPHIC) for the tests.

TEST INFRASTRUCTURE.  Two small shared libraries, built on first use from tests/ortho_reference/:
  * ortho_oracle.c -- the orthographic projection of the CPU oracle (project_one with the orthographic cull, Jacobian, view direction
    and depth key), compiled together with oracle/gsr_oracle.c, plus a frame on the oracle's own sort, tile ranges and compositor;
  * ortho_emu.cpp  -- projection_kernel<INSTANCED, B, true> compiled for the CPU on top of tests/kernel_emu.
Instances compose like tests/instance_reference.py: instance k is the orthographic projection with view matrix V_k = V * M_k.
They are written next to their sources, or to a temporary directory when the tree is read-only.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from godotgaussiansplatting_b200 import camera as cam
from oracle import oracle as orc
from tests import depth_reference as dref
from tests import instance_reference as iref
from tests.scenes import uniforms_bytes

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ortho_reference")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "godotgaussiansplatting_b200", "csrc")
CUDA_INC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")

_ORACLE_DEPS = [os.path.join(HERE, "ortho_oracle.c"), os.path.join(ROOT, "oracle", "gsr_oracle.c"), os.path.abspath(__file__)]
_EMU_DEPS = [os.path.join(HERE, "ortho_emu.cpp"), os.path.abspath(__file__), os.path.join(ROOT, "include", "gsr.h")] + [
    os.path.join(ROOT, "tests", "kernel_emu", f) for f in ("kernel_emu.cpp", "cuda_shim.h")] + [
    os.path.join(ROOT, "oracle", "glsl_cpu", "glsl_emu.hpp")] + [
    os.path.join(CSRC, f) for f in ("compositor.cu", "ranges.cu", "radix_sort.cu", "projection.cu", "ingest.cu", "present.cu", "group.cu",
                                    "common.cuh")]
# the oracle's build flags (oracle/Makefile) and the kernel emulator's (tests/kernel_emu/build.py)
_ORC_FLAGS = ["-O3", "-march=x86-64-v3", "-mfma", "-ffp-contract=off", "-fno-fast-math", "-fopenmp", "-fPIC", "-std=gnu11", "-shared"]
_EMU_FLAGS = ["-std=gnu++17", "-O1", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-w"]

F32 = np.float32
_oracle = None
_emu = None


def _out_dir() -> str:
    if os.access(HERE, os.W_OK):
        return HERE
    d = os.path.join(tempfile.gettempdir(), f"gsr_ortho_reference_{os.getuid()}")
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
        L = C.CDLL(_build("libortho_oracle.so", _ORACLE_DEPS, lambda out: [cc] + _ORC_FLAGS + [_ORACLE_DEPS[0], "-o", out, "-lm"]))
        fp, u32p, i64 = C.POINTER(C.c_float), C.POINTER(C.c_uint32), C.c_int64
        L.oro_project.restype = i64
        L.oro_project.argtypes = [fp, i64, fp, C.POINTER(orc._Uniforms), C.c_void_p, u32p, u32p, i64, C.POINTER(i64), C.POINTER(i64)]
        L.oro_frame.restype = C.c_int
        L.oro_frame.argtypes = [fp, i64, fp, C.POINTER(orc._Uniforms), C.c_float, C.c_int, C.c_void_p, u32p, u32p, i64, u32p, fp,
                                C.POINTER(orc._FrameStats)]
        L.oro_set_blend_contraction.argtypes = [C.c_int]
        _oracle = L
    return _oracle


def emu_lib():
    global _emu
    if _emu is None:
        cxx = os.environ.get("ORC_CXX", "/usr/bin/g++")
        L = C.CDLL(_build("libortho_emu.so", _EMU_DEPS, lambda out: [cxx] + _EMU_FLAGS + ["-I", CUDA_INC, _EMU_DEPS[0], "-o", out]))
        L.emu_ortho_projection.restype = C.c_longlong
        L.emu_ortho_projection.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_ulonglong, C.c_uint, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.c_uint, C.POINTER(C.c_uint), C.POINTER(C.c_int), C.c_void_p, C.c_void_p,
                                           C.c_void_p]
        _emu = L
    return _emu


def _f(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _u(a):
    return a.ctypes.data_as(C.POINTER(C.c_uint32))


def is_orthographic(vp32) -> bool:
    """The library's rule on a GSR_FLAG_ORTHOGRAPHIC context: the projection's w row is exactly (0, 0, 0, 1)."""
    v = np.asarray(vp32, dtype=F32).reshape(32)
    return bool(v[19] == 0 and v[23] == 0 and v[27] == 0 and v[31] == 1)


# ---- cameras -----------------------------------------------------------------------------------------------------------------
def ortho_camera(width, height, size=4.0, near=0.05, far=4000.0, frame=None, keep_aspect=cam.KEEP_HEIGHT):
    """(vp32, uniforms bytes) of an orthographic Camera3D: the default camera (frame None) or orbit frame `frame`, packed with the
    projection's w row kept."""
    c = cam.default_camera(aspect=width / height) if frame is None else cam.orbit_camera(frame, aspect=width / height)
    c.projection, c.size, c.near, c.far, c.keep_aspect = cam.PROJECTION_ORTHOGONAL, float(size), float(near), float(far), keep_aspect
    vp = cam.pack_camera_push_constants(c.get_camera_transform(), c.get_camera_projection(), keep_w_row=True)
    return vp, uniforms_bytes(c.global_position, 1.0, width, height, 10.0)


# ---- the oracle --------------------------------------------------------------------------------------------------------------
def project(splat60, vp32, uniforms, cap=None) -> orc.Projection:
    """The orthographic projection of the oracle (pairs in emission order), like oracle.project."""
    splat60 = np.ascontiguousarray(splat60, dtype=F32).reshape(-1, 60)
    vp32 = np.ascontiguousarray(vp32, dtype=F32).reshape(32)
    n = splat60.shape[0]
    cap = int(cap if cap is not None else 64 * max(n, 1))
    recs = np.zeros(n, dtype=orc.RECORD_DTYPE)
    keys = np.zeros(max(cap, 1), dtype=np.uint32)
    vals = np.zeros(max(cap, 1), dtype=np.uint32)
    vis, last = C.c_int64(0), C.c_int64(-1)
    m = oracle_lib().oro_project(_f(splat60), n, _f(vp32), C.byref(uniforms), recs.ctypes.data, _u(keys), _u(vals), cap, C.byref(vis),
                                 C.byref(last))
    mm = min(int(m), cap)
    return orc.Projection(recs, keys[:mm].copy(), vals[:mm].copy(), int(vis.value), int(m), int(last.value))


def project_instanced(splat60, vp32, uniforms, ranges, xf) -> iref.InstanceProjection:
    """tests/instance_reference.project with the orthographic projection: instance k is projected with vp = (V_k, P); records move to
    drawn ids with frame-space positions; pairs are concatenated in instance order.  xf: (n, 24) float32 (GSR_BUF_INSTANCES)."""
    splat60 = np.ascontiguousarray(splat60, dtype=F32).reshape(-1, 60)
    vp32 = np.asarray(vp32, dtype=F32).reshape(32)
    w0, D = iref.layout(ranges)
    recs = np.zeros(D, dtype=orc.RECORD_DTYPE)
    keys, vals = [], []
    vis, m, last = 0, 0, -1
    for k, (first, count) in enumerate(ranges):
        first, count = int(first), int(count)
        if count == 0:
            continue
        Vk, _ = iref.compose(vp32[:16], uniforms.camera_pos[:], xf[k])
        pr = project(splat60[first:first + count], np.concatenate([Vk, vp32[16:]]), uniforms, cap=64 * count + 1024)
        assert pr.duplicates <= 64 * count + 1024
        emitted = np.unique(pr.values)
        r = pr.records[emitted].copy()
        sp = np.stack([r["pos_xy"][:, 0], r["pos_xy"][:, 1], r["pos_z"]], axis=1)
        w = iref.frame_position(xf[k], sp)
        r["pos_xy"] = w[:, :2]
        r["pos_z"] = w[:, 2]
        recs[32 * w0[k] + emitted] = r
        keys.append(pr.keys)
        vals.append(pr.values.astype(np.uint32) + np.uint32(32 * w0[k]))
        vis += pr.visible
        m += pr.duplicates
        last = max(last, pr.last_tile)
    cat = lambda xs: np.concatenate(xs).astype(np.uint32) if xs else np.zeros(0, dtype=np.uint32)
    return iref.InstanceProjection(recs, cat(keys), cat(vals), vis, m, last, D)


def oracle_frame(splat60, vp32, ub, heat=0.0, contract=True, inst=None, scene_depth=None, depth=False, quirks=True):
    """A whole orthographic frame: the orthographic projection (or its instanced composition; inst = [(first, count, to_frame12)]),
    then the oracle's sort, tile ranges and compositor -- or the depth-compositing oracle.  Returns a dict of every stage."""
    u = orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8))
    W, H = u.dims[0], u.dims[1]
    if inst is not None:
        pr = project_instanced(splat60, vp32, u, [(f, n) for f, n, _ in inst], np.stack([iref.inverse(x) for _, _, x in inst]))
    else:
        pr = project(splat60, vp32, u)
    T = ((W + 15) // 16) * ((H + 15) // 16)
    k, v = orc.sort_pairs(pr.keys, pr.values)
    b = orc.boundaries(k, T, quirks=quirks)
    dep = None
    if depth or scene_depth is not None:
        rgba, dep, staged = dref.render_depth(pr.records, v, b, W, H, vp32, scene_depth, heat, contract)
    else:
        orc.set_blend_contraction(contract)
        try:
            rgba, staged, _ = orc.render(pr.records, v, b, W, H, heat)
        finally:
            orc.set_blend_contraction(True)
    return dict(rgba=rgba, records=pr.records, keys=k, values=v, bounds=b, visible=pr.visible, m=pr.duplicates, last_tile=pr.last_tile,
                staged=staged, depth=dep)


def frame(splat60, vp32, ub, heat=0.0, quirks=True, contract=True):
    """oro_frame: the orthographic frame computed entirely inside the oracle library (projection, sort, tile ranges, compositor)."""
    splat60 = np.ascontiguousarray(splat60, dtype=F32).reshape(-1, 60)
    vp32 = np.ascontiguousarray(vp32, dtype=F32).reshape(32)
    u = orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8))
    n = splat60.shape[0]
    W, H = u.dims[0], u.dims[1]
    cap = 64 * max(n, 1)
    recs = np.zeros(n, dtype=orc.RECORD_DTYPE)
    keys = np.zeros(cap, dtype=np.uint32)
    vals = np.zeros(cap, dtype=np.uint32)
    bounds = np.zeros((((W + 15) // 16) * ((H + 15) // 16), 2), dtype=np.uint32)
    out = np.zeros((H, W, 4), dtype=F32)
    st = orc._FrameStats()
    L = oracle_lib()
    L.oro_set_blend_contraction(int(bool(contract)))
    try:
        rc = L.oro_frame(_f(splat60), n, _f(vp32), C.byref(u), float(heat), int(bool(quirks)), recs.ctypes.data, _u(keys), _u(vals), cap,
                         _u(bounds), _f(out), C.byref(st))
    finally:
        L.oro_set_blend_contraction(1)
    assert rc == 0
    m = int(st.duplicates)
    return dict(rgba=out, records=recs, keys=keys[:m].copy(), values=vals[:m].copy(), bounds=bounds, visible=int(st.visible), m=m,
                last_tile=int(st.last_tile), staged=int(st.staged))


# ---- the emulated kernels ----------------------------------------------------------------------------------------------------
def emu_project(store, bands, vp, ub, bulk_min, num_splats, ranges=None, xf=None):
    """projection_kernel<ranges is not None, bands, true> over `store` (soa_planes(store bands) x stride float4) on the CPU.
    Returns (records, keys, values, M, V, last tile) with the pairs in emission order."""
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
        warp_inst = np.full(((D + 255) // 256) * 8 + 1, 0xFFFFFFFF, dtype=np.uint32)
        for k, (_, c) in enumerate(ranges):
            warp_inst[w0[k]:w0[k] + (c + 31) // 32] = k
        desc = np.zeros(max(len(ranges), 1), dtype=np.dtype([("first", "<u8"), ("count", "<u4"), ("warp0", "<u4")]))
        for k, (f, c) in enumerate(ranges):
            desc[k] = (f, c, w0[k])
        n = D
    cap = 64 * max(n, 1)
    recs = np.zeros(max(n, 1), dtype=orc.RECORD_DTYPE)
    keys = np.zeros(cap, dtype=np.uint32)
    vals = np.zeros(cap, dtype=np.uint32)
    vis, last = C.c_uint(0), C.c_int(-1)
    vp32 = np.ascontiguousarray(vp, dtype=F32)
    ubuf = np.frombuffer(ub, dtype=np.uint8).copy()
    m = emu_lib().emu_ortho_projection(int(inst), int(bands), store.ctypes.data, stride, n, vp32.ctypes.data, ubuf.ctypes.data, int(bulk_min),
                                       recs.ctypes.data, keys.ctypes.data, vals.ctypes.data, cap, C.byref(vis), C.byref(last),
                                       None if frame_c is None else frame_c.ctypes.data, None if desc is None else desc.ctypes.data,
                                       None if warp_inst is None else warp_inst.ctypes.data)
    assert 0 <= m <= cap
    return recs[:n], keys[:m].copy(), vals[:m].copy(), int(m), int(vis.value), int(last.value)
