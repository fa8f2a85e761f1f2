"""Reference implementations of anti-aliased frames (include/gsr.h gsr_set_antialiasing) and of the filtered PLY ingest
(gsr_upload_ply_filtered) for the tests.

TEST INFRASTRUCTURE.  Two small shared libraries, built on first use from tests/aa_reference/:
  * aa_oracle.c -- the anti-aliased projection of the CPU oracle (project_one with the filter's dilation and the compensated opacity,
    optionally with the orthographic lines of tests/ortho_reference), compiled together with oracle/gsr_oracle.c, plus a frame on the
    oracle's own sort, tile ranges and compositor;
  * aa_emu.cpp  -- projection_kernel<INSTANCED, B, ORTHO, true> and ply_to_soa_kernel<true> compiled for the CPU on top of
    tests/kernel_emu.
Instances compose like tests/instance_reference.py: instance k is the anti-aliased projection with view matrix V_k = V * M_k.
They are written next to their sources, or to a temporary directory when the tree is read-only.
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

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "aa_reference")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "godotgaussiansplatting_b200", "csrc")
CUDA_INC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")

_ORACLE_DEPS = [os.path.join(HERE, "aa_oracle.c"), os.path.join(ROOT, "oracle", "gsr_oracle.c"), os.path.abspath(__file__)]
_EMU_DEPS = [os.path.join(HERE, "aa_emu.cpp"), os.path.abspath(__file__), os.path.join(ROOT, "include", "gsr.h")] + [
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
    d = os.path.join(tempfile.gettempdir(), f"gsr_aa_reference_{os.getuid()}")
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
        L = C.CDLL(_build("libaa_oracle.so", _ORACLE_DEPS, lambda out: [cc] + _ORC_FLAGS + [_ORACLE_DEPS[0], "-o", out, "-lm"]))
        fp, u32p, i64 = C.POINTER(C.c_float), C.POINTER(C.c_uint32), C.c_int64
        L.aao_project.restype = i64
        L.aao_project.argtypes = [fp, i64, fp, C.POINTER(orc._Uniforms), C.c_float, C.c_int, C.c_void_p, u32p, u32p, i64, C.POINTER(i64),
                                  C.POINTER(i64)]
        L.aao_frame.restype = C.c_int
        L.aao_frame.argtypes = [fp, i64, fp, C.POINTER(orc._Uniforms), C.c_float, C.c_int, C.c_float, C.c_int, C.c_void_p, u32p, u32p, i64,
                                u32p, fp, C.POINTER(orc._FrameStats)]
        L.aao_set_blend_contraction.argtypes = [C.c_int]
        _oracle = L
    return _oracle


def emu_lib():
    global _emu
    if _emu is None:
        cxx = os.environ.get("ORC_CXX", "/usr/bin/g++")
        L = C.CDLL(_build("libaa_emu.so", _EMU_DEPS, lambda out: [cxx] + _EMU_FLAGS + ["-I", CUDA_INC, _EMU_DEPS[0], "-o", out]))
        L.emu_aa_projection.restype = C.c_longlong
        L.emu_aa_projection.argtypes = [C.c_int, C.c_int, C.c_int, C.c_float, C.c_void_p, C.c_ulonglong, C.c_uint, C.c_void_p, C.c_void_p,
                                        C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint, C.POINTER(C.c_uint), C.POINTER(C.c_int),
                                        C.c_void_p, C.c_void_p, C.c_void_p]
        L.emu_aa_ply_to_soa.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_ulonglong, C.c_float, C.c_void_p, C.c_ulonglong, C.c_ulonglong,
                                        C.c_int]
        _emu = L
    return _emu


def _f(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _u(a):
    return a.ctypes.data_as(C.POINTER(C.c_uint32))


# ---- the oracle --------------------------------------------------------------------------------------------------------------
def project(splat60, vp32, uniforms, v, ortho=False, cap=None) -> orc.Projection:
    """The anti-aliased projection of the oracle with filter variance v (pairs in emission order), like oracle.project."""
    splat60 = np.ascontiguousarray(splat60, dtype=F32).reshape(-1, 60)
    vp32 = np.ascontiguousarray(vp32, dtype=F32).reshape(32)
    n = splat60.shape[0]
    cap = int(cap if cap is not None else 64 * max(n, 1))
    recs = np.zeros(n, dtype=orc.RECORD_DTYPE)
    keys = np.zeros(max(cap, 1), dtype=np.uint32)
    vals = np.zeros(max(cap, 1), dtype=np.uint32)
    vis, last = C.c_int64(0), C.c_int64(-1)
    m = oracle_lib().aao_project(_f(splat60), n, _f(vp32), C.byref(uniforms), float(v), int(bool(ortho)), recs.ctypes.data, _u(keys), _u(vals),
                                 cap, C.byref(vis), C.byref(last))
    mm = min(int(m), cap)
    return orc.Projection(recs, keys[:mm].copy(), vals[:mm].copy(), int(vis.value), int(m), int(last.value))


def project_instanced(splat60, vp32, uniforms, ranges, xf, v, ortho=False) -> iref.InstanceProjection:
    """tests/instance_reference.project with the anti-aliased projection: instance k is projected with vp = (V_k, P); records move to
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
        Vk, camk = iref.compose(vp32[:16], uniforms.camera_pos[:], xf[k])
        uk = orc.make_uniforms(camk, uniforms.model_scale, uniforms.dims[0], uniforms.dims[1], uniforms.time)
        uk.camera_pos[:] = [float(c) for c in camk]
        pr = project(splat60[first:first + count], np.concatenate([Vk, vp32[16:]]), uk, v, ortho, cap=64 * count + 1024)
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


def oracle_frame(splat60, vp32, ub, v, ortho=False, heat=0.0, contract=True, inst=None, scene_depth=None, depth=False, quirks=True):
    """A whole anti-aliased frame: the anti-aliased projection (or its instanced composition; inst = [(first, count, to_frame12)]),
    then the oracle's sort, tile ranges and compositor -- or the depth-compositing oracle.  Returns a dict of every stage."""
    u = orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8))
    W, H = u.dims[0], u.dims[1]
    if inst is not None:
        pr = project_instanced(splat60, vp32, u, [(f, n) for f, n, _ in inst], np.stack([iref.inverse(x) for _, _, x in inst]), v, ortho)
    else:
        pr = project(splat60, vp32, u, v, ortho)
    T = ((W + 15) // 16) * ((H + 15) // 16)
    k, vals = orc.sort_pairs(pr.keys, pr.values)
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
    return dict(rgba=rgba, records=pr.records, keys=k, values=vals, bounds=b, visible=pr.visible, m=pr.duplicates, last_tile=pr.last_tile,
                staged=staged, depth=dep)


def frame(splat60, vp32, ub, v, ortho=False, heat=0.0, quirks=True, contract=True):
    """aao_frame: the anti-aliased frame computed entirely inside the oracle library (projection, sort, tile ranges, compositor)."""
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
    L.aao_set_blend_contraction(int(bool(contract)))
    try:
        rc = L.aao_frame(_f(splat60), n, _f(vp32), C.byref(u), float(v), int(bool(ortho)), float(heat), int(bool(quirks)), recs.ctypes.data,
                         _u(keys), _u(vals), cap, _u(bounds), _f(out), C.byref(st))
    finally:
        L.aao_set_blend_contraction(1)
    assert rc == 0
    m = int(st.duplicates)
    return dict(rgba=out, records=recs, keys=keys[:m].copy(), values=vals[:m].copy(), bounds=bounds, visible=int(st.visible), m=m,
                last_tile=int(st.last_tile), staged=int(st.staged))


# ---- the emulated kernels ----------------------------------------------------------------------------------------------------
def emu_project(store, bands, vp, ub, bulk_min, num_splats, v, ortho=False, ranges=None, xf=None):
    """projection_kernel<ranges is not None, bands, ortho, true> with aa_variance v over `store` (soa_planes(store bands) x stride
    float4) on the CPU.  Returns (records, keys, values, M, V, last tile) with the pairs in emission order."""
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
    m = emu_lib().emu_aa_projection(int(inst), int(bands), int(bool(ortho)), float(v), store.ctypes.data, stride, n, vp32.ctypes.data,
                                    ubuf.ctypes.data, int(bulk_min), recs.ctypes.data, keys.ctypes.data, vals.ctypes.data, cap, C.byref(vis),
                                    C.byref(last), None if frame_c is None else frame_c.ctypes.data,
                                    None if desc is None else desc.ctypes.data, None if warp_inst is None else warp_inst.ctypes.data)
    assert 0 <= m <= cap
    return recs[:n], keys[:m].copy(), vals[:m].copy(), int(m), int(vis.value), int(last.value)


def emu_ply_to_soa(table, layout, creation_time, planes, stride, first=0):
    """ply_to_soa_kernel<true> (gsr_upload_ply_filtered) of `table` with PlyLayout `layout` (filter_3d >= 0) on the CPU: the stored
    planes, (planes, stride, 4) float32, NaN where nothing was written."""
    t = np.ascontiguousarray(table, dtype=F32)
    lay = np.array([layout.nprops, layout.sh_degree, layout.x, layout.f_dc, layout.f_rest, layout.opacity, layout.scale, layout.rot],
                   dtype=np.int32)
    soa = np.full((planes, stride, 4), np.nan, dtype=F32)
    assert emu_lib().emu_aa_ply_to_soa(t.ctypes.data, lay.ctypes.data, int(layout.filter_3d), t.shape[0], float(creation_time), soa.ctypes.data,
                                       stride, first, planes) == 0
    return soa
