"""Splat clouds of SH degree 0, 1 and 2 on the CPU (include/gsr.h gsr_config.sh_bands, gsr_upload_ply, gsr_set_sh_degree): the PLY layout
of the Python mirror, the generalised swizzle, and the degree variants of the ingest and projection kernels compiled for the CPU
(tests/sh_reference/sh_emu.cpp on top of tests/kernel_emu) against the unchanged oracle on the zero-padded cloud, bit for bit."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from godotgaussiansplatting_b200.ply_file import PLY_LAYOUT_3DGS, PlyFile, degree_properties, narrow_table, swizzle_splats
from godotgaussiansplatting_b200.synthetic import synthetic_ply_table
from oracle import oracle as orc
from tests import instance_reference as iref
from tests.scenes import make_scene

F32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.join(ROOT, "tests", "sh_reference")
CSRC = os.path.join(ROOT, "godotgaussiansplatting_b200", "csrc")
CUDA_INC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
_DEPS = [os.path.join(HERE, "sh_emu.cpp"), os.path.join(ROOT, "tests", "kernel_emu", "kernel_emu.cpp"), os.path.join(ROOT, "tests", "kernel_emu", "cuda_shim.h"),
         os.path.join(ROOT, "oracle", "glsl_cpu", "glsl_emu.hpp"), os.path.join(ROOT, "include", "gsr.h")] + [
    os.path.join(CSRC, f) for f in ("compositor.cu", "ranges.cu", "radix_sort.cu", "projection.cu", "ingest.cu", "present.cu", "group.cu", "common.cuh")]
_FLAGS = ["-std=gnu++17", "-O1", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-w"]
_emu = None

REST = (0, 9, 24, 45)


def sh_planes(bands):
    return (3 * bands * bands + 3) // 4


def emu():
    global _emu
    if _emu is None:
        d = HERE if os.access(HERE, os.W_OK) else os.path.join(tempfile.gettempdir(), f"gsr_sh_reference_{os.getuid()}")
        os.makedirs(d, exist_ok=True)
        out = os.path.join(d, "libsh_emu.so")
        if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(p) for p in _DEPS):
            subprocess.run([os.environ.get("ORC_CXX", "/usr/bin/g++")] + _FLAGS + ["-I", CUDA_INC, _DEPS[0], "-o", out], check=True)
        L = C.CDLL(out)
        L.emu_sh_ply_to_soa.argtypes = [C.c_void_p, C.c_void_p, C.c_ulonglong, C.c_float, C.c_void_p, C.c_ulonglong, C.c_ulonglong, C.c_int]
        L.emu_sh_aos_to_soa.argtypes = [C.c_void_p, C.c_ulonglong, C.c_void_p, C.c_ulonglong, C.c_ulonglong, C.c_int]
        L.emu_sh_projection.restype = C.c_longlong
        L.emu_sh_projection.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_ulonglong, C.c_uint, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_uint, C.POINTER(C.c_uint), C.POINTER(C.c_int), C.c_void_p, C.c_void_p, C.c_void_p]
        _emu = L
    return _emu


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def zero_above(table62, degree):
    """The standard table with every SH coefficient above `degree` set to zero (the zero-padded cloud of a degree-`degree` file)."""
    t = np.array(table62, dtype=F32, copy=True)
    t[:, 9:54].reshape(-1, 3, 15)[:, :, REST[degree] // 3:] = 0.0
    return t


def layout_ints(lay):
    return np.array([lay.nprops, lay.sh_degree, lay.x, lay.f_dc, lay.f_rest, lay.opacity, lay.scale, lay.rot], dtype=np.int32)


def expected_planes(splat60, bands, stride):
    """The planes a `bands` store holds for `splat60`: the first 3 + P planes of the 15-plane layout, floats past 3K zero."""
    n = splat60.shape[0]
    s = np.array(splat60, dtype=F32, copy=True)
    s[:, 12 + 3 * bands * bands:] = 0.0
    out = np.zeros((3 + sh_planes(bands), stride, 4), dtype=F32)
    out[:, :n] = s.reshape(n, 15, 4).transpose(1, 0, 2)[:3 + sh_planes(bands)]
    return out


# ---- PlyFile.layout ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("normals", [True, False])
@pytest.mark.parametrize("degree", [0, 1, 2, 3])
def test_layout_from_property_names(degree, normals):
    for extra in ((), ("semantic", "age")):
        names = degree_properties(degree, normals, extra)
        lay = PlyFile.from_array(np.zeros((1, len(names)), F32), names).layout()
        off = 0 if normals else -3
        assert lay.nprops == len(names) and lay.sh_degree == degree and lay.x == 0 and lay.f_dc == 6 + off
        assert lay.f_rest == (9 + off if degree else -1)
        assert lay.opacity == 9 + off + REST[degree] and lay.scale == lay.opacity + 1 and lay.rot == lay.scale + 3
    assert PlyFile.from_array(np.zeros((1, 62), F32)).layout() == PLY_LAYOUT_3DGS


def test_layout_rejects():
    def lay(names):
        return PlyFile.from_array(np.zeros((1, len(names)), F32), names).layout()
    names = degree_properties(1)
    with pytest.raises(ValueError, match="f_rest"):
        lay(names + ["f_rest_9"])                       # 10 f_rest floats
    with pytest.raises(ValueError, match="contiguous"):
        lay(["y", "x", "z"] + names[3:])                # x y z out of order
    with pytest.raises(ValueError, match="contiguous"):
        lay(names[:10] + ["extra"] + names[10:])        # a gap inside f_rest
    with pytest.raises(ValueError, match="opacity"):
        lay([n for n in names if n != "opacity"])


# ---- the generalised swizzle ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("normals", [True, False])
@pytest.mark.parametrize("degree", [0, 1, 2, 3])
def test_swizzle_of_a_narrow_table_is_the_zero_padded_one(degree, normals):
    t62 = zero_above(synthetic_ply_table(700, 3), degree)
    names = degree_properties(degree, normals, ("extra",))
    narrow = np.concatenate([narrow_table(t62, degree, normals), np.full((700, 1), 7.0, F32)], axis=1)
    got = swizzle_splats(narrow, 1.25, PlyFile.from_array(narrow, names).layout())
    assert np.array_equal(bits(got), bits(swizzle_splats(t62, 1.25)))


# ---- emulated ingest --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("file_degree", [0, 1, 2, 3])
def test_emulated_ply_ingest_stores_the_zero_padded_planes(file_degree):
    n, first, stride = 300, 5, 512
    t62 = synthetic_ply_table(n, 4)
    t62[:, 9:54] += 0.01   # no coefficient of the file is zero
    names = degree_properties(file_degree, normals=file_degree % 2 == 0)
    narrow = narrow_table(t62, file_degree, normals=file_degree % 2 == 0)
    lay = PlyFile.from_array(narrow, names).layout()
    for bands in (1, 2, 3, 4):
        soa = np.full((3 + sh_planes(bands), stride, 4), np.nan, dtype=F32)
        assert emu().emu_sh_ply_to_soa(narrow.ctypes.data, layout_ints(lay).ctypes.data, n, 2.5, soa.ctypes.data, stride, first, 3 + sh_planes(bands)) == 0
        want = expected_planes(swizzle_splats(zero_above(t62, min(file_degree, bands - 1)), 2.5), bands, n)
        assert np.array_equal(bits(soa[:, first:first + n]), bits(want)), (file_degree, bands)
        assert np.isnan(soa[:, :first]).all() and np.isnan(soa[:, first + n:]).all()   # nothing outside the range


def test_emulated_aos_ingest_with_fewer_planes():
    n, first, stride = 300, 7, 512
    splat60 = swizzle_splats(synthetic_ply_table(n, 5), 0.5)
    splat60[:, 12:] += 0.01
    for bands in (1, 2, 3, 4):
        soa = np.full((3 + sh_planes(bands), stride, 4), np.nan, dtype=F32)
        emu().emu_sh_aos_to_soa(splat60.ctypes.data, n, soa.ctypes.data, stride, first, 3 + sh_planes(bands))
        assert np.array_equal(bits(soa[:, first:first + n]), bits(expected_planes(splat60, bands, n))), bands
        assert np.isnan(soa[:, :first]).all() and np.isnan(soa[:, first + n:]).all()


# ---- emulated projection against the oracle ---------------------------------------------------------------------------------------
N, W, H = 2048, 128, 96


def desc_bytes(ranges):
    w0, _ = iref.layout(ranges)
    d = np.zeros(max(len(ranges), 1), dtype=np.dtype([("first", "<u8"), ("count", "<u4"), ("warp0", "<u4")]))
    for k, (f, c) in enumerate(ranges):
        d[k] = (f, c, w0[k])
    return d


def emu_project(store, bands, vp, ub, bulk_min, ranges=None, xf=None):
    """projection_kernel<ranges is not None, bands> over the store planes.  Returns (records, keys, values, M, V, last tile)."""
    stride = store.shape[1]
    inst = ranges is not None
    if inst:
        w0, D = iref.layout(ranges)
        u = orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8))
        frame = np.zeros((len(ranges), 32), dtype=F32)
        for k in range(len(ranges)):
            Vk, camk = iref.compose(vp[:16], u.camera_pos[:], xf[k])
            frame[k, :16], frame[k, 16:19], frame[k, 19:31] = Vk, camk, xf[k][:12]
        warp_inst = np.full(((D + 255) // 256) * 8 + 1, 0xFFFFFFFF, dtype=np.uint32)
        for k, (_, c) in enumerate(ranges):
            warp_inst[w0[k]:w0[k] + (c + 31) // 32] = k
        desc = desc_bytes(ranges)
        n = D
    else:
        n = N
    cap = 64 * n
    recs = np.zeros(max(n, 1), dtype=orc.RECORD_DTYPE)
    keys = np.zeros(cap, dtype=np.uint32)
    vals = np.zeros(cap, dtype=np.uint32)
    vis, last = C.c_uint(0), C.c_int(-1)
    vp32 = np.ascontiguousarray(vp, dtype=F32)
    ubuf = np.frombuffer(ub, dtype=np.uint8).copy()
    m = emu().emu_sh_projection(int(inst), bands, store.ctypes.data, stride, n, vp32.ctypes.data, ubuf.ctypes.data, bulk_min, recs.ctypes.data,
                                keys.ctypes.data, vals.ctypes.data, cap, C.byref(vis), C.byref(last),
                                frame.ctypes.data if inst else None, desc.ctypes.data if inst else None, warp_inst.ctypes.data if inst else None)
    assert 0 <= m <= cap
    return recs, keys[:m], vals[:m], int(m), int(vis.value), int(last.value)


def oracle_project(splat60, vp, ub, ranges=None, xf=None):
    u = orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8))
    if ranges is not None:
        p = iref.project(splat60, vp, u, ranges, xf)
        return p.records, p.keys, p.values, p.duplicates, p.visible, p.last_tile
    p = orc.project(splat60, vp, u, cap=64 * N)
    return p.records, p.keys, p.values, p.duplicates, p.visible, p.last_tile


def assert_same_projection(got, want):
    recs, keys, vals, m, vis, last = got
    wr, wk, wv, wm, wvis, wlast = want
    assert (m, vis, last) == (wm, wvis, wlast)
    assert np.array_equal(keys, wk) and np.array_equal(vals, wv)
    ids = np.unique(wv)
    assert np.array_equal(bits(recs[ids].view(np.float32).reshape(len(ids), 12)), bits(wr[ids].view(np.float32).reshape(len(ids), 12)))


def scene(time, seed=11, camera_splat=False):
    t62 = synthetic_ply_table(N, seed)
    t62[:, 9:54] += 0.02   # every coefficient non-zero
    splat60, vp, ub = make_scene(16, 1, W, H, frame=5, time=time)
    splat60 = swizzle_splats(t62, 0.0)
    if camera_splat:   # uniforms.camera_pos on a visible splat: its view direction is 0/0 = NaN
        u = np.frombuffer(ub, dtype=F32).copy()
        p = orc.project(splat60, vp, orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8)), cap=64 * N)
        i = int(p.values[len(p.values) // 2])
        u[0:3] = splat60[i, 0:3]
        ub = u.tobytes()
    return splat60, vp, ub


def store_of(splat60, bands):
    return np.ascontiguousarray(expected_planes(splat60, bands, (N + 255) // 256 * 256))


def zero_splat_coeffs(splat60, bands):
    s = np.array(splat60, dtype=F32, copy=True)
    s[:, 12 + 3 * bands * bands:] = 0.0
    return s




@pytest.mark.parametrize("time", [10.0, 0.6], ids=["static", "load_in"])
@pytest.mark.parametrize("bulk_min", [1, 33], ids=["bulk", "gather"])
@pytest.mark.parametrize("instanced", [False, True], ids=["default", "instances"])
@pytest.mark.parametrize("bands", [1, 2, 3])
def test_emulated_projection_is_the_zero_padded_oracle(bands, instanced, bulk_min, time):
    splat60, vp, ub = scene(time)
    ranges = xf = None
    if instanced:
        from tests.test_instances import SCALED, rigid
        ranges = [(0, 600), (600, 700), (1300, 748), (100, 33)]
        xf = [iref.inverse(m) for m in (rigid(4), SCALED, rigid(6), rigid(7))]
    padded = zero_splat_coeffs(splat60, bands)
    want = oracle_project(padded, vp, ub, ranges, xf)
    assert want[3] > 0
    # a reduced store of the padded cloud, and a 4-band store of the full cloud (non-zero higher coefficients) rendered at bands - 1
    assert_same_projection(emu_project(store_of(padded, bands), bands, vp, ub, bulk_min, ranges, xf), want)
    assert_same_projection(emu_project(store_of(splat60, 4), bands, vp, ub, bulk_min, ranges, xf), want)


@pytest.mark.parametrize("bands", [1, 2, 3, 4])
def test_emulated_projection_of_a_splat_at_the_camera_position(bands):
    splat60, vp, ub = scene(10.0, camera_splat=True)
    padded = zero_splat_coeffs(splat60, bands)
    want = oracle_project(padded, vp, ub)
    cols = want[0]["color"]
    assert (~np.isfinite(np.frombuffer(ub, dtype=F32)[:3])).sum() == 0
    for bulk_min in (1, 33):
        assert_same_projection(emu_project(store_of(splat60, 4), bands, vp, ub, bulk_min), want)
        assert_same_projection(emu_project(store_of(padded, bands), bands, vp, ub, bulk_min), want)
    # the splat at the camera position is black at every degree, as the degree-3 evaluation makes it
    u = np.frombuffer(ub, dtype=F32)
    at = np.where((splat60[:, 0:3] == u[0:3]).all(axis=1))[0]
    assert at.size >= 1 and (cols[at[0], :3] == 0.0).all()
