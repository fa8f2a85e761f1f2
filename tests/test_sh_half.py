"""The binary16 SH store (include/gsr.h GSR_FLAG_SH_HALF) without a GPU: the two conversions, the packed layout the ingest kernels write,
and the binary16-store projection kernels compiled for the CPU (tests/sh_half_reference/sh_half_emu.cpp on top of tests/kernel_emu),
bit for bit against the unchanged oracle and the per-feature references on the cloud whose coefficients were rounded to binary16 once."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from godotgaussiansplatting_b200 import _lib
from godotgaussiansplatting_b200.ply_file import PlyFile, PlyLayout, degree_properties, narrow_table, swizzle_splats
from godotgaussiansplatting_b200.synthetic import synthetic_ply_table
from oracle import oracle as orc
from tests import cutout_reference as cr
from tests import depth_order_reference as dor
from tests import instance_appearance_reference as ar
from tests import ortho_reference as oref
from tests.test_cutouts import crop_set, frame_positions
from tests.test_depth_order import H, N, W, instances, scene
from tests.test_sh_degree import zero_splat_coeffs

F32, U32, F16 = np.float32, np.uint32, np.float16
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.join(ROOT, "tests", "sh_half_reference")
CSRC = os.path.join(ROOT, "godotgaussiansplatting_b200", "csrc")
CUDA_INC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
_DEPS = [os.path.join(HERE, "sh_half_emu.cpp"), os.path.join(ROOT, "tests", "kernel_emu", "kernel_emu.cpp"),
         os.path.join(ROOT, "tests", "kernel_emu", "cuda_shim.h"), os.path.join(ROOT, "oracle", "glsl_cpu", "glsl_emu.hpp"),
         os.path.join(ROOT, "include", "gsr.h")] + [
    os.path.join(CSRC, f) for f in ("compositor.cu", "ranges.cu", "radix_sort.cu", "projection.cu", "ingest.cu", "present.cu", "group.cu", "common.cuh")]
_FLAGS = ["-std=gnu++17", "-O1", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-w"]
_emu = None


def emu():
    global _emu
    if _emu is None:
        d = HERE if os.access(HERE, os.W_OK) else os.path.join(tempfile.gettempdir(), f"gsr_sh_half_reference_{os.getuid()}")
        os.makedirs(d, exist_ok=True)
        out = os.path.join(d, "libsh_half_emu.so")
        if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(p) for p in _DEPS):
            tmp = f"{out}.{os.getpid()}.tmp"   # concurrent test processes each build their own copy and swap it in whole
            subprocess.run([os.environ.get("ORC_CXX", "/usr/bin/g++")] + _FLAGS + ["-I", CUDA_INC, _DEPS[0], "-o", tmp], check=True)
            os.replace(tmp, out)
        L = C.CDLL(out)
        vp, uint = C.c_void_p, C.c_uint
        L.emu_sh_half_encode.argtypes = [vp, vp, C.c_ulonglong]
        L.emu_sh_half_decode.argtypes = [vp, vp, C.c_ulonglong]
        L.emu_sh_half_aos_to_soa.argtypes = [vp, C.c_ulonglong, vp, C.c_ulonglong, C.c_ulonglong, C.c_int]
        L.emu_sh_half_ply_to_soa.argtypes = [vp, vp, C.c_ulonglong, C.c_float, vp, C.c_ulonglong, C.c_ulonglong, C.c_int, C.c_int]
        L.emu_sh_half_projection.restype = C.c_longlong
        L.emu_sh_half_projection.argtypes = [C.c_int, C.c_int, C.c_float, vp, C.c_ulonglong, uint, vp, vp, C.c_int, uint, vp, vp, vp, vp, vp, vp,
                                             vp, uint, C.POINTER(uint), C.POINTER(C.c_int), C.POINTER(uint), vp]
        _emu = L
    return _emu


def bits(a):
    return np.ascontiguousarray(a).view(U32)


# ---- the rule and the layout in numpy ---------------------------------------------------------------------------------------------
def half_planes_count(bands):
    return (3 * bands * bands + 7) // 8


def h(c):
    """h(c): round to nearest even binary16 (numpy's conversion), with values beyond +-65504 saturated (NaN stays NaN)."""
    c = np.asarray(c, dtype=F32)
    with np.errstate(invalid="ignore"):
        s = np.where(np.abs(c) > F32(65504.0), np.copysign(F32(65504.0), c), c).astype(F32)
    with np.errstate(over="ignore"):
        return s.astype(F16)


def rounded(splat60, bands=4):
    """The cloud a `bands` binary16 store draws: coefficients above the store's degree zero, the others float(h(c))."""
    s = zero_splat_coeffs(splat60, bands)
    s[:, 12:] = h(s[:, 12:]).astype(F32)
    return s


def half_planes(splat60, bands, stride=None):
    """The planes a `bands` binary16 store holds for `splat60`: planes 0-2 as floats, then P_h planes of 8 halves (slots past 3K +0)."""
    s = np.ascontiguousarray(splat60, dtype=F32).reshape(-1, 60)
    n = s.shape[0]
    stride = n if stride is None else stride
    P, K3 = half_planes_count(bands), 3 * bands * bands
    out = np.zeros((3 + P, stride, 4), dtype=F32)
    out[:3, :n] = s[:, :12].reshape(n, 3, 4).transpose(1, 0, 2)
    hv = np.zeros((n, 8 * P), dtype=F16)
    hv[:, :K3] = h(s[:, 12:12 + K3])
    out[3:, :n] = hv.view(U32).reshape(n, P, 4).transpose(1, 0, 2).view(F32)
    return out


def store_of(splat60, bands):
    return np.ascontiguousarray(half_planes(splat60, bands, (splat60.shape[0] + 255) // 256 * 256))


# ---- the conversions --------------------------------------------------------------------------------------------------------------
def test_flag_value():
    assert _lib.GSR_FLAG_SH_HALF == 0x40
    assert [half_planes_count(b) for b in (1, 2, 3, 4)] == [1, 2, 4, 6]
    assert [16 * (3 + half_planes_count(b)) for b in (1, 2, 3, 4)] == [64, 80, 112, 144]


def test_decode_of_every_pattern_is_numpys():
    pat = np.arange(65536, dtype=np.uint32).astype(np.uint16)
    got = np.zeros(65536, dtype=F32)
    emu().emu_sh_half_decode(pat.ctypes.data, got.ctypes.data, 65536)
    np.testing.assert_array_equal(bits(got), bits(pat.view(F16).astype(F32)))


def encode(x):
    x = np.ascontiguousarray(x, dtype=F32)
    out = np.zeros(x.size, dtype=np.uint16)
    emu().emu_sh_half_encode(x.ctypes.data, out.ctypes.data, x.size)
    return out


def test_encode_is_round_to_nearest_even_with_saturation():
    rng = np.random.default_rng(5)
    special = np.array([0.0, -0.0, 1.0, 1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11, 1.0 + 2.0 ** -11 + 2.0 ** -23, 2.0 ** -24, 2.0 ** -25,
                        2.0 ** -25 + 2.0 ** -40, 3 * 2.0 ** -25, 2.0 ** -14, 2.0 ** -14 - 2.0 ** -25, 2.0 ** -26, 1e-30, 1.4e-45,
                        65504.0, 65519.99, 65520.0, 65536.0, 1e30, np.inf, 2048.0 + 1.0, 2048.0 + 3.0, 0.1, 1 / 3], dtype=F32)
    special = np.concatenate([special, -special])
    dense = np.concatenate([
        rng.integers(0, 2 ** 32, size=1 << 20, dtype=np.uint64).astype(U32).view(F32),              # every exponent
        np.arange(0x33000000, 0x33000000 + (1 << 20), 7, dtype=U32).view(F32),                      # around 2^-25: the subnormal edge
        np.arange(0x387FF000, 0x38801000, dtype=U32).view(F32),                                     # the subnormal / normal boundary
        np.arange(0x477FD000, 0x47801000, dtype=U32).view(F32),                                     # 65504 .. 65536: the saturation edge
        np.arange(0x3F800000, 0x3F800000 + (1 << 16), dtype=U32).view(F32),                         # ties and neighbours above 1
    ])
    x = np.concatenate([special, dense, -dense])
    nan = np.isnan(x)
    got = encode(x)
    want = h(x).view(np.uint16)
    np.testing.assert_array_equal(got[~nan], want[~nan])
    assert np.isnan(got[nan].view(F16)).all()                 # NaN stays a NaN (payload and sign unspecified)
    one = lambda v: int(encode(np.array([v], dtype=F32))[0])
    assert one(65519.99) == one(65520.0) == one(np.inf) == one(1e30) == 0x7BFF and one(-np.inf) == 0xFBFF   # saturated, never inf
    assert one(1.0 + 2.0 ** -11) == 0x3C00 and one(1.0 + 3 * 2.0 ** -11) == 0x3C02                            # ties to even
    assert one(2.0 ** -24) == 0x0001 and one(2.0 ** -25) == 0x0000 and one(3 * 2.0 ** -25) == 0x0002          # subnormal halves
    assert one(-0.0) == 0x8000 and one(0.0) == 0x0000                                                          # signed zeros
    assert np.isnan(encode(np.array([np.nan, -np.nan], dtype=F32)).view(F16)).all()


# ---- emulated ingest --------------------------------------------------------------------------------------------------------------
def test_emulated_aos_ingest_packs_the_planes():
    n, first, stride = 300, 7, 512
    splat60 = swizzle_splats(synthetic_ply_table(n, 5), 0.5)
    splat60[:, 12:] += 0.01
    splat60[::7, 12:] *= 1e5                  # saturated coefficients
    splat60[1::7, 12:] *= 1e-6                # subnormal halves
    splat60[2, 12:] = -0.0
    for bands in (1, 2, 3, 4):
        P = 3 + half_planes_count(bands)
        soa = np.full((P, stride, 4), np.nan, dtype=F32)
        emu().emu_sh_half_aos_to_soa(splat60.ctypes.data, n, soa.ctypes.data, stride, first, P)
        assert np.array_equal(bits(soa[:, first:first + n]), bits(half_planes(splat60, bands))), bands
        assert np.isnan(soa[:, :first]).all() and np.isnan(soa[:, first + n:]).all()


def layout_ints(lay):
    return np.array([lay.nprops, lay.sh_degree, lay.x, lay.f_dc, lay.f_rest, lay.opacity, lay.scale, lay.rot], dtype=np.int32)


@pytest.mark.parametrize("filtered", [False, True], ids=["plain", "filter_3d"])
@pytest.mark.parametrize("file_degree", [0, 1, 2, 3])
def test_emulated_ply_ingest_packs_the_planes(file_degree, filtered):
    n, first, stride = 300, 5, 512
    t62 = synthetic_ply_table(n, 4)
    t62[:, 9:54] += 0.01
    names = degree_properties(file_degree, normals=file_degree % 2 == 0, extra=("filter_3D",) if filtered else ())
    narrow = narrow_table(t62, file_degree, normals=file_degree % 2 == 0)
    if filtered:
        f = np.random.default_rng(2).uniform(-0.01, 0.05, size=(n, 1)).astype(F32)   # some f <= 0: stored without the filter
        narrow = np.ascontiguousarray(np.concatenate([narrow, f], axis=1))
    lay = PlyFile.from_array(narrow, names).layout()
    assert (lay.filter_3d >= 0) == filtered
    mirror = swizzle_splats(narrow, 2.5, lay)   # the float store's splats (the 3D filter folded in)
    for bands in (1, 2, 3, 4):
        P = 3 + half_planes_count(bands)
        soa = np.full((P, stride, 4), np.nan, dtype=F32)
        assert emu().emu_sh_half_ply_to_soa(narrow.ctypes.data, layout_ints(lay).ctypes.data, n, 2.5, soa.ctypes.data, stride, first, P,
                                            int(lay.filter_3d)) == 0
        assert np.array_equal(bits(soa[:, first:first + n]), bits(half_planes(mirror, bands))), (file_degree, bands)
        assert np.isnan(soa[:, :first]).all() and np.isnan(soa[:, first + n:]).all()


# ---- emulated projection against the references on the rounded cloud -------------------------------------------------------------
def emu_project(store, bands, vp, ub, bulk_min, num_splats, v=0.0, ortho=False, inst=None, app=None, vols=None, depth=False):
    """projection_kernel<inst is not None, bands, ortho, v > 0, depth, vols is not None, true> over the binary16 `store`.
    Returns (records, keys, values, depth words or None, M, V, last tile) with the pairs in emission order."""
    stride = store.shape[1]
    n = 0 if inst is None else len(inst)
    if n:
        ranges = [(int(f), int(c)) for f, c, _ in inst]
        D = ar.iref.layout(ranges)[1]
        rng = np.array(ranges, dtype=np.uint64).reshape(-1)
        xf = np.ascontiguousarray(np.stack([ar.iref.inverse(x) for _, _, x in inst]), dtype=F32).reshape(-1)
        rws = None if app is None else np.ascontiguousarray(ar.rows(ranges, app))
    else:
        D, rng, xf, rws = num_splats, None, None, None
    cap = 64 * max(D, 1)
    recs = np.zeros(max(D, 1), dtype=orc.RECORD_DTYPE)
    keys, vals = np.zeros(cap, dtype=U32), np.zeros(cap, dtype=U32)
    words = np.zeros(cap, dtype=U32) if depth else None
    args = None if vols is None else np.array([cr.cutout_args(vols)], dtype=cr.ARGS_DTYPE)
    vis, last, ovf = C.c_uint(0), C.c_int(-1), C.c_uint(0)
    vp32 = np.ascontiguousarray(vp, dtype=F32)
    ubuf = np.frombuffer(ub, dtype=np.uint8).copy()
    ptr = lambda a: None if a is None else a.ctypes.data
    m = emu().emu_sh_half_projection(int(bands), int(bool(ortho)), float(v), store.ctypes.data, stride, int(num_splats), vp32.ctypes.data,
                                     ubuf.ctypes.data, int(bulk_min), n, ptr(xf), ptr(rng), ptr(rws), recs.ctypes.data, keys.ctypes.data,
                                     vals.ctypes.data, ptr(words), cap, C.byref(vis), C.byref(last), C.byref(ovf), ptr(args))
    assert 0 <= m <= cap and ovf.value == 0
    return recs[:D], keys[:m].copy(), vals[:m].copy(), None if words is None else words[:m].copy(), int(m), int(vis.value), int(last.value)


def check(got, want_recs, want_keys, want_vals, want_m, want_vis, want_last, vp=None):
    recs, keys, vals, words, m, vis, last = got
    assert (m, vis, last) == (want_m, want_vis, want_last)
    np.testing.assert_array_equal(keys, want_keys)
    np.testing.assert_array_equal(vals, want_vals)
    ids = np.unique(want_vals)
    np.testing.assert_array_equal(bits(recs[ids].view(F32)), bits(want_recs[ids].view(F32)))
    if words is not None:
        np.testing.assert_array_equal(words, dor.ord_words(dor.view_depth(want_recs, want_vals, vp)))


def check_plain(store, bands, cloud, vp, ub, v=0.0, ortho=False, depth=False, bulk=(1, 33)):
    """The kernel without instances against the reference projection of `cloud` (tests/depth_order_reference.project)."""
    pr = dor.project(cloud, vp, orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8)), v, ortho, None)
    assert pr.duplicates > 0
    for bulk_min in bulk:
        got = emu_project(store, bands, vp, ub, bulk_min, N, v, ortho, depth=depth)
        check(got, pr.records, pr.keys, pr.values, pr.duplicates, pr.visible, pr.last_tile, vp)
    return pr


def check_instanced(store, bands, cloud, vp, ub, inst, app, v=0.0, ortho=False, vols=None, depth=False, bulk=(1, 33)):
    """The instanced kernel with an appearance table against the composed reference (tests/instance_appearance_reference)."""
    ref = ar.frame(cloud, vp, ub, inst, app, v, ortho, vols)
    assert ref["m"] > 0
    for bulk_min in bulk:
        got = emu_project(store, bands, vp, ub, bulk_min, 0, v, ortho, inst, app, vols, depth)
        check(got, ref["records"], ref["unsorted_keys"], ref["unsorted_values"], ref["m"], ref["visible"], ref["last_tile"], vp)
    return ref


def mixed_appearance(inst):
    return [((0.3, 1.0, 2.5), 0.5, None), ((1.0, 1.0, 1.0), 0.75, inst[1][1] // 3 + 1), ((2.0, 0.5, 1.0), 1.0, inst[2][1] - 1), ar.DEFAULT]


@pytest.mark.parametrize("time", [10.0, 0.6], ids=["static", "load_in"])
@pytest.mark.parametrize("bands", [1, 2, 3, 4])
def test_emulated_projection_is_the_oracle_on_the_rounded_cloud(bands, time):
    splat60, vp, ub = scene(time)
    want = rounded(splat60, bands)
    # a store of `bands`, and a 4-band store rendered at degree bands - 1
    check_plain(store_of(splat60, bands), bands, want, vp, ub)
    check_plain(store_of(splat60, 4), bands, want, vp, ub)
    # the rounding is real: the float cloud's colours differ somewhere
    assert not np.array_equal(bits(want[:, 12:12 + 3 * bands * bands]), bits(splat60[:, 12:12 + 3 * bands * bands]))


@pytest.mark.parametrize("bands", [1, 2, 3, 4])
def test_emulated_instances_with_appearance(bands):
    splat60, vp, ub = scene(0.6)
    inst = instances()
    check_instanced(store_of(splat60, 4), bands, rounded(splat60, bands), vp, ub, inst, mixed_appearance(inst))


@pytest.mark.parametrize("mode", ["ortho", "aa_0.3", "ortho_aa_0.1"])
@pytest.mark.parametrize("instanced", [False, True], ids=["default", "instances"])
def test_emulated_orthographic_and_antialiased(mode, instanced):
    splat60, vp, ub = scene(seed=13)
    ortho = mode.startswith("ortho")
    v = {"aa_0.3": 0.3, "ortho_aa_0.1": 0.1}.get(mode, 0.0)
    if ortho:
        vp, _ = oref.ortho_camera(W, H, size=2.5, near=0.5, far=4.5, frame=5)
    store, want = store_of(splat60, 4), rounded(splat60, 4)
    if instanced:
        inst = instances()
        check_instanced(store, 4, want, vp, ub, inst, mixed_appearance(inst), v=v, ortho=ortho)
    else:
        check_plain(store, 4, want, vp, ub, v=v, ortho=ortho)


@pytest.mark.parametrize("instanced", [False, True], ids=["default", "instances"])
def test_emulated_depth_words(instanced):
    splat60, vp, ub = scene(seed=19)
    store, want = store_of(splat60, 3), rounded(splat60, 3)
    if instanced:
        inst = instances()
        check_instanced(store, 3, want, vp, ub, inst, mixed_appearance(inst), depth=True)
    else:
        check_plain(store, 3, want, vp, ub, depth=True)


@pytest.mark.parametrize("kind", ["keep_box", "source"])
def test_emulated_cutouts(kind):
    splat60, vp, ub = scene(seed=17)
    inst = instances()
    vols = crop_set(splat60, kind, frame_positions(splat60, ub, inst), seed=7)
    app = mixed_appearance(inst)
    ref = check_instanced(store_of(splat60, 4), 4, rounded(splat60, 4), vp, ub, inst, app, vols=vols)
    assert 0 < ref["visible"] < ar.frame(rounded(splat60, 4), vp, ub, inst, app)["visible"]


@pytest.mark.parametrize("bands", [1, 2, 3, 4])
def test_emulated_splat_at_the_camera_position(bands):
    splat60, vp, ub = scene()
    u = np.frombuffer(ub, dtype=F32).copy()
    pr = orc.project(splat60, vp, orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8)), cap=64 * N)
    i = int(pr.values[len(pr.values) // 2])
    u[0:3] = splat60[i, 0:3]
    ub = u.tobytes()
    want = rounded(splat60, bands)
    ref = check_plain(store_of(splat60, 4), bands, want, vp, ub)
    assert (ref.records["color"][i, :3] == 0.0).all()   # black at every degree, as the float store draws it
