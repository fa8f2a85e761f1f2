"""Splat selection without a GPU (include/gsr.h "Splat selection"): the emulated selection kernels of selection.cu and the emulated CUT
projection kernels with splat masks, bit for bit against the numpy rules and the composed reference of tests/selection_reference, and the
mask packing of the Python mirror."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from godotgaussiansplatting_b200.rasterizer import pack_mask, unpack_mask
from oracle import oracle as orc
from tests import cutout_reference as cr
from tests import depth_order_reference as dor
from tests import instance_reference as iref
from tests import ortho_reference as oref
from tests import selection_reference as sref
from tests.test_depth_order import H, W, scene
from tests.test_instances import rigid
from tests.test_orthographic import store_of

F32, U32 = np.float32, np.uint32
HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "selection_reference")
_emu = None


def emu():
    global _emu
    if _emu is None:
        out_dir = HERE if os.access(HERE, os.W_OK) else tempfile.mkdtemp(prefix="gsr_selection_emu_")
        out = os.path.join(out_dir, "libselection_emu.so")
        deps = [os.path.join(HERE, "selection_emu.cpp")] + cr._EMU_DEPS[1:] + [os.path.join(cr.CSRC, "selection.cu")]
        if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(d) for d in deps):
            tmp = f"{out}.{os.getpid()}.tmp"
            subprocess.run([os.environ.get("ORC_CXX", "/usr/bin/g++")] + cr._EMU_FLAGS + ["-I", cr.CUDA_INC, deps[0], "-o", tmp], check=True)
            os.replace(tmp, out)
        L = C.CDLL(out)
        vp = C.c_void_p
        L.emu_selection_projection.restype = C.c_longlong
        L.emu_selection_projection.argtypes = [C.c_int, C.c_int, C.c_int, C.c_float, vp, C.c_ulonglong, C.c_uint, vp, vp, C.c_int, vp, vp, vp,
                                               C.c_uint, C.POINTER(C.c_uint), C.POINTER(C.c_int), vp, vp, vp, vp, vp, vp, C.c_float, vp, C.c_int]
        L.emu_select_region.argtypes = [C.c_int, vp, vp, C.c_uint, C.c_uint, C.c_ulonglong, C.c_ulonglong, C.c_ulonglong, vp, C.c_float, vp,
                                        vp, C.c_float, C.c_float, vp, C.c_int, C.c_uint, vp]
        _emu = L
    return _emu


def ptr(a):
    return None if a is None else a.ctypes.data


def plane0(splat60, n):
    p = np.zeros((n, 4), dtype=F32)
    s = np.asarray(splat60, dtype=F32)
    p[:s.shape[0], 0:3] = s[:, 0:3]
    p[:s.shape[0], 3] = s[:, 3]
    return p


def emu_region(kind, sel, hid, op, p0, vp=None, wh=(W, H), instance=None, vol=None, xy=None, ms=1.0):
    n = sel.size
    s, h = pack_mask(sel, n), pack_mask(hid, n)
    first, count, A = (0, n, None) if instance is None else (instance[0], instance[1], np.asarray(instance[2], dtype=F32))
    vp32 = None if vp is None else np.ascontiguousarray(vp, dtype=F32)
    c12 = None if vol is None else np.asarray(vol[0], dtype=F32)
    xy32 = None if xy is None else np.ascontiguousarray(xy, dtype=F32)
    emu().emu_select_region(kind, ptr(s), ptr(h), s.size, op, n, first, count, ptr(p0), ms, ptr(A), ptr(vp32), F32(wh[0] - 1), F32(wh[1] - 1),
                            ptr(c12), 0 if vol is None else vol[1] | (vol[3] << 1), 0 if xy is None else xy32.shape[0], ptr(xy32))
    return unpack_mask(s, n)


# ---- the region kernels against the rules ---------------------------------------------------------------------------------------
CONVEX = np.array([[20, 20], [140, 10], [150, 80], [30, 90]], dtype=F32)
CONCAVE = np.array([[10, 10], [150, 10], [80, 40], [150, 80], [10, 80], [60, 45]], dtype=F32)
STAR = np.array([[80, 2], [110, 88], [10, 30], [150, 30], [50, 88]], dtype=F32)
RECT = np.array([[0, 0], [W - 1, 0], [W - 1, 44], [0, 44]], dtype=F32)


@pytest.mark.parametrize("shape", ["convex", "concave", "star", "rect", "on_py"])
@pytest.mark.parametrize("op", [sref.SET, sref.ADD, sref.SUBTRACT, sref.TOGGLE])
def test_polygon_kernel_is_the_rule(shape, op):
    splat60, vp, ub = scene()
    n = splat60.shape[0] + 45   # past the upload: zero splats, and max_splats not a multiple of 32
    p0 = plane0(splat60, n)
    rng = np.random.default_rng(op)
    hid = rng.random(n) < 0.2
    sel = (rng.random(n) < 0.4) & ~hid
    xy = dict(convex=CONVEX, concave=CONCAVE, star=STAR, rect=RECT)[shape] if shape != "on_py" else None
    if shape == "on_py":   # vertices exactly on splats' projected rows, and a horizontal edge through one
        x, y, _ = sref.mref.pix(vp, p0[:, 0], p0[:, 1], p0[:, 2], W, H)
        ok = np.flatnonzero((x > 20) & (x < W - 20) & (y > 20) & (y < H - 20))[:3]
        xy = np.array([[5, y[ok[0]]], [x[ok[1]], y[ok[1]]], [W - 5, y[ok[1]]], [W - 5, H - 5], [x[ok[2]], y[ok[0]]]], dtype=F32)
    inside = sref.polygon_set(splat60, n, vp, W, H, xy)
    got = emu_region(1, sel, hid, op, p0, vp=vp, xy=xy)
    np.testing.assert_array_equal(got, sref.combine(op, sel, inside, hid))
    assert 0 < inside.sum() < n


def test_polygon_behind_the_camera_and_orthographic():
    splat60, vp, ub = scene()
    n = splat60.shape[0]
    V = np.asarray(vp, dtype=np.float64)[:16]
    eye = -np.array([sum(V[4 * j + r] * V[12 + r] for r in range(3)) for j in range(3)])
    back = np.array([V[2], V[6], V[10]])   # the camera's +z axis: behind it
    splat60 = splat60.copy()
    splat60[:200, 0:3] = (eye + (1.0 + np.arange(200)[:, None] * 0.01) * back).astype(F32)
    p0 = plane0(splat60, n)
    everything = np.array([[-1e6, -1e6], [1e6, -1e6], [1e6, 1e6], [-1e6, 1e6]], dtype=F32)
    inside = sref.polygon_set(splat60, n, vp, W, H, everything)
    x, y, w = sref.mref.pix(vp, p0[:, 0], p0[:, 1], p0[:, 2], W, H)
    assert (~(w > 0)).any() and not inside[~(w > 0)].any()   # behind the camera: never inside
    np.testing.assert_array_equal(emu_region(1, np.zeros(n, bool), np.zeros(n, bool), sref.SET, p0, vp=vp, xy=everything), inside)
    ovp, oub = oref.ortho_camera(W, H, size=2.6, near=0.5, far=4.5, frame=25)
    inside = sref.polygon_set(splat60, n, ovp, W, H, CONCAVE)
    assert 0 < inside.sum() < n
    np.testing.assert_array_equal(emu_region(1, np.zeros(n, bool), np.zeros(n, bool), sref.ADD, p0, vp=ovp, xy=CONCAVE), inside)


@pytest.mark.parametrize("shape", [cr.BOX, cr.ELLIPSOID])
@pytest.mark.parametrize("space", [cr.FRAME, cr.SOURCE])
@pytest.mark.parametrize("inst", [None, (37, 901), (64, 96), (1, 31)])
def test_volume_kernel_and_instance_ranges(shape, space, inst):
    splat60, vp, ub = scene()
    n = splat60.shape[0] + 13
    p0 = plane0(splat60, n)
    rng = np.random.default_rng(3)
    hid = rng.random(n) < 0.1
    sel = (rng.random(n) < 0.5) & ~hid
    vol = cr.box([0.1, 0.0, 0.1], [0.4, 0.6, 0.5], shape, space=space)
    instance = None if inst is None else (inst[0], inst[1], rigid(2))
    for op in (sref.SET, sref.TOGGLE):
        inside = sref.volume_set(splat60, n, vol[0], vol[1], vol[3], instance=instance)
        got = emu_region(2, sel, hid, op, p0, vol=vol, instance=instance)
        np.testing.assert_array_equal(got, sref.combine(op, sel, inside, hid))
        if op == sref.SET and inst is not None:   # SET clears every splat outside the tested range
            out = np.ones(n, bool)
            out[inst[0]:inst[0] + inst[1]] = False
            assert not got[out].any()
    np.testing.assert_array_equal(emu_region(0, sel, hid, sref.TOGGLE, p0), (sel ^ np.ones(n, bool)) & ~hid)


# ---- the CUT projection with masks against the composed reference ------------------------------------------------------------
def emu_frame(splat60, vp, ub, hid, sel, style, inst=None, ortho=False, bands=4, v=0.0, vols=None):
    store = store_of(splat60, bands)
    stride = store.shape[1]
    n = splat60.shape[0]
    frame_c = desc = warp_inst = None
    num = n
    if inst is not None:
        ranges = [(f, c) for f, c, _ in inst]
        w0, D = iref.layout(ranges)
        u = orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8))
        xf = [iref.inverse(x) for _, _, x in inst]
        frame_c = np.zeros((len(ranges), 32), dtype=F32)
        for k in range(len(ranges)):
            Vk, camk = iref.compose(vp[:16], u.camera_pos[:], xf[k])
            frame_c[k, :16], frame_c[k, 16:19], frame_c[k, 19:31] = Vk, camk, xf[k][:12]
        warp_inst = np.full(((D + 255) // 256) * 8 + 1, 0xFFFFFFFF, dtype=U32)
        for k, (_, c) in enumerate(ranges):
            warp_inst[w0[k]:w0[k] + (c + 31) // 32] = k
        desc = np.zeros(len(ranges), dtype=np.dtype([("first", "<u8"), ("count", "<u4"), ("warp0", "<u4")]))
        for k, (f, c) in enumerate(ranges):
            desc[k] = (f, c, w0[k])
        num = D
    cap = 64 * num
    recs = np.zeros(num, dtype=orc.RECORD_DTYPE)
    keys, vals = np.zeros(cap, U32), np.zeros(cap, U32)
    k, h, on = sref.highlight(style)
    hw, sw = pack_mask(hid, n), pack_mask(sel, n)
    vis, last = C.c_uint(0), C.c_int(-1)
    vp32 = np.ascontiguousarray(vp, dtype=F32)
    ubuf = np.frombuffer(ub, dtype=np.uint8).copy()
    args = None if vols is None else np.array([cr.cutout_args(vols)], dtype=cr.ARGS_DTYPE)
    m = emu().emu_selection_projection(int(inst is not None), bands, int(ortho), v, ptr(store), stride, num, ptr(vp32), ptr(ubuf), 12, ptr(recs),
                                       ptr(keys), ptr(vals), cap, C.byref(vis), C.byref(last), ptr(frame_c), ptr(desc), ptr(warp_inst), ptr(args),
                                       ptr(hw), ptr(sw), float(k), ptr(np.ascontiguousarray(h)), int(on))
    assert m >= 0
    return recs, keys[:m], vals[:m], int(vis.value), int(last.value)


@pytest.mark.parametrize("case", ["plain", "instances", "orthographic", "highlight_off", "empty"])
def test_emulated_projection_is_the_reference(case):
    splat60, vp, ub = scene()
    ortho = case == "orthographic"
    if ortho:
        vp, ub = oref.ortho_camera(W, H, size=2.6, near=0.5, far=4.5, frame=25)
    n = splat60.shape[0]
    rng = np.random.default_rng(7)
    hid = rng.random(n) < 0.3
    sel = (rng.random(n) < 0.2) & ~hid
    if case == "empty":
        hid[:], sel[:] = False, False
    st = ((0.3, 1.0, 2.0), 0.0 if case == "highlight_off" else 0.45)
    inst = [(3, 700, rigid(3)), (100, 999, rigid(4)), (0, 33, rigid(5))] if case == "instances" else None
    u = orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8))
    pr = dor.project(splat60, vp, u, 0.0, ortho, inst)
    ref = sref.oracle_frame(splat60, vp, ub, hid, sel, st, inst=inst, ortho=ortho)
    keep = ref["mask"][pr.values.astype(np.int64)]
    recs, keys, vals, vis, last = emu_frame(splat60, vp, ub, hid, sel, st, inst, ortho)
    np.testing.assert_array_equal(keys, pr.keys[keep])
    np.testing.assert_array_equal(vals, pr.values[keep])
    assert vis == ref["visible"] and last == ref["last_tile"]
    ids = np.unique(vals)
    np.testing.assert_array_equal(recs[ids].view(F32).view(U32), ref["records"][ids].view(F32).view(U32))
    if case in ("empty", "highlight_off"):   # the default records, bit for bit
        drawn = ids if case == "empty" else ids[~np.isin(ids, np.flatnonzero(hid))]
        np.testing.assert_array_equal(recs[drawn].view(U32), pr.records[drawn].view(U32))
    if case == "plain":
        assert sel[ids].sum() > 20 and len(ids) > 200


@pytest.mark.parametrize("bands", [1, 2, 3])
@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("cut", [False, True])
@pytest.mark.parametrize("inst", [False, True])
def test_emulated_projection_with_features(bands, aa, cut, inst):
    """The masks and the highlight with reduced SH bands, anti-aliasing and a cutout set (KEEP box + REMOVE ellipsoid), with and
    without instances: hidden splats and cutout volumes together, the highlight after the reduced-degree colour."""
    from tests.test_sh_degree import zero_splat_coeffs
    from tests import variant_matrix as vm
    splat60, vp, ub = scene()
    n = splat60.shape[0]
    rng = np.random.default_rng(bands * 8 + aa * 4 + cut * 2 + inst)
    hid = rng.random(n) < 0.25
    sel = (rng.random(n) < 0.3) & ~hid
    st = ((0.5, 2.0, 0.0), 0.3)
    v = 0.3 if aa else 0.0
    layout = [(3, 700, rigid(3)), (100, 999, rigid(4)), (0, 33, rigid(5))] if inst else None
    vols = vm.cutouts(splat60, cr.positions(splat60, 1.0, layout)[1]) if cut else None
    src = zero_splat_coeffs(splat60, bands)
    u = orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8))
    pr = dor.project(src, vp, u, v, False, layout)
    ref = sref.oracle_frame(src, vp, ub, hid, sel, st, vols or (), layout, v=v)
    keep = ref["mask"][pr.values.astype(np.int64)]
    recs, keys, vals, vis, last = emu_frame(splat60, vp, ub, hid, sel, st, layout, False, bands, v, vols)
    np.testing.assert_array_equal(keys, pr.keys[keep])
    np.testing.assert_array_equal(vals, pr.values[keep])
    assert vis == ref["visible"] and last == ref["last_tile"]
    ids = np.unique(vals)
    np.testing.assert_array_equal(recs[ids].view(F32).view(U32), ref["records"][ids].view(F32).view(U32))
    src_of = sref.drawn_sources(n, None if layout is None else [(f, c) for f, c, _ in layout])
    assert sel[src_of[ids]].sum() > 20
    if cut:   # both rules removed splats: some ids are hidden-only, some cut-only
        cut_mask = cr.drawn_mask(vols, *cr.positions(splat60, 1.0, layout))[:src_of.size]
        emitted_before = np.unique(pr.values)
        valid = src_of[emitted_before] >= 0
        e = emitted_before[valid]
        assert (~cut_mask[e] & ~hid[src_of[e]]).any() and (cut_mask[e] & hid[src_of[e]]).any()


def test_mask_packing():
    for n in (1, 31, 32, 33, 1000):
        m = np.random.default_rng(n).random(n) < 0.5
        w = pack_mask(m, n)
        assert w.size == (n + 31) // 32
        np.testing.assert_array_equal(unpack_mask(w, n), m)
        for s in range(n):
            assert bool((int(w[s >> 5]) >> (s & 31)) & 1) == m[s]
