"""Splat clouds of SH degree 0, 1 and 2 on the GPU (include/gsr.h gsr_config.sh_bands, gsr_upload_ply, gsr_set_sh_degree), through the
C-ABI: a frame drawn at degree d is bit for bit the unchanged oracle's frame of the cloud with the coefficients above d set to zero, for
reduced stores loaded from narrow PLY tables or 60-float structs and for a degree-3 store rendered at a lower degree."""
import ctypes as C

import numpy as np
import pytest

from godotgaussiansplatting_b200 import _lib
from godotgaussiansplatting_b200.ply_file import PlyFile, degree_properties, narrow_table, swizzle_splats
from godotgaussiansplatting_b200.synthetic import synthetic_ply_table
from oracle import oracle as orc
from tests import depth_reference as dref
from tests import instance_reference as iref
from tests.gsr_direct import REC_DTYPE, Ctx
from tests.scenes import make_scene
from tests.test_sh_degree import expected_planes, sh_planes, zero_above, zero_splat_coeffs

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

W, H = 320, 200


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


class ShCtx(Ctx):
    """gsr_direct.Ctx with gsr_config.sh_bands."""

    def __init__(self, max_splats, width, height, sh_bands=0, flags=0, factor=10):
        self.L = _lib.lib()
        self.h = C.c_void_p()
        cfg = _lib.GsrConfig(0, flags, max_splats, factor, sh_bands)
        _lib.check(self.L.gsr_create(C.byref(cfg), C.byref(self.h)), "gsr_create")
        self.max_splats, self.w, self.hgt = max_splats, width, height
        _lib.check(self.L.gsr_resize(self.h, width, height), "gsr_resize")

    def upload_ply(self, table, layout, first=0, creation_time=0.0):
        t = np.ascontiguousarray(table, dtype=np.float32)
        lay = _lib.GsrPlyLayout(layout.nprops, layout.sh_degree, layout.x, layout.f_dc, layout.f_rest, layout.opacity, layout.scale, layout.rot)
        return self.L.gsr_upload_ply(self.h, t.ctypes.data_as(C.POINTER(C.c_float)), C.byref(lay), first, t.shape[0], float(creation_time))

    def degree(self, d):
        return self.L.gsr_set_sh_degree(self.h, d)


def scene(n, seed=2, frame=25):
    t62 = synthetic_ply_table(n, seed)
    t62[:, 55:58] += 0.5
    t62[:, 9:54] += 0.02   # every coefficient non-zero
    _, vp, ub = make_scene(16, 1, W, H, frame=frame)
    return t62, vp, ub


def set_instances(c, inst):
    arr = (_lib.GsrInstance * max(1, len(inst)))()
    for k, (first, count, xf12) in enumerate(inst):
        arr[k].first, arr[k].count = int(first), int(count)
        arr[k].to_frame[:] = [float(v) for v in np.asarray(xf12, dtype=np.float32)]
    _lib.check(c.L.gsr_set_instances(c.h, arr, len(inst)), "gsr_set_instances")


def oracle_frame(splat60, vp, ub, heat=0.0, contract=True, inst=None, scene_depth=None, depth=False):
    u = orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8))
    if inst is not None:
        pr = iref.project(splat60, vp, u, [(f, n) for f, n, _ in inst], np.stack([iref.inverse(x) for _, _, x in inst]))
        recs, keys, vals, vis, m = pr.records, pr.keys, pr.values, pr.visible, pr.duplicates
    else:
        pr = orc.project(splat60, vp, u, cap=64 * splat60.shape[0])
        recs, keys, vals, vis, m = pr.records, pr.keys, pr.values, pr.visible, pr.duplicates
    T = ((W + 15) // 16) * ((H + 15) // 16)
    k, v = orc.sort_pairs(keys, vals)
    b = orc.boundaries(k, T)
    dep = None
    if depth:
        rgba, dep, _ = dref.render_depth(recs, v, b, W, H, vp, scene_depth, heat, contract)
    else:
        orc.set_blend_contraction(contract)
        try:
            rgba, _, _ = orc.render(recs, v, b, W, H, heat)
        finally:
            orc.set_blend_contraction(True)
    return dict(rgba=rgba, records=recs, keys=k, values=v, bounds=b, visible=vis, m=m, depth=dep)


def check(c, rgba, ref, drawn):
    np.testing.assert_array_equal(bits(rgba), bits(ref["rgba"]))
    st = c.stats()
    assert st.duplicates == ref["m"] and st.visible == ref["visible"] and not st.overflow
    m = int(min(st.duplicates, st.capacity))
    T = st.tiles_x * st.tiles_y
    np.testing.assert_array_equal(c.copy(_lib.GSR_BUF_KEYS, m, np.uint32), ref["keys"])
    np.testing.assert_array_equal(c.copy(_lib.GSR_BUF_VALUES, m, np.uint32), ref["values"])
    np.testing.assert_array_equal(c.copy(_lib.GSR_BUF_BOUNDS, T * 2, np.uint32).reshape(T, 2), ref["bounds"])
    recs = c.copy(_lib.GSR_BUF_RECORDS, drawn, REC_DTYPE)
    ids = np.unique(ref["values"])
    np.testing.assert_array_equal(bits(recs[ids].view(np.float32)), bits(ref["records"][ids].view(np.float32)))


@pytest.mark.parametrize("contract", [True, False], ids=["spec", "uncontracted"])
def test_degree_3_and_default_degree_are_the_default_frame(contract):
    n = 12000
    t62, vp, ub = scene(n)
    splat60 = swizzle_splats(t62, 0.0)
    flags = 0 if contract else _lib.GSR_FLAG_UNCONTRACTED_BLEND
    with ShCtx(n, W, H, 0, flags) as a, ShCtx(n, W, H, 4, flags) as b:
        a.upload(splat60)
        b.upload(splat60)
        want = a.render(vp, ub)
        for d in (-1, 3):
            _lib.check(b.degree(d), "gsr_set_sh_degree")
            np.testing.assert_array_equal(bits(b.render(vp, ub)), bits(want))
            for which in (_lib.GSR_BUF_KEYS, _lib.GSR_BUF_VALUES):
                m = int(a.stats().duplicates)
                np.testing.assert_array_equal(b.copy(which, m, np.uint32), a.copy(which, m, np.uint32))


VARIANTS = ["plain", "ragged", "heatmap", "instances", "depth_plane", "uncontracted"]


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("degree", [0, 1, 2])
def test_frames_are_the_zero_padded_oracle(degree, variant):
    n = 12001 if variant == "ragged" else 12288
    t62, vp, ub = scene(n, seed=3 + degree)
    splat60 = swizzle_splats(t62, 0.0)
    padded = zero_splat_coeffs(splat60, degree + 1)
    names = degree_properties(degree, normals=degree != 1, extra=("extra",))
    narrow = np.concatenate([narrow_table(t62, degree, normals=degree != 1), np.ones((n, 1), np.float32)], axis=1)
    layout = PlyFile.from_array(narrow, names).layout()
    flags = _lib.GSR_FLAG_UNCONTRACTED_BLEND if variant == "uncontracted" else 0
    heat = 1.0 if variant == "heatmap" else 0.0
    inst = None
    if variant == "instances":
        from tests.test_instances import SCALED, rigid
        inst = [(0, 5000, rigid(4)), (4000, 6000, SCALED), (n - 301, 301, rigid(5))]
    Z = None
    if variant == "depth_plane":
        u = orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8))
        pr = orc.project(padded, vp, u, cap=64 * n)
        V = np.asarray(vp, dtype=np.float32)
        r = pr.records[np.unique(pr.values)]
        d = -(((V[2] * r["pos_xy"][:, 0] + V[6] * r["pos_xy"][:, 1]) + V[10] * r["pos_z"]) + V[14] * np.float32(1.0))
        Z = np.full((H, W), np.inf, dtype=np.float32)
        Z[:, W // 2:] = np.median(d)
    ref = oracle_frame(padded, vp, ub, heat, flags == 0, inst, Z, Z is not None)
    assert ref["visible"] > 0
    for how in ("ply", "aos", "degree"):
        with ShCtx(n, W, H, degree + 1 if how != "degree" else 4, flags) as c:
            if how == "ply":
                _lib.check(c.upload_ply(narrow, layout), "gsr_upload_ply")
            elif how == "aos":
                c.upload(splat60)
            else:
                c.upload(splat60)
                _lib.check(c.degree(degree), "gsr_set_sh_degree")
            depth = None
            if Z is not None:
                Zt = torch.from_numpy(Z).cuda()
                depth = torch.zeros((H, W), dtype=torch.float32, device="cuda")
                torch.cuda.synchronize()
                _lib.check(c.L.gsr_set_depth_compositing(c.h, C.c_void_p(Zt.data_ptr()), C.c_void_p(depth.data_ptr())), "depth")
            if inst is not None:
                set_instances(c, inst)
            rgba = c.render(vp, ub, heatmap=heat)
            check(c, rgba, ref, iref.layout([(f, k) for f, k, _ in inst])[1] if inst else n)
            if depth is not None:
                c.sync()
                np.testing.assert_array_equal(bits(depth.cpu().numpy()), bits(ref["depth"]))


@pytest.mark.parametrize("bands", [1, 2, 3, 4])
def test_stored_planes_are_the_emulated_ingest(bands):
    n = 3000
    stride = (n + 255) // 256 * 256
    t62, _, _ = scene(n)
    splat60 = swizzle_splats(t62, 0.0)
    with ShCtx(n, W, H, bands) as c:
        c.upload(splat60)
        size = (3 + sh_planes(bands)) * stride * 4
        got = c.copy(_lib.GSR_BUF_SPLATS, size, np.float32).reshape(3 + sh_planes(bands), stride, 4)
        np.testing.assert_array_equal(bits(got), bits(expected_planes(splat60, bands, stride)))
        assert _lib.GSR_BUF_SPLATS == 10
        big = np.empty(size * 4 + 1, dtype=np.uint8)
        assert c.L.gsr_debug_copy(c.h, _lib.GSR_BUF_SPLATS, C.c_void_p(big.ctypes.data), big.nbytes) == _lib.GSR_ERR_INVALID
        # the standard PLY path gives the same planes, and a degree-1 file the zero-padded ones
        _lib.check(c.L.gsr_upload_ply_raw(c.h, t62.ctypes.data_as(C.POINTER(C.c_float)), 62, 0, n, 0.0), "gsr_upload_ply_raw")
        np.testing.assert_array_equal(bits(c.copy(_lib.GSR_BUF_SPLATS, size, np.float32)), bits(got.reshape(-1)))
        narrow = narrow_table(t62, 1, normals=False)
        _lib.check(c.upload_ply(narrow, PlyFile.from_array(narrow, degree_properties(1, False)).layout()), "gsr_upload_ply")
        want = expected_planes(swizzle_splats(zero_above(t62, min(1, bands - 1)), 0.0), bands, stride)
        np.testing.assert_array_equal(bits(c.copy(_lib.GSR_BUF_SPLATS, size, np.float32)), bits(want.reshape(-1)))


@pytest.mark.parametrize("overlap", [0, 1], ids=["serial", "overlap"])
def test_degree_changes_between_async_frames(overlap):
    n = 12288
    t62, vp, ub = scene(n, seed=9)
    splat60 = swizzle_splats(t62, 0.0)
    degrees = [3, 0, 2, -1, 1, 0]
    with ShCtx(n, W, H, 4) as c:
        c.upload(splat60)
        _lib.check(c.L.gsr_debug_pipeline(c.h, overlap), "gsr_debug_pipeline")
        hosts = [torch.empty((H, W, 4), dtype=torch.float32, pin_memory=True) for _ in degrees]
        for d, hb in zip(degrees, hosts):
            _lib.check(c.degree(d), "gsr_set_sh_degree")
            c.render_async(vp, ub, host_ptr=hb.data_ptr())
        c.sync()
        for d, hb in zip(degrees, hosts):
            ref = oracle_frame(zero_splat_coeffs(splat60, 4 if d < 0 else d + 1), vp, ub)
            np.testing.assert_array_equal(bits(hb.numpy()), bits(ref["rgba"]), err_msg=f"degree {d}")


def test_state_rules_and_invalid_input():
    n = 4096
    t62, vp, ub = scene(n)
    L = _lib.lib()
    h = C.c_void_p()
    assert L.gsr_create(C.byref(_lib.GsrConfig(0, 0, n, 10, 5)), C.byref(h)) == _lib.GSR_ERR_INVALID and not h.value
    blob = (C.c_ubyte * _lib.GSR_GROUP_BLOB_BYTES)()
    handles = (C.c_ubyte * 128)()
    with ShCtx(n, W, H, 2) as c:   # a reduced store: single-context only
        assert c.degree(2) == _lib.GSR_ERR_INVALID and c.degree(-2) == _lib.GSR_ERR_INVALID
        _lib.check(c.degree(0), "degree 0")
        _lib.check(c.degree(-1), "degree -1")
        assert L.gsr_set_band(c.h, 0, 3) == _lib.GSR_ERR_STATE
        assert L.gsr_set_row_interleave(c.h, 0, 2) == _lib.GSR_ERR_STATE
        assert L.gsr_group_export(c.h, blob) == _lib.GSR_ERR_STATE
        assert L.gsr_peer_export_framebuffers(c.h, handles) == _lib.GSR_ERR_STATE
        _lib.check(L.gsr_set_band(c.h, 0, (H + 15) // 16), "full band")
        _lib.check(L.gsr_set_row_interleave(c.h, 0, 1), "row_mod 1")
        lay = _lib.GsrPlyLayout(17, 0, 0, 6, -1, 9, 10, 13)
        t = np.zeros((4, 17), np.float32)
        tp = t.ctypes.data_as(C.POINTER(C.c_float))
        _lib.check(L.gsr_upload_ply(c.h, tp, C.byref(lay), 0, 4, 0.0), "degree-0 layout")
        for bad in (dict(nprops=0), dict(nprops=257), dict(sh_degree=4), dict(f_rest=3), dict(rot=14), dict(x=-1), dict(sh_degree=1)):
            b = _lib.GsrPlyLayout(17, 0, 0, 6, -1, 9, 10, 13)
            for k, v in bad.items():
                setattr(b, k, v)
            assert L.gsr_upload_ply(c.h, tp, C.byref(b), 0, 4, 0.0) == _lib.GSR_ERR_INVALID, bad
        assert L.gsr_upload_ply(c.h, tp, None, 0, 4, 0.0) == _lib.GSR_ERR_INVALID
        assert L.gsr_upload_ply(c.h, tp, C.byref(lay), n - 2, 4, 0.0) == _lib.GSR_ERR_INVALID
    with ShCtx(n, W, H, 4) as c:   # a degree-3 store: the rules apply while a lower degree is set
        _lib.check(L.gsr_set_band(c.h, 0, 3), "band")
        assert c.degree(1) == _lib.GSR_ERR_STATE
        _lib.check(c.degree(3), "degree 3 with a band")
        _lib.check(L.gsr_set_band(c.h, 0, (H + 15) // 16), "full band")
        _lib.check(L.gsr_set_row_interleave(c.h, 0, 2), "row interleave")
        assert c.degree(0) == _lib.GSR_ERR_STATE
        _lib.check(L.gsr_set_row_interleave(c.h, 0, 1), "row_mod 1")
        _lib.check(c.degree(0), "degree 0")
        assert L.gsr_set_band(c.h, 0, 3) == _lib.GSR_ERR_STATE
        assert L.gsr_group_export(c.h, blob) == _lib.GSR_ERR_STATE
        assert L.gsr_peer_export_framebuffers(c.h, handles) == _lib.GSR_ERR_STATE
        _lib.check(c.degree(-1), "back to degree 3")
        _lib.check(L.gsr_group_export(c.h, blob), "group export")
