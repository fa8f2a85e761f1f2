"""Depth-ordered frames on the GPU (include/gsr.h gsr_set_depth_order), through the C-ABI: every mode-1 frame is bit for bit the
depth-order oracle's (tests/depth_order_reference) in sorted pairs, tile bounds, RGBA and depth; the projection's depth words are the
oracle's; tile ranges of a large frame are in view-depth order; the mode follows the frames it was enqueued with; the single-context
rules hold; and the Python mirror sets it."""
import ctypes as C

import numpy as np
import pytest

from godotgaussiansplatting_b200 import _lib
from godotgaussiansplatting_b200 import camera as cam
from godotgaussiansplatting_b200.ply_file import PlyFile, swizzle_splats
from godotgaussiansplatting_b200.rasterizer import GaussianSplattingRasterizer
from godotgaussiansplatting_b200.synthetic import synthetic_ply_table
from oracle import oracle as orc
from tests import depth_order_reference as dor
from tests import depth_reference as dref
from tests import ortho_reference as oref
from tests.gsr_direct import REC_DTYPE
from tests.scenes import make_scene
from tests.test_gpu_sh_degree import ShCtx, set_instances
from tests.test_sh_degree import zero_splat_coeffs

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

W, H = 320, 200
VIEW = _lib.GSR_DEPTH_ORDER_VIEW_DEPTH


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def cloud(n, seed=3):
    t62 = synthetic_ply_table(n, seed)
    t62[:, 55:58] += 0.5
    t62[:, 9:54] += 0.02
    return swizzle_splats(t62, 0.0)


def view(width=W, height=H, frame=25):
    _, vp, ub = make_scene(16, 1, width, height, frame=frame)
    return vp, ub


def order(c, mode):
    return c.L.gsr_set_depth_order(c.h, mode)


def check(c, rgba, ref, drawn, overflow=False):
    np.testing.assert_array_equal(bits(rgba), bits(ref["rgba"]))
    st = c.stats()
    assert st.duplicates == ref["m"] and st.visible == ref["visible"] and bool(st.overflow) == overflow
    m = int(min(st.duplicates, st.capacity))
    T = st.tiles_x * st.tiles_y
    np.testing.assert_array_equal(c.copy(_lib.GSR_BUF_KEYS, m, np.uint32), ref["keys"])
    np.testing.assert_array_equal(c.copy(_lib.GSR_BUF_VALUES, m, np.uint32), ref["values"])
    np.testing.assert_array_equal(c.copy(_lib.GSR_BUF_BOUNDS, T * 2, np.uint32).reshape(T, 2), ref["bounds"])
    recs = c.copy(_lib.GSR_BUF_RECORDS, drawn, REC_DTYPE)
    ids = np.unique(ref["values"])
    np.testing.assert_array_equal(bits(recs[ids].view(np.float32)), bits(ref["records"][ids].view(np.float32)))


VARIANTS = ["plain", "heatmap", "uncontracted", "instances", "orthographic", "aa_0.3", "aa_0.1", "reduced_store", "ragged"]


@pytest.mark.parametrize("variant", VARIANTS)
def test_frames_are_the_depth_order_oracle(variant):
    n = 12288
    splat60 = cloud(n)
    w, h = (321, 181) if variant == "ragged" else (W, H)
    ortho = variant == "orthographic"
    vp, ub = oref.ortho_camera(w, h, size=2.6, near=0.5, far=4.5, frame=25) if ortho else view(w, h)
    v = {"aa_0.3": 0.3, "aa_0.1": 0.1}.get(variant, 0.0)
    flags = (_lib.GSR_FLAG_UNCONTRACTED_BLEND if variant == "uncontracted" else 0) | (_lib.GSR_FLAG_ORTHOGRAPHIC if ortho else 0)
    heat = 1.0 if variant == "heatmap" else 0.0
    bands = 2 if variant == "reduced_store" else 0
    src = zero_splat_coeffs(splat60, 2) if bands else splat60
    inst = None
    if variant == "instances":   # overlapping and repeated ranges
        from tests.test_instances import SCALED, rigid
        inst = [(0, 5000, rigid(4)), (4000, 6000, SCALED), (n - 301, 301, rigid(5)), (0, 5000, rigid(6))]
    ref = dor.oracle_frame(src, vp, ub, v, ortho, heat, contract=variant != "uncontracted", inst=inst)
    assert ref["visible"] > 1000
    with ShCtx(n, w, h, bands, flags) as c:
        c.upload(splat60)
        if inst is not None:
            set_instances(c, inst)
        if v:
            _lib.check(c.L.gsr_set_antialiasing(c.h, C.c_float(v)), "gsr_set_antialiasing")
        _lib.check(order(c, VIEW), "gsr_set_depth_order")
        check(c, c.render(vp, ub, heatmap=heat), ref, len(ref["records"]))
        if variant == "plain":   # more orbit frames on the same context
            for f in (3, 40, 77):
                vpf, ubf = view(frame=f)
                check(c, c.render(vpf, ubf), dor.oracle_frame(splat60, vpf, ubf), n)


def tied_scene():
    from tests.test_depth_order import H as h, W as w, tied_pair
    s, vp, ub, d = tied_pair()
    return s, vp, ub, d, w, h


@pytest.mark.parametrize("mode", [0, 1])
def test_depth_compositing_with_a_plane_between_tied_splats(mode):
    """The scene depth lies between two splats that tie in the 16-bit key: the default order draws the far one first, whose depth is not
    in front of the scene, so the pixel stops and the near splat is lost; the view-depth order blends the near one first."""
    s, vp, ub, d, w, h = tied_scene()
    Z = np.full((h, w), (float(d[0]) + float(d[1])) * 0.5, dtype=np.float32)
    assert d[1] < Z[0, 0] < d[0]
    if mode:
        ref = dor.oracle_frame(s, vp, ub, scene_depth=Z)
    else:
        u = orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8))
        pr = orc.project(s, vp, u, cap=4096)
        k, vals = orc.sort_pairs(pr.keys, pr.values)
        b = orc.boundaries(k, ((w + 15) // 16) * ((h + 15) // 16))
        rgba, dep, _ = dref.render_depth(pr.records, vals, b, w, h, vp, Z)
        ref = dict(rgba=rgba, depth=dep)
    centre = ref["rgba"][h // 2, w // 2]
    if mode:
        assert centre[0] > 0.8 and centre[3] > 0.8, centre   # the near red splat
    else:
        assert centre[3] == 0.0, centre                       # nothing: the pixel stopped at the far splat
    with ShCtx(2, w, h) as c:
        c.upload(s)
        Zt = torch.from_numpy(Z).cuda()
        depth = torch.zeros((h, w), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        _lib.check(c.L.gsr_set_depth_compositing(c.h, C.c_void_p(Zt.data_ptr()), C.c_void_p(depth.data_ptr())), "depth")
        _lib.check(order(c, mode), "gsr_set_depth_order")
        rgba = c.render(vp, ub)
        c.sync()
        np.testing.assert_array_equal(bits(rgba), bits(ref["rgba"]))
        np.testing.assert_array_equal(bits(depth.cpu().numpy()), bits(ref["depth"]))


def test_first_frame_overflows_and_grows():
    from tests.test_instances import rigid
    n = 4096
    splat60, vp, ub = make_scene(n, 3, W, H, frame=5, scale_boost=0.5)
    inst = [(0, n, rigid(30 + k, 0.3, 0.5)) for k in range(6)]   # D = 6 N
    ref = dor.oracle_frame(splat60, vp, ub, inst=inst)
    with ShCtx(n, W, H, 0, 0, factor=1) as c:
        c.upload(splat60)
        set_instances(c, inst)
        _lib.check(order(c, VIEW), "gsr_set_depth_order")
        rgba = c.render(vp, ub)   # overflows the initial capacity: grows (depth words too) and renders again
        check(c, rgba, ref, len(ref["records"]))


def test_static_capacity_truncates_to_the_emission_prefix():
    n = 12288
    splat60 = cloud(n, seed=4)
    vp, ub = view()
    with ShCtx(n, W, H, 0, _lib.GSR_FLAG_STATIC_CAPACITY, factor=1) as c:
        c.upload(splat60)
        _lib.check(order(c, VIEW), "gsr_set_depth_order")
        c.L.gsr_render(c.h, np.ascontiguousarray(vp, dtype=np.float32).ctypes.data_as(C.POINTER(C.c_float)), ub, 0.0, None)
        cap = int(c.stats().capacity)
        ref = dor.oracle_frame(splat60, vp, ub, cap=cap)
        assert ref["m"] > cap
        out = np.empty((H, W, 4), dtype=np.float32)
        rc = c.L.gsr_render(c.h, np.ascontiguousarray(vp, dtype=np.float32).ctypes.data_as(C.POINTER(C.c_float)), ub, 0.0,
                            C.c_void_p(out.ctypes.data))
        assert rc in (_lib.GSR_OK, _lib.GSR_ERR_OVERFLOW)
        check(c, out, ref, n, overflow=True)


def test_unsorted_depth_words_are_the_oracles():
    n = 12288
    splat60 = cloud(n, seed=5)
    vp, ub = view()
    ref = dor.oracle_frame(splat60, vp, ub)
    with ShCtx(n, W, H) as c:
        c.upload(splat60)
        c.keep_unsorted()
        _lib.check(order(c, VIEW), "gsr_set_depth_order")
        c.render(vp, ub)
        m = ref["m"]
        np.testing.assert_array_equal(c.copy(_lib.GSR_BUF_DEPTH_WORDS_UNSORTED, m, np.uint32), ref["unsorted_words"])
        np.testing.assert_array_equal(c.copy(_lib.GSR_BUF_KEYS_UNSORTED, m, np.uint32),
                                      orc.project(splat60, vp, orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8)), cap=64 * n).keys)


def test_large_scene_tile_ranges_are_in_view_depth_order():
    n, w, h = 1_500_000, 1280, 720
    splat60, vp, ub = make_scene(n, 7, w, h, frame=12)
    with ShCtx(n, w, h) as c:
        c.upload(splat60)
        c.render(vp, ub, readback=False)
        s0 = c.stats()
        T = s0.tiles_x * s0.tiles_y
        b0 = c.copy(_lib.GSR_BUF_BOUNDS, T * 2, np.uint32).reshape(T, 2)
        _lib.check(order(c, VIEW), "gsr_set_depth_order")
        c.render(vp, ub, readback=False)
        s1 = c.stats()
        assert (s1.duplicates, s1.visible, s1.capacity) == (s0.duplicates, s0.visible, s0.capacity) and s1.duplicates > 1_000_000
        np.testing.assert_array_equal(c.copy(_lib.GSR_BUF_BOUNDS, T * 2, np.uint32).reshape(T, 2), b0)
        m = int(s1.duplicates)
        keys = c.copy(_lib.GSR_BUF_KEYS, m, np.uint32)
        vals = c.copy(_lib.GSR_BUF_VALUES, m, np.uint32)
        recs = c.copy(_lib.GSR_BUF_RECORDS, n, REC_DTYPE)
    d = dor.view_depth(recs, vals, vp)
    tile = keys >> np.uint32(16)
    assert np.all(np.diff(tile.astype(np.int64)) >= 0)
    same = tile[1:] == tile[:-1]
    assert np.all(d[1:][same] >= d[:-1][same])                            # non-decreasing d inside every tile
    tie = same & (d[1:] == d[:-1])
    assert np.all(vals[1:][tie] > vals[:-1][tie])                          # equal d: id order


@pytest.mark.parametrize("overlap", [0, 1], ids=["serial", "overlap"])
def test_mode_changes_between_async_frames(overlap):
    n = 12288
    splat60 = cloud(n, seed=9)
    modes = [0, 1, 1, 0, 1, 0]
    frames = [view(frame=20 + k) for k in range(len(modes))]
    with ShCtx(n, W, H) as c, ShCtx(n, W, H) as never:
        c.upload(splat60)
        never.upload(splat60)
        for x in (c, never):
            _lib.check(x.L.gsr_debug_pipeline(x.h, overlap), "gsr_debug_pipeline")
        hosts = [torch.empty((H, W, 4), dtype=torch.float32, pin_memory=True) for _ in frames]
        for mode, (vp, ub), hb in zip(modes, frames, hosts):
            _lib.check(order(c, mode), "gsr_set_depth_order")
            c.render_async(vp, ub, host_ptr=hb.data_ptr())
        c.sync()
        vp, ub = frames[-1]
        want = never.render(vp, ub)
        m = int(never.stats().duplicates)
        np.testing.assert_array_equal(bits(c.render(vp, ub)), bits(want))   # back in mode 0: byte for byte a context that never switched
        for which in (_lib.GSR_BUF_KEYS, _lib.GSR_BUF_VALUES):
            np.testing.assert_array_equal(c.copy(which, m, np.uint32), never.copy(which, m, np.uint32))
    for k, (mode, (vp, ub), hb) in enumerate(zip(modes, frames, hosts)):
        if mode:
            want = dor.oracle_frame(splat60, vp, ub)["rgba"]
        else:
            want = orc.frame(splat60, vp, orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8)), cap=64 * n).rgba
        np.testing.assert_array_equal(bits(hb.numpy()), bits(want), err_msg=f"frame {k}")


def test_state_rules_and_invalid_modes():
    n = 4096
    splat60 = cloud(n)
    vp, ub = view()
    handles = (C.c_ubyte * 128)()
    blob = (C.c_ubyte * _lib.GSR_GROUP_BLOB_BYTES)()
    with ShCtx(n, W, H) as c:
        c.upload(splat60)
        L = c.L
        want = dor.oracle_frame(splat60, vp, ub)
        _lib.check(order(c, VIEW), "gsr_set_depth_order")
        for bad in (-1, 2, 7, 1 << 30):
            assert order(c, bad) == _lib.GSR_ERR_INVALID
        check(c, c.render(vp, ub), want, n)   # the previous state is kept
        # while the mode is on, the multi-context calls are refused
        assert L.gsr_set_band(c.h, 0, 3) == _lib.GSR_ERR_STATE
        assert L.gsr_set_row_interleave(c.h, 0, 2) == _lib.GSR_ERR_STATE
        assert L.gsr_peer_export_framebuffers(c.h, handles) == _lib.GSR_ERR_STATE
        assert L.gsr_peer_import_framebuffers(c.h, handles) == _lib.GSR_ERR_STATE
        assert L.gsr_group_export(c.h, blob) == _lib.GSR_ERR_STATE
        check(c, c.render(vp, ub), want, n)
        # and switching it on is refused on a multi-context setup
        _lib.check(order(c, 0), "off")
        for setup, undo in ((lambda: L.gsr_set_band(c.h, 0, 3), lambda: L.gsr_set_band(c.h, 0, (H + 15) // 16)),
                            (lambda: L.gsr_set_row_interleave(c.h, 0, 2), lambda: L.gsr_set_row_interleave(c.h, 0, 1)),
                            (lambda: L.gsr_peer_export_framebuffers(c.h, handles), lambda: L.gsr_resize(c.h, W, H))):
            _lib.check(setup(), "setup")
            assert order(c, VIEW) == _lib.GSR_ERR_STATE
            assert order(c, 0) == _lib.GSR_OK
            _lib.check(undo(), "undo")
        _lib.check(order(c, VIEW), "on")
        c.resize(W, H)   # keeps the setting
        check(c, c.render(vp, ub), want, n)


def test_rasterizer_depth_order():
    n = 12288
    t62 = synthetic_ply_table(n, 12)
    t62[:, 55:58] += 0.5
    ply = PlyFile.from_array(t62)
    r = GaussianSplattingRasterizer(ply, (W, H), None, cam.orbit_camera(25, aspect=W / H), depth_order=1)
    r.init_gpu()
    try:
        out = np.empty((H, W, 4), dtype=np.float32)
        r.rasterize(time=10.0, out_host=out)
        vp, ub = r.camera_push_constants, r.uniforms_bytes(10.0)
        splat60 = swizzle_splats(t62, 0.0)
        np.testing.assert_array_equal(bits(out), bits(dor.oracle_frame(splat60, vp, ub)["rgba"]))
        r.set_depth_order(0)
        r.rasterize(time=10.0, out_host=out)
        vp, ub = r.camera_push_constants, r.uniforms_bytes(10.0)
        want = orc.frame(splat60, vp, orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8)), cap=64 * n).rgba
        np.testing.assert_array_equal(bits(out), bits(want))
    finally:
        r.cleanup_gpu()
