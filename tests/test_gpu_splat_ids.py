"""Splat and instance IDs on the GPU (include/gsr.h gsr_set_splat_ids), through the C-ABI with torch CUDA tensors as the caller's planes:
every case of tests/variant_matrix drawn with the depth (or motion) compositor plus IDs, bit for bit against the ID oracle on the
composed reference, with rgba, depth and motion unchanged; and the state rules, double-buffered planes, gsr_pick, the overflow
re-render and GSR_FLAG_STATIC_CAPACITY."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

from godotgaussiansplatting_b200 import _lib
from godotgaussiansplatting_b200.rasterizer import pack_instance_appearance
from oracle import oracle as orc
from tests import id_reference as idr
from tests import variant_matrix as vm
from tests.gsr_direct import REC_DTYPE, Ctx
from tests.scenes import make_scene
from tests.test_gpu_sh_degree import ShCtx, set_instances
from tests.test_gpu_variant_matrix import N, RAGGED, SIZE, flags_of, set_cutouts

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

NO_ID = idr.NO_ID
SENTINEL = 0x5A5A5A5A
bits = vm.bits


def ids_plane(w, h, tail=0):
    """A uint32 (h * w * 2 + tail) plane filled with SENTINEL (as int32: torch has no uint32 fill)."""
    t = torch.full((h * w * 2 + tail,), SENTINEL, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    return t


def read_ids(t, w, h):
    a = t.cpu().numpy().view(np.uint32)
    return a[:h * w * 2].reshape(h, w, 2), a[h * w * 2:]


def ptr(t):
    return C.c_void_p(t.data_ptr())


def set_splat_ids(c, address):
    """gsr_set_splat_ids on a gsr_direct.Ctx: the return code (address: a device address, or None to switch the IDs off)."""
    return c.L.gsr_set_splat_ids(c.h, None if address is None else C.c_void_p(address))


# ---- every variant-matrix case with IDs ----------------------------------------------------------------------------------------
def id_case(case):
    """The case drawn with IDs: its own depth or motion compositor, the depth compositor for a plain case."""
    return dataclasses.replace(case, compositor="depth") if case.compositor == "plain" else case


def render_case_with_ids(fr):
    case = fr.case
    L = _lib.lib()
    heat = 1.0 if case.heat else 0.0
    with ShCtx(fr.n, fr.w, fr.h, case.store_bands, flags_of(case), factor=16) as c:
        c.upload(fr.splat60)
        if case.store_bands != case.bands:
            _lib.check(c.degree(case.bands - 1), "gsr_set_sh_degree")
        if case.aa:
            _lib.check(L.gsr_set_antialiasing(c.h, C.c_float(case.v)), "gsr_set_antialiasing")
        if case.dord:
            _lib.check(L.gsr_set_depth_order(c.h, _lib.GSR_DEPTH_ORDER_VIEW_DEPTH), "gsr_set_depth_order")
        if case.cut:
            set_cutouts(c, fr.vols)
        if case.inst:
            set_instances(c, fr.prev_inst if fr.prev_inst is not None else fr.inst)
            if fr.app is not None:
                app = pack_instance_appearance(fr.app)
                _lib.check(L.gsr_set_instance_appearance(c.h, app, len(app)), "gsr_set_instance_appearance")
        Zt = None if fr.Z is None else torch.from_numpy(fr.Z).cuda()
        depth = torch.full((fr.h, fr.w), float("nan"), dtype=torch.float32, device="cuda")
        ids = ids_plane(fr.w, fr.h, tail=64)
        _lib.check(L.gsr_set_depth_compositing(c.h, None if Zt is None else ptr(Zt), ptr(depth)), "gsr_set_depth_compositing")
        _lib.check(set_splat_ids(c, ids.data_ptr()), "gsr_set_splat_ids")
        motion = None
        if case.compositor == "motion":
            motion = torch.full((fr.h, fr.w, 2), float("nan"), dtype=torch.float32, device="cuda")
            torch.cuda.synchronize()
            _lib.check(L.gsr_set_motion_vectors(c.h, ptr(motion)), "gsr_set_motion_vectors")
            c.render(fr.pvp, fr.pub, heatmap=heat)
            if case.inst:
                set_instances(c, fr.inst)
        rgba = c.render(fr.vp, fr.ub, heatmap=heat)
        c.sync()
        got_ids, tail = read_ids(ids, fr.w, fr.h)
        return dict(rgba=rgba, depth=depth.cpu().numpy(), motion=None if motion is None else motion.cpu().numpy(), ids=got_ids,
                    tail=tail, staged=c.stats().staged)


@pytest.mark.parametrize("i", range(len(vm.CASES)), ids=vm.IDS)
def test_case_with_ids_is_the_reference(i):
    case = id_case(vm.CASES[i])
    fr = vm.frame_of(case, N, SIZE, RAGGED)
    ref = vm.reference(fr)
    heat = 1.0 if case.heat else 0.0
    ranges = [(f, k) for f, k, _ in fr.inst] if case.inst else None
    o_rgba, o_depth, o_ids, o_staged = idr.render_ids(ref["records"], ref["values"], ref["bounds"], fr.w, fr.h, fr.vp, fr.Z, heat,
                                                      case.contract, ranges)
    np.testing.assert_array_equal(bits(o_rgba), bits(ref["rgba"]))
    np.testing.assert_array_equal(bits(o_depth), bits(ref["depth"]))
    got = render_case_with_ids(fr)
    np.testing.assert_array_equal(got["ids"], o_ids)
    np.testing.assert_array_equal(bits(got["rgba"]), bits(ref["rgba"]))
    np.testing.assert_array_equal(bits(got["depth"]), bits(ref["depth"]))
    assert got["staged"] == ref["staged"] == o_staged
    if case.compositor == "motion":
        np.testing.assert_array_equal(bits(got["motion"]), bits(ref["motion"]))
    assert (got["tail"] == SENTINEL).all(), "a pixel outside the image was written"
    has = o_ids[..., 0] != NO_ID
    assert has.any() and (~has).any()
    np.testing.assert_array_equal(has, o_rgba[..., 3] > 0)


# ---- the rules -----------------------------------------------------------------------------------------------------------------
def last_frame_lists(c, n_records):
    st = c.stats()
    m = int(min(st.duplicates, st.capacity))
    T = st.tiles_x * st.tiles_y
    recs = c.copy(_lib.GSR_BUF_RECORDS, n_records, REC_DTYPE).view(orc.RECORD_DTYPE)
    return recs, c.copy(_lib.GSR_BUF_VALUES, m, np.uint32), c.copy(_lib.GSR_BUF_BOUNDS, T * 2, np.uint32).reshape(T, 2)


def oracle_ids(c, n, vp, w, h, contract=True):
    recs, vals, bnds = last_frame_lists(c, n)
    return idr.render_ids(recs, vals, bnds, w, h, vp, None, 0.0, contract)


def test_state_and_argument_rules():
    n, w, h = 6000, 160, 120
    splat60, vp, ub = make_scene(n, 2, w, h, frame=13, scale_boost=0.5)
    with Ctx(n, w, h) as c:
        c.upload(splat60)
        L = c.L
        depth = torch.empty((h, w), dtype=torch.float32, device="cuda")
        scene = torch.full((h, w), float("inf"), dtype=torch.float32, device="cuda")
        motion = torch.empty((h, w, 2), dtype=torch.float32, device="cuda")
        a, b = ids_plane(w, h), ids_plane(w, h)
        assert set_splat_ids(c, a.data_ptr()) == _lib.GSR_ERR_STATE          # depth compositing is off
        _lib.check(L.gsr_set_depth_compositing(c.h, ptr(scene), ptr(depth)), "gsr_set_depth_compositing")
        _lib.check(L.gsr_set_motion_vectors(c.h, ptr(motion)), "gsr_set_motion_vectors")
        _lib.check(set_splat_ids(c, a.data_ptr()), "gsr_set_splat_ids")
        for bad in (depth, scene, motion):                                   # refused; the plane stays a
            assert set_splat_ids(c, bad.data_ptr()) == _lib.GSR_ERR_INVALID
        assert L.gsr_set_motion_vectors(c.h, ptr(a)) == _lib.GSR_ERR_INVALID  # nor may motion take the ID plane
        c.render(vp, ub)
        ref = oracle_ids(c, n, vp, w, h)
        np.testing.assert_array_equal(read_ids(a, w, h)[0], ref[2])
        assert (read_ids(b, w, h)[0] == SENTINEL).all()
        # NULL switches the IDs off
        _lib.check(set_splat_ids(c, None), "gsr_set_splat_ids")
        a.fill_(SENTINEL)
        torch.cuda.synchronize()
        c.render(vp, ub)
        c.sync()
        assert (read_ids(a, w, h)[0] == SENTINEL).all()
        # depth compositing off switches them off: on again, no IDs until they are set again
        _lib.check(set_splat_ids(c, a.data_ptr()), "gsr_set_splat_ids")
        _lib.check(L.gsr_set_depth_compositing(c.h, None, None), "gsr_set_depth_compositing")
        assert set_splat_ids(c, b.data_ptr()) == _lib.GSR_ERR_STATE
        _lib.check(L.gsr_set_depth_compositing(c.h, None, ptr(depth)), "gsr_set_depth_compositing")
        c.render(vp, ub)
        c.sync()
        assert (read_ids(a, w, h)[0] == SENTINEL).all()
        # so does gsr_resize
        _lib.check(set_splat_ids(c, a.data_ptr()), "gsr_set_splat_ids")
        c.resize(w, h)
        _lib.check(L.gsr_set_depth_compositing(c.h, None, ptr(depth)), "gsr_set_depth_compositing")
        c.render(vp, ub)
        c.sync()
        assert (read_ids(a, w, h)[0] == SENTINEL).all()


def test_double_buffered_planes_and_pick():
    n, w, h = 6000, 160, 120
    splat60, vp0, ub0 = make_scene(n, 3, w, h, frame=10, scale_boost=0.5)
    _, vp1, ub1 = make_scene(n, 3, w, h, frame=40, scale_boost=0.5)
    with Ctx(n, w, h, factor=1000) as c:
        c.upload(splat60)
        depth = torch.empty((h, w), dtype=torch.float32, device="cuda")
        _lib.check(c.L.gsr_set_depth_compositing(c.h, None, ptr(depth)), "gsr_set_depth_compositing")
        planes = [ids_plane(w, h), ids_plane(w, h)]
        refs = []
        for vp, ub, plane in ((vp0, ub0, planes[0]), (vp1, ub1, planes[1])):
            _lib.check(set_splat_ids(c, plane.data_ptr()), "gsr_set_splat_ids")
            c.render_async(vp, ub)
        c.sync()
        # the second frame's lists are the library's last ones; the first frame's come from the oracle's own frame
        f0 = orc.frame(splat60, vp0, orc.uniforms_from_bytes(np.frombuffer(ub0, dtype=np.uint8)), cap=1000 * n)
        refs.append(idr.render_ids(f0.records, f0.values, f0.bounds, w, h, vp0)[2])
        refs.append(oracle_ids(c, n, vp1, w, h)[2])
        for plane, ref in zip(planes, refs):
            np.testing.assert_array_equal(read_ids(plane, w, h)[0], ref)
        assert not np.array_equal(refs[0], refs[1])
        st = c.stats()
        c.pick((st.tiles_y // 2) * st.tiles_x + st.tiles_x // 2)   # gsr_pick keeps the default path and leaves the plane as it is
        np.testing.assert_array_equal(read_ids(planes[1], w, h)[0], refs[1])


def test_overflow_rerender_writes_the_same_ids():
    n, w, h = 6000, 160, 120
    splat60, vp, ub = make_scene(n, 2, w, h, frame=13, scale_boost=1.0)
    _, pvp, pub = make_scene(n, 2, w, h, frame=10, scale_boost=1.0)
    pvp[14] -= np.float32(40.0)   # far away: few pairs, the capacity stays small
    with Ctx(n, w, h, factor=1) as c:   # the second synchronous render overflows and is rendered again
        c.upload(splat60)
        depth = torch.empty((h, w), dtype=torch.float32, device="cuda")
        _lib.check(c.L.gsr_set_depth_compositing(c.h, None, ptr(depth)), "gsr_set_depth_compositing")
        ids = ids_plane(w, h)
        _lib.check(set_splat_ids(c, ids.data_ptr()), "gsr_set_splat_ids")
        c.render(pvp, pub)
        m0 = c.stats().duplicates
        rgba = c.render(vp, ub)
        assert c.stats().capacity > 3 * m0, "the frame did not overflow"
        o_rgba, _, o_ids, _ = oracle_ids(c, n, vp, w, h)
        np.testing.assert_array_equal(read_ids(ids, w, h)[0], o_ids)
        np.testing.assert_array_equal(bits(rgba), bits(o_rgba))


def test_static_capacity():
    n, w, h = 6000, 160, 120
    splat60, vp, ub = make_scene(n, 2, w, h, frame=13, scale_boost=1.0)
    with ShCtx(n, w, h, 0, _lib.GSR_FLAG_STATIC_CAPACITY, factor=1) as c:
        c.upload(splat60)
        depth = torch.empty((h, w), dtype=torch.float32, device="cuda")
        _lib.check(c.L.gsr_set_depth_compositing(c.h, None, ptr(depth)), "gsr_set_depth_compositing")
        ids = ids_plane(w, h)
        _lib.check(set_splat_ids(c, ids.data_ptr()), "gsr_set_splat_ids")
        out = np.empty((h, w, 4), dtype=np.float32)
        rc = c.L.gsr_render(c.h, np.ascontiguousarray(vp, dtype=np.float32).ctypes.data_as(C.POINTER(C.c_float)), ub, 0.0,
                            C.c_void_p(out.ctypes.data))
        assert rc in (_lib.GSR_OK, _lib.GSR_ERR_OVERFLOW)
        assert c.stats().overflow, "the frame did not overflow its static capacity"
        o_rgba, _, o_ids, _ = oracle_ids(c, n, vp, w, h)   # the truncated lists the frame drew
        np.testing.assert_array_equal(read_ids(ids, w, h)[0], o_ids)
        np.testing.assert_array_equal(bits(out), bits(o_rgba))
