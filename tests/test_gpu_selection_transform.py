"""Selection transform edits on the GPU (include/gsr.h "Splat transform edits"), through the C-ABI: the edited store against the numpy
rule of tests/transform_reference bit for bit, frames after edits against the frames of the oracle-edited cloud, a drag of asynchronous
frames from a snapshot with and without front / back overlap, the physical meaning (a whole-cloud rigid edit against the same cloud
drawn as an instance), store snapshots to device, pinned and pageable memory, the argument and state rules, and the export."""
import ctypes as C

import numpy as np
import pytest

from godotgaussiansplatting_b200 import _lib
from godotgaussiansplatting_b200.rasterizer import store_to_table
from tests import transform_reference as tref
from tests.gsr_direct import REC_DTYPE
from tests.test_gpu_cutouts import cloud, view
from tests.test_gpu_sh_degree import ShCtx, set_instances
from tests.test_gpu_splat_selection import seeded_masks, set_masks, style
from tests.test_instances import rigid
from tests.test_selection_transform import RIGID, TRANSFORMS, rot, ts12

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

W, H = 320, 200
N = 12288 - 77   # not a multiple of 32
STRIDE = (N + 255) // 256 * 256
FP = C.POINTER(C.c_float)
U32 = np.uint32


def store_of(c):
    nbytes = int(c.L.gsr_splat_store_bytes(c.h))
    return c.copy(_lib.GSR_BUF_SPLATS, nbytes // 4, np.float32).reshape(-1, STRIDE, 4)


def transform(c, ts, snapshot=None):
    t = np.ascontiguousarray(ts, dtype=np.float32)
    return c.L.gsr_transform_selection(c.h, t.ctypes.data_as(FP), None if snapshot is None else C.c_void_p(snapshot))


def device_buffer(c):
    return torch.empty(int(c.L.gsr_splat_store_bytes(c.h)), dtype=torch.uint8, device="cuda")


def restore_host(c, store):
    s = np.ascontiguousarray(store, dtype=np.float32)
    _lib.check(c.L.gsr_restore_splat_store(c.h, C.c_void_p(s.ctypes.data)), "restore")
    c.sync()


def drag(i):
    """The i-th transform of a drag: a growing rotation about a pivot and a slide."""
    L = rot(2, 3.0 * i) @ rot(0, 1.5 * i)
    p = np.array([0.1, 0.0, 2.5])
    return ts12(L, p - L @ p + np.array([0.01 * i, 0.0, 0.0]))


@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("bands", [1, 2, 3, 4])
def test_store_is_the_oracle(bands, half):
    splat60 = cloud(N)
    hid, sel = seeded_masks(N, bands)
    with ShCtx(N, W, H, bands, _lib.GSR_FLAG_SH_HALF if half else 0) as c:
        c.upload(splat60)
        _lib.check(set_masks(c, hid, sel), "masks")
        before = store_of(c)
        a = ts12(*TRANSFORMS["nonuniform"])
        _lib.check(transform(c, a), "transform in place")
        m_a = c.copy(_lib.GSR_BUF_EDIT_TRANSFORM, 95, np.float32)
        np.testing.assert_array_equal(m_a.view(U32), tref.matrices(a).view(U32))
        edited = store_of(c)
        tref.assert_store_equal(edited, tref.oracle(before, bands, half, sel, m_a), half, "in place")
        snap = device_buffer(c)
        _lib.check(c.L.gsr_copy_splat_store(c.h, C.c_void_p(snap.data_ptr())), "copy")
        b = ts12(*TRANSFORMS["reflection"])
        _lib.check(transform(c, b, snap.data_ptr()), "transform from a snapshot")
        _lib.check(transform(c, b, snap.data_ptr()), "again: the snapshot is unchanged")
        m_b = c.copy(_lib.GSR_BUF_EDIT_TRANSFORM, 95, np.float32)
        np.testing.assert_array_equal(m_b.view(U32), tref.matrices(b).view(U32))
        tref.assert_store_equal(store_of(c), tref.oracle(edited, bands, half, sel, m_b, src=edited), half, "from a snapshot")


def frame(c, vp, ub):
    return c.render(vp, ub)


@pytest.mark.parametrize("variant", ["plain", "instances", "half", "depth_motion_ids"])
def test_frame_after_edit_is_the_edited_cloud(variant):
    """The frame after an edit is the default frame of the oracle-edited cloud (uploaded into a second context as a store)."""
    splat60 = cloud(N)
    vp, ub = view()
    half = variant == "half"
    flags = _lib.GSR_FLAG_SH_HALF if half else 0
    hid, sel = seeded_masks(N, 9, hidden=0.1, selected=0.4)
    inst = [(0, N, rigid(4)), (0, N, rigid(5))] if variant in ("instances", "depth_motion_ids") else None
    planes = {}
    with ShCtx(N, W, H, 0, flags) as c, ShCtx(N, W, H, 0, flags) as r:
        for x in (c, r):
            x.upload(splat60)
            if inst:
                set_instances(x, inst)
            _lib.check(set_masks(x, hid, sel), "masks")
            _lib.check(style(x, (1.0, 0.5, 0.0), 0.0), "style")
            if variant == "depth_motion_ids":
                p = planes.setdefault(id(x), dict(d=torch.zeros(H * W, device="cuda"), m=torch.zeros(H * W * 2, device="cuda"),
                                                  i=torch.zeros(H * W * 2, dtype=torch.int32, device="cuda")))
                _lib.check(x.L.gsr_set_depth_compositing(x.h, None, C.c_void_p(p["d"].data_ptr())), "depth")
                _lib.check(x.L.gsr_set_motion_vectors(x.h, C.c_void_p(p["m"].data_ptr())), "motion")
                _lib.check(x.L.gsr_set_splat_ids(x.h, C.c_void_p(p["i"].data_ptr())), "ids")
        frame(c, vp, ub)
        frame(r, vp, ub)
        a = ts12(RIGID, [0.05, -0.1, 0.2])
        before = store_of(c)
        _lib.check(transform(c, a), "transform")
        restore_host(r, tref.oracle(before, 4, half, sel, tref.matrices(a)))
        got, want = frame(c, vp, ub), frame(r, vp, ub)
        np.testing.assert_array_equal(got.view(U32), want.view(U32))
        if variant == "depth_motion_ids":
            pc, pr = planes[id(c)], planes[id(r)]
            torch.cuda.synchronize()
            for k in ("d", "m", "i"):
                assert torch.equal(pc[k], pr[k]), k
            assert torch.count_nonzero(pc["m"]).item() == 0   # an edit is not motion (static camera, same instance transforms)


@pytest.mark.parametrize("overlap", [0, 1])
def test_drag_from_a_snapshot(overlap):
    splat60 = cloud(N)
    vp, ub = view()
    inst = [(0, N, rigid(4)), (100, 5000, rigid(6))]
    hid, sel = seeded_masks(N, 3, hidden=0.05, selected=0.3)
    steps = 24
    with ShCtx(N, W, H) as c, ShCtx(N, W, H) as r:
        planes = []
        for x in (c, r):
            x.upload(splat60)
            set_instances(x, inst)
            _lib.check(set_masks(x, hid, sel), "masks")
            _lib.check(style(x, (0.2, 0.4, 1.0), 0.3), "style")
            d = torch.zeros(H * W, device="cuda")
            planes.append(d)
            _lib.check(x.L.gsr_set_depth_compositing(x.h, None, C.c_void_p(d.data_ptr())), "depth")
        _lib.check(c.L.gsr_debug_pipeline(c.h, overlap), "pipeline")
        motion = [torch.full((H * W * 2,), 7.0, device="cuda") for _ in range(steps + 2)]
        host = [torch.empty((H, W, 4), dtype=torch.float32).pin_memory() for _ in range(steps + 2)]
        _lib.check(c.L.gsr_set_motion_vectors(c.h, C.c_void_p(motion[0].data_ptr())), "motion")
        c.render_async(vp, ub, host_ptr=host[0].data_ptr())
        original = store_of(c)
        snap = device_buffer(c)
        _lib.check(c.L.gsr_copy_splat_store(c.h, C.c_void_p(snap.data_ptr())), "snapshot")
        for i in range(1, steps + 1):   # no host synchronisation from here on
            _lib.check(transform(c, drag(i), snap.data_ptr()), "drag")
            _lib.check(c.L.gsr_set_motion_vectors(c.h, C.c_void_p(motion[i].data_ptr())), "motion")
            c.render_async(vp, ub, host_ptr=host[i].data_ptr())
        _lib.check(c.L.gsr_restore_splat_store(c.h, C.c_void_p(snap.data_ptr())), "undo")
        _lib.check(c.L.gsr_set_motion_vectors(c.h, C.c_void_p(motion[steps + 1].data_ptr())), "motion")
        c.render_async(vp, ub, host_ptr=host[steps + 1].data_ptr())
        c.sync()
        torch.cuda.synchronize()
        for i in range(steps + 2):
            m95 = tref.matrices(drag(min(max(i, 1), steps)))
            store = original if i in (0, steps + 1) else tref.oracle(original, 4, False, sel, m95)
            restore_host(r, store)
            want = r.render(vp, ub)
            np.testing.assert_array_equal(host[i].numpy().view(U32), want.view(U32), err_msg=f"frame {i}")
            assert torch.count_nonzero(motion[i]).item() == 0, f"motion of frame {i}"


def test_physical_meaning_rigid_edit_is_the_instance():
    splat60 = cloud(N)
    vp, ub = view()
    L, t = RIGID, np.array([0.05, -0.1, 0.2])
    a = ts12(L, t)
    with ShCtx(N, W, H) as c, ShCtx(N, W, H) as r:
        c.upload(splat60)
        r.upload(splat60)
        _lib.check(c.L.gsr_select_all(c.h, _lib.GSR_SELECT_SET), "select")
        _lib.check(style(c, (1.0, 0.5, 0.0), 0.0), "style")
        _lib.check(transform(c, a), "transform")
        set_instances(r, [(0, N, a)])
        c.render(vp, ub)
        r.render(vp, ub)
        rc, rr = c.copy(_lib.GSR_BUF_RECORDS, N, REC_DTYPE), r.copy(_lib.GSR_BUF_RECORDS, N, REC_DTYPE)
        vc = np.unique(c.taps()["values"])
        vr = np.unique(r.taps()["values"])
        both = np.intersect1d(vc, vr)
        assert both.size > 1000
        np.testing.assert_array_equal(rc["pos_xy"][both].view(U32), rr["pos_xy"][both].view(U32))
        np.testing.assert_array_equal(rc["pos_z"][both].view(U32), rr["pos_z"][both].view(U32))
        np.testing.assert_allclose(rc["color"][both, :3], rr["color"][both, :3], atol=1e-5)
        np.testing.assert_allclose(rc["conic"][both], rr["conic"][both], rtol=1e-3, atol=1e-3 * np.abs(rr["conic"][both]).max())


def test_snapshots_round_trip():
    splat60 = cloud(N)
    with ShCtx(N, W, H) as c:
        c.upload(splat60)
        want = store_of(c)
        nbytes = int(c.L.gsr_splat_store_bytes(c.h))
        assert nbytes == want.nbytes == 15 * STRIDE * 16
        dev = device_buffer(c)
        pinned = torch.empty(nbytes, dtype=torch.uint8).pin_memory()
        pageable = np.empty(nbytes, dtype=np.uint8)
        for ptr in (dev.data_ptr(), pinned.data_ptr(), pageable.ctypes.data):
            _lib.check(c.L.gsr_copy_splat_store(c.h, C.c_void_p(ptr)), "copy")
            c.sync()
            restore_host(c, np.zeros_like(want))
            assert not store_of(c).any()
            _lib.check(c.L.gsr_restore_splat_store(c.h, C.c_void_p(ptr)), "restore")
            c.sync()
            np.testing.assert_array_equal(store_of(c).view(U32), want.view(U32))
        np.testing.assert_array_equal(pageable.view(U32), want.reshape(-1).view(U32))


def test_rules_leave_the_store_unchanged():
    splat60 = cloud(N)
    with ShCtx(N, W, H) as c:
        c.upload(splat60)
        want = store_of(c)
        ok = ts12(RIGID, [0, 0, 0])
        assert transform(c, ok) == _lib.GSR_ERR_STATE   # masks not in use
        _lib.check(c.L.gsr_select_all(c.h, _lib.GSR_SELECT_SET), "select")
        _lib.check(c.L.gsr_clear_splat_masks(c.h), "clear")
        assert transform(c, ok) == _lib.GSR_ERR_STATE
        _lib.check(c.L.gsr_select_all(c.h, _lib.GSR_SELECT_SET), "select")
        for bad in (np.float32(np.nan), np.float32(np.inf), np.float32(-np.inf)):
            for e in (0, 4, 11):
                x = ok.copy()
                x[e] = bad
                assert transform(c, x) == _lib.GSR_ERR_INVALID
        assert transform(c, ts12(np.diag([1.0, 1.0, 0.0]), [0, 0, 0])) == _lib.GSR_ERR_INVALID
        assert c.L.gsr_transform_selection(c.h, None, None) == _lib.GSR_ERR_INVALID
        assert c.L.gsr_transform_selection(None, ok.ctypes.data_as(FP), None) == _lib.GSR_ERR_INVALID
        assert c.L.gsr_copy_splat_store(c.h, None) == _lib.GSR_ERR_INVALID
        assert c.L.gsr_restore_splat_store(c.h, None) == _lib.GSR_ERR_INVALID
        np.testing.assert_array_equal(c.copy(_lib.GSR_BUF_EDIT_TRANSFORM, 95, np.float32), 0.0)
        np.testing.assert_array_equal(store_of(c).view(U32), want.view(U32))


def test_export_renders_like_the_edited_context():
    from godotgaussiansplatting_b200.synthetic import synthetic_ply_table
    table = synthetic_ply_table(N, 3)
    vp, ub = view()
    hid, sel = seeded_masks(N, 17, hidden=0.2, selected=0.3)
    with ShCtx(N, W, H) as c:
        c.upload_ply_raw(table)
        _lib.check(set_masks(c, hid, sel), "masks")
        _lib.check(style(c, (1.0, 0.5, 0.0), 0.0), "style")
        _lib.check(transform(c, ts12(1.3 * rot(1, 40), [0.1, 0.2, -0.1])), "transform")
        got = c.render(vp, ub)
        kept = store_to_table(store_of(c), N, 4, False, hid)
    with ShCtx(kept.shape[0], W, H) as k:
        k.upload_ply_raw(kept)
        want = k.render(vp, ub)
    err = np.abs(got - want)
    assert err.max() <= 2e-3 and err.mean() <= 1e-5, (err.max(), err.mean())
