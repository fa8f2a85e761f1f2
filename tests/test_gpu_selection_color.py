"""Selection colour edits on the GPU (include/gsr.h "Splat colour edits"), through the C-ABI: the edited store against the numpy rule of
tests/color_reference bit for bit, frames after edits against the frames of the oracle-edited cloud, the identity edit, the record
colours against A colour + b, a slider drag of asynchronous frames from a snapshot with and without front / back overlap, the
composition with a transform edit, the argument and state rules, and the export."""
import ctypes as C

import numpy as np
import pytest

from godotgaussiansplatting_b200 import _lib
from godotgaussiansplatting_b200.rasterizer import color_edit, store_to_table
from godotgaussiansplatting_b200.synthetic import synthetic_ply_table
from godotgaussiansplatting_b200.ply_file import swizzle_splats
from tests import color_reference as cref
from tests import transform_reference as tref
from tests.gsr_direct import REC_DTYPE
from tests.test_gpu_cutouts import cloud, view
from tests.test_gpu_selection_transform import H, N, W, device_buffer, restore_host, store_of, transform
from tests.test_gpu_sh_degree import ShCtx, set_instances
from tests.test_gpu_splat_selection import seeded_masks, set_masks, style
from tests.test_instances import rigid
from tests.test_selection_transform import TRANSFORMS, ts12

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

U32 = np.uint32
GRADE = color_edit(gain=(1.1, 0.9, 1.05), saturation=1.3, hue=25.0, brightness=0.05)


def recolor(c, e, snapshot=None):
    return c.L.gsr_recolor_selection(c.h, C.byref(e), None if snapshot is None else C.c_void_p(snapshot))


def last_constants(c):
    return c.copy(_lib.GSR_BUF_EDIT_COLOR, 41, np.float32)


@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("bands", [1, 2, 3, 4])
def test_store_is_the_oracle(bands, half):
    splat60 = cloud(N)
    hid, sel = seeded_masks(N, bands)
    with ShCtx(N, W, H, bands, _lib.GSR_FLAG_SH_HALF if half else 0) as c:
        c.upload(splat60)
        _lib.check(set_masks(c, hid, sel), "masks")
        before = store_of(c)
        a = color_edit(gain=(1.2, 0.8, 1.05), saturation=1.6, view_dependence=0.5, opacity=2.5, opacity_offset=-0.6)
        _lib.check(recolor(c, a), "recolour in place")
        k_a = last_constants(c)
        np.testing.assert_array_equal(k_a.view(U32), cref.constants(a).view(U32))
        edited = store_of(c)
        tref.assert_store_equal(edited, cref.oracle(before, bands, half, sel, k_a), half, "in place")
        snap = device_buffer(c)
        _lib.check(c.L.gsr_copy_splat_store(c.h, C.c_void_p(snap.data_ptr())), "copy")
        b = color_edit(hue=-60.0, contrast=1.3, brightness=-0.1, opacity=0.5, opacity_offset=0.2)
        _lib.check(recolor(c, b, snap.data_ptr()), "recolour from a snapshot")
        _lib.check(recolor(c, b, snap.data_ptr()), "again: the snapshot is unchanged")
        k_b = last_constants(c)
        np.testing.assert_array_equal(k_b.view(U32), cref.constants(b).view(U32))
        tref.assert_store_equal(store_of(c), cref.oracle(edited, bands, half, sel, k_b, src=edited), half, "from a snapshot")


@pytest.mark.parametrize("variant", ["plain", "instances", "half", "depth_motion_ids", "degree1"])
def test_frame_after_edit_is_the_edited_cloud(variant):
    """The frame after an edit is the default frame of the oracle-edited cloud (restored into a second context as a store)."""
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
            if variant == "degree1":
                _lib.check(x.degree(1), "degree")
            _lib.check(set_masks(x, hid, sel), "masks")
            _lib.check(style(x, (1.0, 0.5, 0.0), 0.0), "style")
            if variant == "depth_motion_ids":
                p = planes.setdefault(id(x), dict(d=torch.zeros(H * W, device="cuda"), m=torch.zeros(H * W * 2, device="cuda"),
                                                  i=torch.zeros(H * W * 2, dtype=torch.int32, device="cuda")))
                _lib.check(x.L.gsr_set_depth_compositing(x.h, None, C.c_void_p(p["d"].data_ptr())), "depth")
                _lib.check(x.L.gsr_set_motion_vectors(x.h, C.c_void_p(p["m"].data_ptr())), "motion")
                _lib.check(x.L.gsr_set_splat_ids(x.h, C.c_void_p(p["i"].data_ptr())), "ids")
        c.render(vp, ub)
        r.render(vp, ub)
        e = color_edit(gain=(1.3, 0.8, 1.0), saturation=1.4, hue=30.0, brightness=0.02, view_dependence=0.6, opacity=1.5, opacity_offset=-0.2)
        before = store_of(c)
        _lib.check(recolor(c, e), "recolour")
        restore_host(r, cref.oracle(before, 4, half, sel, cref.constants(e)))
        got, want = c.render(vp, ub), r.render(vp, ub)
        np.testing.assert_array_equal(got.view(U32), want.view(U32))
        if variant == "depth_motion_ids":
            pc, pr = planes[id(c)], planes[id(r)]
            torch.cuda.synchronize()
            for k in ("d", "m", "i"):
                assert torch.equal(pc[k], pr[k]), k


def test_identity_edit_keeps_the_frame():
    splat60 = cloud(N)
    vp, ub = view()
    hid, sel = seeded_masks(N, 11, hidden=0.1, selected=0.5)
    with ShCtx(N, W, H) as c:
        c.upload(splat60)
        _lib.check(set_masks(c, hid, sel), "masks")
        _lib.check(style(c, (1.0, 0.5, 0.0), 0.0), "style")
        want = c.render(vp, ub)
        _lib.check(recolor(c, color_edit()), "identity")
        np.testing.assert_array_equal(c.render(vp, ub).view(U32), want.view(U32))


def unclamped_cloud(n, seed=4):
    """A cloud whose colours stay inside (0, 1) before and after GRADE, from every direction: DC near grey, small SH."""
    t62 = synthetic_ply_table(n, seed)
    rng = np.random.default_rng(seed)
    t62[:, 55:58] += 0.5
    t62[:, 6:9] = rng.uniform(-0.6, 0.6, size=(n, 3))
    t62[:, 9:54] = rng.uniform(-0.02, 0.02, size=(n, 45))
    return swizzle_splats(t62, 0.0)


def test_record_colours_are_the_affine_map():
    splat60 = unclamped_cloud(N)
    vp, ub = view()
    vp2, ub2 = view(frame=60)
    with ShCtx(N, W, H) as c, ShCtx(N, W, H) as r:
        for x in (c, r):
            x.upload(splat60)
            _lib.check(x.L.gsr_select_all(x.h, _lib.GSR_SELECT_SET), "select")
            _lib.check(style(x, (1.0, 0.5, 0.0), 0.0), "style")
        _lib.check(recolor(c, GRADE), "recolour")
        c.render(vp, ub)
        r.render(vp, ub)
        rc, rr = c.copy(_lib.GSR_BUF_RECORDS, N, REC_DTYPE), r.copy(_lib.GSR_BUF_RECORDS, N, REC_DTYPE)
        vis = np.unique(c.taps()["values"])
        assert vis.size > 1000
        col0 = rr["color"][vis, :3].astype(np.float64)
        assert (col0 > 0).all() and (rc["color"][vis, :3] > 0).all(), "the cloud's colours are unclamped"
        A, b = cref.affine(GRADE)
        np.testing.assert_allclose(rc["color"][vis, :3], col0 @ A.T + b, atol=1e-5, rtol=0)
        # without the view-dependent colour an edited splat shows the same colour from every camera
        _lib.check(recolor(c, color_edit(view_dependence=0.0)), "flatten")
        c.render(vp, ub)
        one = c.copy(_lib.GSR_BUF_RECORDS, N, REC_DTYPE)
        v1 = np.unique(c.taps()["values"])
        c.render(vp2, ub2)
        two = c.copy(_lib.GSR_BUF_RECORDS, N, REC_DTYPE)
        v2 = np.unique(c.taps()["values"])
        both = np.intersect1d(v1, v2)
        assert both.size > 1000
        np.testing.assert_array_equal(one["color"][both, :3].view(U32), two["color"][both, :3].view(U32))
        r.render(vp2, ub2)
        unflat = r.copy(_lib.GSR_BUF_RECORDS, N, REC_DTYPE)
        assert not np.array_equal(unflat["color"][both, :3], rr["color"][both, :3])   # the unedited cloud is view-dependent


def slider(i):
    """The i-th edit of a slider drag: a growing warm grade that also fades."""
    return color_edit(gain=(1.0 + 0.02 * i, 1.0, 1.0 - 0.01 * i), saturation=1.0 + 0.03 * i, opacity=1.0 - 0.02 * i)


@pytest.mark.parametrize("overlap", [0, 1])
def test_slider_drag_from_a_snapshot(overlap):
    splat60 = cloud(N)
    vp, ub = view()
    inst = [(0, N, rigid(4)), (100, 5000, rigid(6))]
    hid, sel = seeded_masks(N, 3, hidden=0.05, selected=0.3)
    steps = 24
    with ShCtx(N, W, H) as c, ShCtx(N, W, H) as r:
        for x in (c, r):
            x.upload(splat60)
            set_instances(x, inst)
            _lib.check(set_masks(x, hid, sel), "masks")
            _lib.check(style(x, (0.2, 0.4, 1.0), 0.3), "style")
            d = torch.zeros(H * W, device="cuda")
            x.depth_plane = d
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
            _lib.check(recolor(c, slider(i), snap.data_ptr()), "drag")
            _lib.check(c.L.gsr_set_motion_vectors(c.h, C.c_void_p(motion[i].data_ptr())), "motion")
            c.render_async(vp, ub, host_ptr=host[i].data_ptr())
        _lib.check(c.L.gsr_restore_splat_store(c.h, C.c_void_p(snap.data_ptr())), "undo")
        _lib.check(set_masks(c, hid, sel), "undo masks")
        _lib.check(c.L.gsr_set_motion_vectors(c.h, C.c_void_p(motion[steps + 1].data_ptr())), "motion")
        c.render_async(vp, ub, host_ptr=host[steps + 1].data_ptr())
        c.sync()
        torch.cuda.synchronize()
        for i in range(steps + 2):
            store = original if i in (0, steps + 1) else cref.oracle(original, 4, False, sel, cref.constants(slider(i)))
            restore_host(r, store)
            want = r.render(vp, ub)
            np.testing.assert_array_equal(host[i].numpy().view(U32), want.view(U32), err_msg=f"frame {i}")
            assert torch.count_nonzero(motion[i]).item() == 0, f"motion of frame {i}"
        np.testing.assert_array_equal(host[steps + 1].numpy().view(U32), host[0].numpy().view(U32))


def test_transform_then_recolour():
    splat60 = cloud(N)
    hid, sel = seeded_masks(N, 21, hidden=0.1, selected=0.4)
    with ShCtx(N, W, H) as c:
        c.upload(splat60)
        _lib.check(set_masks(c, hid, sel), "masks")
        before = store_of(c)
        a = ts12(*TRANSFORMS["rigid"])
        _lib.check(transform(c, a), "transform")
        _lib.check(recolor(c, GRADE), "recolour")
        moved = tref.oracle(before, 4, False, sel, tref.matrices(a))
        tref.assert_store_equal(store_of(c), cref.oracle(moved, 4, False, sel, cref.constants(GRADE)), False, "transform, recolour")


def test_rules_leave_the_store_unchanged():
    splat60 = cloud(N)
    with ShCtx(N, W, H) as c:
        c.upload(splat60)
        want = store_of(c)
        assert recolor(c, GRADE) == _lib.GSR_ERR_STATE   # masks not in use
        _lib.check(c.L.gsr_select_all(c.h, _lib.GSR_SELECT_SET), "select")
        _lib.check(c.L.gsr_clear_splat_masks(c.h), "clear")
        assert recolor(c, GRADE) == _lib.GSR_ERR_STATE
        _lib.check(c.L.gsr_select_all(c.h, _lib.GSR_SELECT_SET), "select")

        def bad(**kw):
            e = color_edit()
            for name, (i, v) in kw.items():
                if i is None:
                    setattr(e, name, v)
                else:
                    getattr(e, name)[i] = v
            return e
        cases = [bad(matrix=(i, v)) for i in (0, 4, 9, 11) for v in (np.nan, np.inf, -np.inf, 16.5, -17.0)]
        cases += [bad(band_scale=(i, v)) for i in (0, 2) for v in (np.nan, -0.5, 16.5, np.inf)]
        cases += [bad(opacity_scale=(None, v)) for v in (np.nan, -0.1, 16.5)]
        cases += [bad(opacity_offset=(None, v)) for v in (np.nan, -1.5, 1.01, np.inf)]
        for e in cases:
            assert recolor(c, e) == _lib.GSR_ERR_INVALID
        assert c.L.gsr_recolor_selection(c.h, None, None) == _lib.GSR_ERR_INVALID
        assert c.L.gsr_recolor_selection(None, C.byref(GRADE), None) == _lib.GSR_ERR_INVALID
        _lib.check(c.L.gsr_clear_splat_masks(c.h), "clear")
        assert recolor(c, bad(opacity_offset=(None, 2.0))) == _lib.GSR_ERR_INVALID   # the arguments are checked first
        np.testing.assert_array_equal(c.copy(_lib.GSR_BUF_EDIT_COLOR, 41, np.float32), 0.0)
        np.testing.assert_array_equal(store_of(c).view(U32), want.view(U32))
        _lib.check(c.L.gsr_select_all(c.h, _lib.GSR_SELECT_SET), "select")
        edge = color_edit(opacity=16.0, opacity_offset=-1.0)   # the bounds themselves are accepted
        edge.matrix[0], edge.band_scale[1] = -16.0, 16.0
        _lib.check(recolor(c, edge), "edge")


def test_export_renders_like_the_edited_context():
    table = synthetic_ply_table(N, 3)
    vp, ub = view()
    hid, sel = seeded_masks(N, 17, hidden=0.2, selected=0.3)
    with ShCtx(N, W, H) as c:
        c.upload_ply_raw(table)
        _lib.check(set_masks(c, hid, sel), "masks")
        _lib.check(style(c, (1.0, 0.5, 0.0), 0.0), "style")
        _lib.check(recolor(c, color_edit(gain=(0.8, 1.1, 1.2), hue=15.0, view_dependence=0.5, opacity=0.7, opacity_offset=0.1)), "recolour")
        got = c.render(vp, ub)
        kept = store_to_table(store_of(c), N, 4, False, hid)
    with ShCtx(kept.shape[0], W, H) as k:
        k.upload_ply_raw(kept)
        want = k.render(vp, ub)
    err = np.abs(got - want)
    assert err.max() <= 2e-3 and err.mean() <= 1e-5, (err.max(), err.mean())
