"""Splat delete and duplicate on the GPU (include/gsr.h "Splat delete and duplicate"), through the C-ABI: the store, masks and count
after a delete or duplicate of a 6 M-splat store against the numpy rule of tests/delete_reference bit for bit; the frame after a delete
against the frame before it; vacant slots against hidden splats in every case of tests/variant_matrix; duplicate with hide, transform and
instances; exact undo; edits between asynchronous frames with and without front / back overlap; the argument and state rules; a shard
group on a store with vacant slots; the Python mirror and kept_table()."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from godotgaussiansplatting_b200 import _lib
from godotgaussiansplatting_b200.rasterizer import delete_remap, pack_mask, store_to_table, unpack_mask
from tests import delete_reference as dref
from tests import transform_reference as tref
from tests.gsr_direct import REC_DTYPE
from tests.test_gpu_cutouts import cloud, view
from tests.test_gpu_sh_degree import ShCtx, set_instances
from tests.test_gpu_splat_selection import MATRIX_N, MATRIX_STYLE, render_masked_case, seeded_masks, set_masks, style
from tests.test_instances import rigid

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

U32 = np.uint32
U32P = C.POINTER(C.c_uint32)
W, H = 320, 200
N = 12288 - 77            # the cloud: not a multiple of 32
M = N + 3000              # max_splats: room for copies
NO_ID = 0xFFFFFFFF


def bits(a):
    return np.ascontiguousarray(a).view(U32)


def stride_of(m):
    return (m + 255) // 256 * 256


def store_of(c):
    nbytes = int(c.L.gsr_splat_store_bytes(c.h))
    return c.copy(_lib.GSR_BUF_SPLATS, nbytes // 4, np.float32).reshape(-1, stride_of(c.max_splats), 4)


def masks_of(c):
    words = (c.max_splats + 31) // 32
    h, s = np.zeros(words, U32), np.zeros(words, U32)
    _lib.check(c.L.gsr_get_splat_masks(c.h, h.ctypes.data_as(U32P), s.ctypes.data_as(U32P), words), "gsr_get_splat_masks")
    return unpack_mask(h, c.max_splats), unpack_mask(s, c.max_splats)


def count_of(c):
    return int(c.stats().num_splats)


def delete(c):
    k = C.c_uint64(0)
    rc = c.L.gsr_delete_hidden(c.h, C.byref(k))
    return rc, int(k.value)


def duplicate(c):
    s = C.c_uint64(0)
    rc = c.L.gsr_duplicate_selection(c.h, C.byref(s))
    return rc, int(s.value)


def restore_host(c, store):
    s = np.ascontiguousarray(store, dtype=np.float32)
    _lib.check(c.L.gsr_restore_splat_store(c.h, C.c_void_p(s.ctypes.data)), "restore")
    c.sync()


# ---- the store at full size ------------------------------------------------------------------------------------------------------
C3 = 6_000_000


@pytest.mark.parametrize("half", [False, True])
def test_store_is_the_rule_at_full_size(half):
    """A 6 M-splat cloud in a store of 6.6 M slots, random words (NaN and inf included): thousands of CTAs in the look-back."""
    m = C3 + C3 // 10 + 77
    rng = np.random.default_rng(3 + half)
    with ShCtx(m, 64, 64, 4, _lib.GSR_FLAG_SH_HALF if half else 0) as c:
        nbytes = int(c.L.gsr_splat_store_bytes(c.h))
        original = rng.integers(0, 2 ** 32, size=nbytes // 4, dtype=U32).view(np.float32).reshape(-1, stride_of(m), 4)
        block = np.zeros(m, dtype=bool)
        block[C3 // 3:C3 // 3 + (3 * C3) // 10] = True
        deletes = {"random30": rng.random(m) < 0.3, "block30": block, "none": np.zeros(m, dtype=bool), "all": np.ones(m, dtype=bool)}
        for name, hid in deletes.items():
            sel = (rng.random(m) < 0.1) & ~hid
            restore_host(c, original)
            _lib.check(c.L.gsr_set_splat_count(c.h, C3), "count")
            _lib.check(set_masks(c, hid, sel), "masks")
            rc, k = delete(c)
            assert rc == _lib.GSR_OK, _lib.lib().gsr_last_error()
            ws, wh, wsel, wk = dref.delete_rule(original, hid, sel, C3)
            assert (k, count_of(c)) == (wk, wk), name
            np.testing.assert_array_equal(bits(store_of(c)), bits(ws), err_msg=name)
            gh, gsel = masks_of(c)
            np.testing.assert_array_equal(gh, wh)
            np.testing.assert_array_equal(gsel, wsel)
        for f in (0.01, 0.10):
            hid = rng.random(m) < 0.05
            sel = (rng.random(m) < f) & ~hid
            restore_host(c, original)
            _lib.check(c.L.gsr_set_splat_count(c.h, C3), "count")
            _lib.check(set_masks(c, hid, sel), "masks")
            rc, S = duplicate(c)
            assert rc == _lib.GSR_OK, _lib.lib().gsr_last_error()
            ws, wh, wsel, wS = dref.duplicate_rule(original, hid, sel, C3)
            assert (S, count_of(c)) == (wS, C3 + wS)
            np.testing.assert_array_equal(bits(store_of(c)), bits(ws), err_msg=f"duplicate {f}")
            gh, gsel = masks_of(c)
            np.testing.assert_array_equal(gh, wh)
            np.testing.assert_array_equal(gsel, wsel)


# ---- frames ----------------------------------------------------------------------------------------------------------------------
def frame_taps(c, vp, ub, planes=None):
    rgba = c.render(vp, ub)
    c.sync()
    t = c.taps()
    out = dict(rgba=rgba, stats=t["stats"], keys=t["keys"], values=t["values"], bounds=t["bounds"], records=t["records"])
    if planes:
        torch.cuda.synchronize()
        out.update({k: v.cpu().numpy() for k, v in planes.items()})
    return out


@pytest.mark.parametrize("variant", ["plain", "half", "depth_motion_ids"])
def test_frame_after_delete_is_the_frame_before(variant):
    splat60 = cloud(N)
    vp, ub = view()
    hid, sel = seeded_masks(M, 21, hidden=0.3, selected=0.15)
    hid[N:], sel[N:] = False, False
    planes = None
    with ShCtx(M, W, H, 0, _lib.GSR_FLAG_SH_HALF if variant == "half" else 0) as c:
        c.upload(splat60)
        _lib.check(set_masks(c, hid, sel), "masks")
        _lib.check(style(c, (1.0, 0.5, 0.0), 0.45), "style")
        if variant == "depth_motion_ids":
            planes = dict(d=torch.zeros(H, W, device="cuda"), m=torch.zeros(H, W, 2, device="cuda"),
                          i=torch.zeros(H, W, 2, dtype=torch.int32, device="cuda"))
            _lib.check(c.L.gsr_set_depth_compositing(c.h, None, C.c_void_p(planes["d"].data_ptr())), "depth")
            _lib.check(c.L.gsr_set_motion_vectors(c.h, C.c_void_p(planes["m"].data_ptr())), "motion")
            _lib.check(c.L.gsr_set_splat_ids(c.h, C.c_void_p(planes["i"].data_ptr())), "ids")
            c.render(vp, ub)
        before = frame_taps(c, vp, ub, planes)
        rc, k = delete(c)
        assert rc == _lib.GSR_OK and k == N - int(hid[:N].sum()) == count_of(c)
        after = frame_taps(c, vp, ub, planes)
    remap = delete_remap(hid, N)
    sb, sa = before["stats"], after["stats"]
    assert (sa.duplicates, sa.visible, sa.last_tile, sa.overflow) == (sb.duplicates, sb.visible, sb.last_tile, sb.overflow)
    assert sb.duplicates > 1000
    np.testing.assert_array_equal(bits(after["rgba"]), bits(before["rgba"]))
    np.testing.assert_array_equal(after["keys"], before["keys"])
    np.testing.assert_array_equal(after["bounds"], before["bounds"])
    old = before["values"].astype(np.int64)
    assert (remap[old] >= 0).all()
    np.testing.assert_array_equal(after["values"].astype(np.int64), remap[old])
    ids = np.unique(old)
    assert sel[ids].sum() > 20   # the highlight is drawn, and moves with its splats
    for w in REC_DTYPE.names:
        np.testing.assert_array_equal(bits(after["records"][w][remap[ids]]), bits(before["records"][w][ids]), err_msg=w)
    if planes:
        np.testing.assert_array_equal(bits(after["d"]), bits(before["d"]))
        np.testing.assert_array_equal(bits(after["m"]), bits(before["m"]))   # not motion
        bi, ai = before["i"].view(U32), after["i"].view(U32)
        drawn = bi[..., 0] != NO_ID
        assert drawn.sum() > 1000
        np.testing.assert_array_equal(ai[..., 0][drawn], remap[bi[..., 0][drawn]].astype(U32))
        np.testing.assert_array_equal(ai[..., 0][~drawn], bi[..., 0][~drawn])
        np.testing.assert_array_equal(ai[..., 1], bi[..., 1])


def _matrix_cases():
    from tests import variant_matrix as vm
    return range(len(vm.CASES)), vm.IDS


@pytest.mark.parametrize("i", _matrix_cases()[0], ids=_matrix_cases()[1])
def test_vacant_slots_are_hidden_splats_in_every_variant(i, monkeypatch):
    """A store with scattered vacant slots (written into the store as a delete leaves them) and no masks renders bit for bit the frame of
    the same store with those slots' splats hidden: every projection and compositor variant culls a vacant slot."""
    from tests import variant_matrix as vm
    from tests.test_gpu_variant_matrix import render_case
    case = vm.CASES[i]
    fr = vm.frame_of(case, MATRIX_N, (320, 192), (321, 181))
    vac = np.random.default_rng(500 + i).random(fr.n) < 0.2
    none = np.zeros(fr.n, dtype=bool)
    want = render_masked_case(fr, vac, none)
    plain_upload = ShCtx.upload

    def vacant_upload(self, splat60, first=0):
        plain_upload(self, splat60, first)
        store = store_of(self)
        dref.vacate_slots(store, vac)
        restore_host(self, store)

    monkeypatch.setattr(ShCtx, "upload", vacant_upload)
    got = render_case(fr)
    sg, sw = got["stats"], want["stats"]
    assert (sg.duplicates, sg.visible, sg.last_tile, sg.overflow, sg.staged) == (sw.duplicates, sw.visible, sw.last_tile, sw.overflow, sw.staged)
    assert sw.visible > 100
    np.testing.assert_array_equal(got["keys"], want["keys"])
    np.testing.assert_array_equal(got["values"], want["values"])
    np.testing.assert_array_equal(got["bounds"], want["bounds"])
    ids = np.unique(want["values"])
    for w in ("image_pos", "pos_xy", "conic", "pos_z", "color"):
        np.testing.assert_array_equal(bits(got["records"][w][ids]), bits(want["records"][w][ids]), err_msg=w)
    np.testing.assert_array_equal(bits(got["rgba"]), bits(want["rgba"]))
    for k in ("depth", "motion"):
        assert (got[k] is None) == (want[k] is None)
        if got[k] is not None:
            np.testing.assert_array_equal(bits(got[k]), bits(want[k]))


def test_vacant_slots_in_a_shard_group():
    """A 2-rank shard group in one process on a store with vacant slots: its frames, pairs, V and last tile are the single-context
    ones, which equal the frames of the same store with those slots hidden (tests/group_vacancy_worker.py)."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32")
    res = subprocess.run([sys.executable, os.path.join(root, "tests", "group_vacancy_worker.py")], capture_output=True, text=True, timeout=600,
                         cwd=root, env=env)
    assert res.returncode == 0 and "GROUP_VACANCY_OK" in res.stdout, res.stdout[-2000:] + res.stderr[-4000:]


# ---- duplicate ---------------------------------------------------------------------------------------------------------------
def test_duplicate_then_hide_is_the_previous_frame():
    splat60 = cloud(N)
    vp, ub = view()
    hid, sel = seeded_masks(M, 5, hidden=0.1, selected=0.15)
    hid[N:], sel[N:] = False, False
    with ShCtx(M, W, H) as c:
        c.upload(splat60)
        _lib.check(set_masks(c, hid, sel), "masks")
        _lib.check(style(c, (1.0, 0.5, 0.0), 0.0), "style")
        want = c.render(vp, ub)
        rc, S = duplicate(c)
        assert rc == _lib.GSR_OK and S == int(sel[:N].sum()) == count_of(c) - N
        assert not np.array_equal(bits(c.render(vp, ub)), bits(want))   # the copies sit on their originals
        _lib.check(c.L.gsr_hide_selection(c.h), "hide the copies")
        np.testing.assert_array_equal(bits(c.render(vp, ub)), bits(want))


def test_duplicate_and_move_is_the_rule_edited_store():
    splat60 = cloud(N)
    vp, ub = view()
    hid, sel = seeded_masks(M, 6, hidden=0.1, selected=0.1)
    hid[N:], sel[N:] = False, False
    move = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0.4, -0.2, 0.1], dtype=np.float32)
    with ShCtx(M, W, H) as c, ShCtx(M, W, H) as r:
        for x in (c, r):
            x.upload(splat60)
            _lib.check(set_masks(x, hid, sel), "masks")
            _lib.check(style(x, (0.2, 0.4, 1.0), 0.3), "style")
        before = store_of(c)
        rc, S = duplicate(c)
        assert rc == _lib.GSR_OK
        _lib.check(c.L.gsr_transform_selection(c.h, move.ctypes.data_as(C.POINTER(C.c_float)), None), "move the copies")
        m95 = c.copy(_lib.GSR_BUF_EDIT_TRANSFORM, 95, np.float32)
        ds, dh, dsel, dS = dref.duplicate_rule(before, hid, sel, N)
        want_store = tref.oracle(ds, 4, False, dsel, m95)
        tref.assert_store_equal(store_of(c), want_store, False, "duplicate + move")
        restore_host(r, want_store)
        _lib.check(c.L.gsr_set_splat_count(r.h, N + S), "count")
        _lib.check(set_masks(r, dh, dsel), "masks")
        np.testing.assert_array_equal(bits(c.render(vp, ub)), bits(r.render(vp, ub)))


def test_copies_outside_the_instance_ranges_are_not_drawn():
    splat60 = cloud(N)
    vp, ub = view()
    hid, sel = seeded_masks(M, 7, hidden=0.0, selected=0.2)
    hid[N:], sel[N:] = False, False
    with ShCtx(M, W, H) as c:
        c.upload(splat60)
        set_instances(c, [(0, N, rigid(4)), (100, 5000, rigid(6))])
        _lib.check(set_masks(c, hid, sel), "masks")
        _lib.check(style(c, (1.0, 0.5, 0.0), 0.0), "style")
        want = c.render(vp, ub)
        rc, S = duplicate(c)
        assert rc == _lib.GSR_OK and S > 0
        np.testing.assert_array_equal(bits(c.render(vp, ub)), bits(want))


# ---- undo --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("edit", ["delete", "duplicate"])
def test_undo_is_exact(edit):
    splat60 = cloud(N)
    vp, ub = view()
    hid, sel = seeded_masks(M, 8, hidden=0.25, selected=0.1)
    hid[N:], sel[N:] = False, False
    with ShCtx(M, W, H) as c:
        c.upload(splat60)
        _lib.check(set_masks(c, hid, sel), "masks")
        _lib.check(style(c, (1.0, 0.5, 0.0), 0.4), "style")
        frame0 = c.render(vp, ub)
        table0 = store_to_table(store_of(c), count_of(c), 4, False, masks_of(c)[0][:count_of(c)])
        snap = torch.empty(int(c.L.gsr_splat_store_bytes(c.h)), dtype=torch.uint8, device="cuda")
        _lib.check(c.L.gsr_copy_splat_store(c.h, C.c_void_p(snap.data_ptr())), "snapshot")
        h0, s0, n0 = pack_mask(hid, M), pack_mask(sel, M), count_of(c)
        rc, _ = delete(c) if edit == "delete" else duplicate(c)
        assert rc == _lib.GSR_OK
        if edit == "delete":   # the kept table of the compacted cloud is the kept table before the delete
            t = store_to_table(store_of(c), count_of(c), 4, False, masks_of(c)[0][:count_of(c)])
            np.testing.assert_array_equal(bits(t), bits(table0))
        _lib.check(c.L.gsr_restore_splat_store(c.h, C.c_void_p(snap.data_ptr())), "restore")
        _lib.check(c.L.gsr_set_splat_masks(c.h, h0.ctypes.data_as(U32P), s0.ctypes.data_as(U32P), h0.size), "masks")
        _lib.check(c.L.gsr_set_splat_count(c.h, n0), "count")
        np.testing.assert_array_equal(bits(c.render(vp, ub)), bits(frame0))
        t = store_to_table(store_of(c), count_of(c), 4, False, masks_of(c)[0][:count_of(c)])
        np.testing.assert_array_equal(bits(t), bits(table0))


# ---- ordering between asynchronous frames ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("pipeline", [0, 1])
def test_edits_between_asynchronous_frames(pipeline):
    """Frames enqueued before a delete or duplicate show the old cloud, frames after it the new one (each against a context that
    renders the same cloud synchronously)."""
    splat60 = cloud(N)
    vp, ub = view()
    hid, sel = seeded_masks(M, 9, hidden=0.2, selected=0.1)
    hid[N:], sel[N:] = False, False
    move = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0.3, 0.2, 0.0], dtype=np.float32)
    with ShCtx(M, W, H) as c, ShCtx(M, W, H) as r:
        for x in (c, r):
            x.upload(splat60)
            _lib.check(set_masks(x, hid, sel), "masks")
            _lib.check(style(x, (1.0, 0.5, 0.0), 0.4), "style")
        _lib.check(c.L.gsr_debug_pipeline(c.h, pipeline), "pipeline")
        want = [r.render(vp, ub)]
        host = [torch.empty((H, W, 4), dtype=torch.float32).pin_memory() for _ in range(6)]
        c.render_async(vp, ub, host_ptr=host[0].data_ptr())
        c.render_async(vp, ub, host_ptr=host[1].data_ptr())
        rc, k = delete(c)
        assert rc == _lib.GSR_OK
        c.render_async(vp, ub, host_ptr=host[2].data_ptr())
        rc, S = duplicate(c)
        assert rc == _lib.GSR_OK and S == int(sel[:N].sum())
        _lib.check(c.L.gsr_transform_selection(c.h, move.ctypes.data_as(C.POINTER(C.c_float)), None), "move")
        c.render_async(vp, ub, host_ptr=host[3].data_ptr())
        c.render_async(vp, ub, host_ptr=host[4].data_ptr())
        c.sync()
        final = store_of(c)
        fh, fsel = masks_of(c)
        restore_host(r, final)
        _lib.check(r.L.gsr_set_splat_count(r.h, count_of(c)), "count")
        _lib.check(set_masks(r, fh, fsel), "masks")
        want_after = r.render(vp, ub)
        torch.cuda.synchronize()
        for i in (0, 1, 2):
            np.testing.assert_array_equal(bits(host[i].numpy()), bits(want[0]), err_msg=f"frame {i}")
        for i in (3, 4):
            np.testing.assert_array_equal(bits(host[i].numpy()), bits(want_after), err_msg=f"frame {i}")
        assert not np.array_equal(bits(want_after), bits(want[0]))


# ---- errors ----------------------------------------------------------------------------------------------------------------------
def test_refusals_leave_everything_unchanged():
    splat60 = cloud(N)
    m = N + 500
    hid, sel = seeded_masks(m, 10, hidden=0.1, selected=0.2)
    hid[N:], sel[N:] = False, False
    with ShCtx(m, W, H) as c:
        c.upload(splat60)
        k = C.c_uint64(0)
        assert c.L.gsr_delete_hidden(c.h, None) == _lib.GSR_ERR_INVALID
        assert c.L.gsr_delete_hidden(c.h, C.byref(k)) == _lib.GSR_ERR_STATE          # masks not in use
        assert c.L.gsr_duplicate_selection(c.h, None) == _lib.GSR_ERR_INVALID
        assert c.L.gsr_duplicate_selection(c.h, C.byref(k)) == _lib.GSR_ERR_STATE
        assert c.L.gsr_set_splat_count(c.h, m + 1) == _lib.GSR_ERR_INVALID
        _lib.check(set_masks(c, hid, sel), "masks")
        store0 = store_of(c)
        set_instances(c, [(0, N, rigid(4))])
        assert c.L.gsr_delete_hidden(c.h, C.byref(k)) == _lib.GSR_ERR_STATE          # instances set
        assert b"instances" in _lib.lib().gsr_last_error()
        S = int(sel[:N].sum())
        assert S > 500
        assert c.L.gsr_duplicate_selection(c.h, C.byref(k)) == _lib.GSR_ERR_INVALID   # N + S > max_splats
        msg = _lib.lib().gsr_last_error().decode()
        assert str(S) in msg and "500" in msg
        assert k.value == 0 and count_of(c) == N
        np.testing.assert_array_equal(bits(store_of(c)), bits(store0))
        gh, gs = masks_of(c)
        np.testing.assert_array_equal(gh, hid)
        np.testing.assert_array_equal(gs, sel)
        _lib.check(c.L.gsr_set_splat_count(c.h, m), "count up to max_splats")
        assert count_of(c) == m


# ---- the Python mirror -----------------------------------------------------------------------------------------------------------
def test_python_mirror_and_kept_table():
    """GaussianSplattingRasterizer: hide a lasso, delete_hidden, and kept_table() exports what it exported before the delete; then a
    duplicate into the freed slots and set_splat_count for undo."""
    from godotgaussiansplatting_b200 import camera as cam
    from godotgaussiansplatting_b200.rasterizer import GaussianSplattingRasterizer
    from godotgaussiansplatting_b200.synthetic import synthetic_ply
    n = 3001
    r = GaussianSplattingRasterizer(synthetic_ply(n, 4), (160, 96), None, cam.orbit_camera(25, aspect=160 / 96))
    r.init_gpu()
    try:
        r.select_polygon([[0, 0], [159, 0], [159, 40], [0, 40]], _lib.GSR_SELECT_SET)
        r.hide_selection()
        hid, _ = r.splat_masks()
        assert 100 < int(hid.sum()) < n - 100
        before = r.kept_table()
        r.rasterize()
        k = r.delete_hidden()
        assert k == n - int(hid.sum()) == int(r.stats().num_splats) == before.shape[0]
        np.testing.assert_array_equal(bits(r.kept_table()), bits(before))
        r.rasterize()
        sel = np.zeros(n, dtype=bool)
        sel[np.random.default_rng(4).choice(k, 60, replace=False)] = True
        r.set_splat_masks(np.zeros(n, dtype=bool), sel)
        S = r.duplicate_selection()
        assert 0 < S == int(sel.sum()) <= n - k and int(r.stats().num_splats) == k + S
        _, sel2 = r.splat_masks()
        np.testing.assert_array_equal(np.flatnonzero(sel2), np.arange(k, k + S))
        table = r.kept_table()
        np.testing.assert_array_equal(bits(table[:k]), bits(before))
        np.testing.assert_array_equal(bits(table[k:]), bits(before[np.flatnonzero(sel[:k])]))
        r.set_splat_count(k)
        np.testing.assert_array_equal(bits(r.kept_table()), bits(before))
        with pytest.raises(_lib.GsrError):
            r.set_splat_count(n + 1)
    finally:
        r.cleanup_gpu()
