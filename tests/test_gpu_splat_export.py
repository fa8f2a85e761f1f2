"""Splat export on the GPU (include/gsr.h "Splat export"), through the C-ABI: the rule of tests/export_reference for every store format,
scope and degree; equal bits across calls, destinations and edits that move splats (delete, duplicate); a CONNECTED selection; an export
enqueued behind asynchronous edits; the capacity, count-only and argument rules; a partial band with the masks out of use; the Python
mirror's save / parse / upload round trip; a c3-size export."""
import ctypes as C
import os

import numpy as np
import pytest

from godotgaussiansplatting_b200 import _lib
from godotgaussiansplatting_b200.ply_file import PlyFile, degree_properties
from tests import export_reference as xr
from tests.test_gpu_sh_degree import ShCtx
from tests.test_gpu_splat_selection import set_masks
from tests.test_splat_export import cloud

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

U32 = np.uint32
U32P = C.POINTER(C.c_uint32)
KEPT, SELECTED = _lib.GSR_EXPORT_KEPT, _lib.GSR_EXPORT_SELECTED


def stride_of(m):
    return (m + 255) // 256 * 256


def bits(a):
    return np.ascontiguousarray(a).view(U32)


def load(c, store, n):
    s = np.ascontiguousarray(store, dtype=np.float32)
    _lib.check(c.L.gsr_restore_splat_store(c.h, C.c_void_p(s.ctypes.data)), "gsr_restore_splat_store")
    _lib.check(c.L.gsr_set_splat_count(c.h, n), "gsr_set_splat_count")


def count(c, scope, degree=-1):
    r = C.c_uint64(0)
    rc = c.L.gsr_export_ply(c.h, scope, degree, None, 0, C.byref(r))
    return rc, int(r.value)


def export(c, scope, degree, stored_degree):
    """The rows, into pageable host memory."""
    rc, n = count(c, scope, degree)
    assert rc == _lib.GSR_OK, _lib.lib().gsr_last_error()
    d = stored_degree if degree < 0 else degree
    out = np.full((n, xr.row_floats(d)), np.nan, dtype=np.float32)
    r = C.c_uint64(0)
    if n:
        _lib.check(c.L.gsr_export_ply(c.h, scope, degree, C.c_void_p(out.ctypes.data), n, C.byref(r)), "gsr_export_ply")
        assert r.value == n
    return out


def store_of(c):
    nbytes = int(c.L.gsr_splat_store_bytes(c.h))
    return c.copy(_lib.GSR_BUF_SPLATS, nbytes // 4, np.float32).reshape(-1, stride_of(c.max_splats), 4)


def masks_of(c):
    from godotgaussiansplatting_b200.rasterizer import unpack_mask
    words = (c.max_splats + 31) // 32
    h, s = np.zeros(words, U32), np.zeros(words, U32)
    _lib.check(c.L.gsr_get_splat_masks(c.h, h.ctypes.data_as(U32P), s.ctypes.data_as(U32P), words), "gsr_get_splat_masks")
    return unpack_mask(h, c.max_splats), unpack_mask(s, c.max_splats)


M, N = 40_000 + 45, 40_000 - 19   # max_splats and n: not multiples of 32, n below max_splats


@pytest.mark.parametrize("bands", [1, 2, 3, 4])
@pytest.mark.parametrize("half", [False, True])
def test_rule_on_the_device(bands, half):
    rng = np.random.default_rng(bands * 10 + half)
    store = cloud(rng, bands, half, M, N)
    hid = rng.random(M) < 0.3
    sel = (rng.random(M) < 0.4) & ~hid
    with ShCtx(M, 64, 64, bands, _lib.GSR_FLAG_SH_HALF if half else 0) as c:
        load(c, store, N)
        for degree in [-1] + list(range(bands)):
            d = bands - 1 if degree < 0 else degree
            xr.check_rows(export(c, KEPT, degree, bands - 1), store, N, bands, half, None, None, False, d)   # masks not in use
            assert count(c, SELECTED, degree) == (_lib.GSR_OK, 0)
        _lib.check(set_masks(c, hid, sel), "masks")
        for degree in range(bands):
            for scope in (KEPT, SELECTED):
                rows = export(c, scope, degree, bands - 1)
                xr.check_rows(rows, store, N, bands, half, hid, sel, scope == SELECTED, degree)
                if degree == bands - 1:   # the exact columns equal the emulated kernel's
                    emu = xr.emu_export(store, bands, half, hid, sel, N, scope == SELECTED, degree)
                    k = degree_properties(degree).index("opacity")
                    np.testing.assert_array_equal(bits(rows[:, :k]), bits(emu[:, :k]))


def test_bits_repeat_across_calls_and_destinations():
    """Two calls give equal bits; device, page-locked and pageable destinations give equal bytes; count-only mode; a dst one row too
    small is refused with the count named, and the sentinel-filled buffer left intact."""
    rng = np.random.default_rng(5)
    store = cloud(rng, 4, False, M, N)
    hid = rng.random(M) < 0.1
    with ShCtx(M, 64, 64, 4) as c:
        load(c, store, N)
        _lib.check(set_masks(c, hid, np.zeros(M, dtype=bool)), "masks")
        a, b = export(c, KEPT, -1, 3), export(c, KEPT, -1, 3)
        np.testing.assert_array_equal(bits(a), bits(b))
        rows = a.shape[0]
        assert count(c, KEPT) == (_lib.GSR_OK, rows)
        dev = torch.empty((rows + 1) * 62, dtype=torch.float32, device="cuda")
        r = C.c_uint64(0)
        _lib.check(c.L.gsr_export_ply(c.h, KEPT, -1, C.c_void_p(dev.data_ptr()), rows + 1, C.byref(r)), "device")
        torch.cuda.synchronize()
        assert r.value == rows
        np.testing.assert_array_equal(bits(dev[:rows * 62].cpu().numpy().reshape(rows, 62)), bits(a))
        pinned = torch.empty(rows * 62, dtype=torch.float32).pin_memory()
        _lib.check(c.L.gsr_export_ply(c.h, KEPT, -1, C.c_void_p(pinned.data_ptr()), rows, C.byref(r)), "pinned")
        np.testing.assert_array_equal(bits(pinned.numpy().reshape(rows, 62)), bits(a))
        # too small: refused, nothing written, the count still returned and named
        sentinel = np.full((rows - 1, 62), -7.0, dtype=np.float32)
        r = C.c_uint64(0)
        assert c.L.gsr_export_ply(c.h, KEPT, -1, C.c_void_p(sentinel.ctypes.data), rows - 1, C.byref(r)) == _lib.GSR_ERR_INVALID
        assert r.value == rows and str(rows) in _lib.lib().gsr_last_error().decode()
        assert (sentinel == -7.0).all()
        dev.fill_(-7.0)
        assert c.L.gsr_export_ply(c.h, KEPT, -1, C.c_void_p(dev.data_ptr()), rows - 1, C.byref(r)) == _lib.GSR_ERR_INVALID
        assert bool((dev == -7.0).all())


def test_delete_duplicate_and_connected_selection():
    """Export before gsr_delete_hidden equals export after it; the copies of a duplicate export the originals' rows; a SELECTED export
    after a CONNECTED neighbourhood selection is those splats' KEPT rows."""
    rng = np.random.default_rng(6)
    m = n = 12_000 + 7
    store = cloud(rng, 3, True, m, n, specials=False)
    store[0, :n, :3] = rng.normal(size=(n, 3)) * 0.05 + np.where(np.arange(n) < n // 2, 0.0, 50.0)[:, None]   # two separate blobs
    hid = rng.random(m) < 0.2
    with ShCtx(m + 4000, 64, 64, 3, _lib.GSR_FLAG_SH_HALF) as c:
        M2 = c.max_splats
        full = np.zeros((store.shape[0], stride_of(M2), 4), dtype=np.float32)
        full[:, :store.shape[1]] = store
        load(c, full, n)
        h = np.zeros(M2, dtype=bool)
        h[:m] = hid
        _lib.check(set_masks(c, h, np.zeros(M2, dtype=bool)), "masks")
        before = export(c, KEPT, -1, 2)
        k = C.c_uint64(0)
        _lib.check(c.L.gsr_delete_hidden(c.h, C.byref(k)), "delete")
        after = export(c, KEPT, -1, 2)
        np.testing.assert_array_equal(bits(after), bits(before))
        # duplicate: the selection's rows before == the copies' rows after
        sel = np.zeros(M2, dtype=bool)
        sel[rng.choice(k.value, 500, replace=False)] = True
        _lib.check(set_masks(c, np.zeros(M2, dtype=bool), sel), "masks")
        originals = export(c, SELECTED, -1, 2)
        S = C.c_uint64(0)
        _lib.check(c.L.gsr_duplicate_selection(c.h, C.byref(S)), "duplicate")
        assert S.value == 500
        np.testing.assert_array_equal(bits(export(c, SELECTED, -1, 2)), bits(originals))
        # CONNECTED from one seed in the second blob: its rows are exactly the KEPT rows of the selected splats
        _lib.check(c.L.gsr_set_splat_count(c.h, k.value), "count")
        seed = np.zeros(M2, dtype=bool)
        pos = store_of(c)[0, :k.value, 0]
        seed[int(np.flatnonzero(pos > 25.0)[0])] = True
        _lib.check(set_masks(c, np.zeros(M2, dtype=bool), seed), "masks")
        q = _lib.GsrNeighborhood(_lib.GSR_NEIGHBOR_CONNECTED, 1.0, 1, -1)
        _lib.check(c.L.gsr_select_neighborhood(c.h, C.byref(q), _lib.GSR_SELECT_SET, None), "connected")
        _, chosen = masks_of(c)
        assert 1000 < int(chosen.sum()) < k.value - 1000
        kept = export(c, KEPT, -1, 2)
        alive = xr.exported(store_of(c), k.value, np.zeros(M2, dtype=bool), None, False)
        want = kept[np.isin(alive, np.flatnonzero(chosen))]
        np.testing.assert_array_equal(bits(export(c, SELECTED, -1, 2)), bits(want))
        np.testing.assert_array_equal(bits(export(c, SELECTED, 0, 2)), bits(xr.narrow(want, 2, 0)))


def test_export_sees_asynchronous_edits():
    """An export enqueued right behind gsr_transform_selection / gsr_recolor_selection (no host sync between) sees the edit."""
    rng = np.random.default_rng(7)
    store = cloud(rng, 4, False, M, N, specials=False)
    with ShCtx(M, 64, 64, 4) as c:
        load(c, store, N)
        sel = rng.random(M) < 0.5
        _lib.check(set_masks(c, np.zeros(M, dtype=bool), sel), "masks")
        before = export(c, KEPT, -1, 3)
        L = (C.c_float * 12)(*[0.0, 0.0, 1.0, 1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.5, -2.0, 3.0])
        _lib.check(c.L.gsr_transform_selection(c.h, L, None), "transform")
        got = export(c, KEPT, -1, 3)
        c.sync()
        settled = export(c, KEPT, -1, 3)
        np.testing.assert_array_equal(bits(got), bits(settled))
        xr.check_rows(got, store_of(c), N, 4, False, None, None, False, 3)
        moved = sel[xr.exported(store, N, None, None, False)]
        assert not np.array_equal(bits(got[moved, :3]), bits(before[moved, :3]))
        np.testing.assert_array_equal(bits(got[~moved]), bits(before[~moved]))
        e = _lib.GsrColorEdit()
        e.matrix[:] = [0.5, 0, 0, 0, 0.5, 0, 0, 0, 0.5, 0.1, 0.1, 0.1]
        e.band_scale[:] = [0.0, 0.0, 0.0]
        e.opacity_scale, e.opacity_offset = 0.5, 0.0
        _lib.check(c.L.gsr_recolor_selection(c.h, C.byref(e), None), "recolor")
        got = export(c, KEPT, -1, 3)
        c.sync()
        np.testing.assert_array_equal(bits(got), bits(export(c, KEPT, -1, 3)))
        assert (got[moved, 9:54] == 0.0).all()   # band_scale 0 flattened the selected splats' f_rest


def test_partial_band_masks_out_of_use_and_refusals():
    rng = np.random.default_rng(8)
    m = n = 5000
    store = cloud(rng, 4, False, m, n, specials=False)   # a full float store: a lower-degree or binary16 one cannot be banded
    with ShCtx(m, 64, 64, 4) as c:
        load(c, store, n)
        r = C.c_uint64(99)
        for scope, degree in ((2, -1), (-1, -1), (KEPT, -2), (KEPT, 4), (SELECTED, 5)):
            assert c.L.gsr_export_ply(c.h, scope, degree, None, 0, C.byref(r)) == _lib.GSR_ERR_INVALID
        assert r.value == 99
        assert c.L.gsr_export_ply(c.h, KEPT, -1, None, 0, None) == _lib.GSR_ERR_INVALID
        rows = export(c, KEPT, -1, 3)
        # the export left the masks out of use: a partial band (a sharded context) is still accepted, and export runs there too
        assert c.L.gsr_set_band(c.h, 0, 2) == _lib.GSR_OK, _lib.lib().gsr_last_error()
        np.testing.assert_array_equal(bits(export(c, KEPT, -1, 3)), bits(rows))
        np.testing.assert_array_equal(bits(export(c, KEPT, 1, 3)), bits(xr.narrow(rows, 3, 1)))
        assert count(c, SELECTED) == (_lib.GSR_OK, 0)


def test_python_mirror_round_trip(tmp_path):
    """export_ply().save(), PlyFile parse, upload into a second context: positions and coefficients bit for bit, opacity within 2 ulp
    (exact at 0 and 1), covariance words within 1e-5 lambda_max."""
    from godotgaussiansplatting_b200 import camera as cam
    from godotgaussiansplatting_b200.rasterizer import GaussianSplattingRasterizer
    from godotgaussiansplatting_b200.synthetic import synthetic_ply
    n = 20_001
    for half in (False, True):
        r = GaussianSplattingRasterizer(synthetic_ply(n, 4), (160, 96), None, cam.orbit_camera(25, aspect=160 / 96), sh_half=half)
        r.init_gpu(device_ingest=True)
        r2 = None
        try:
            hid = np.zeros(n, dtype=bool)
            hid[::7] = True
            r.set_splat_masks(hid, np.zeros(n, dtype=bool))
            ply = r.export_ply()
            assert ply.properties == degree_properties(3) and ply.size == n - int(hid.sum())
            path = os.path.join(tmp_path, f"export{int(half)}.ply")
            ply.save(path)
            back = PlyFile(path)
            np.testing.assert_array_equal(bits(back.table), bits(ply.table))
            np.testing.assert_array_equal(bits(r.export_ply(sh_degree=1).table), bits(xr.narrow(ply.table, 3, 1)))
            r2 = GaussianSplattingRasterizer(back, (160, 96), None, cam.orbit_camera(25, aspect=160 / 96), sh_half=half)
            r2.init_gpu(device_ingest=True)
            a = store_of_r(r)[:, np.flatnonzero(~hid)]
            b = store_of_r(r2)[:, :back.size]
            np.testing.assert_array_equal(bits(b[0, :, :3]), bits(a[0, :, :3]))
            np.testing.assert_array_equal(bits(b[3:]), bits(a[3:]))
            assert xr.ulp_distance(a[2, :, 2], b[2, :, 2]).max() <= 2
            idx = np.arange(back.size)
            S, S2 = xr.covariances(a, idx), xr.covariances(b, idx)
            lmax = np.abs(np.linalg.eigvalsh(S)).max(axis=1)
            assert (np.abs(S2 - S).max(axis=(1, 2)) <= 1e-5 * lmax).all()
        finally:
            r.cleanup_gpu()
            if r2 is not None:
                r2.cleanup_gpu()


def store_of_r(r):
    nbytes = r.splat_store_bytes()
    stride = (r._max_splats + 255) // 256 * 256
    return r.debug_copy(_lib.GSR_BUF_SPLATS, nbytes // 4, np.float32).reshape(-1, stride, 4)


def test_c3_size_export():
    """6 M splats of a degree-3 store with 10 % hidden: the row count equals the host's count, positions and coefficients are the
    store's, and a sample of rows meets the decomposition's bars."""
    n = 6_000_000
    rng = np.random.default_rng(9)
    store = cloud(rng, 4, False, n, n, specials=False)
    hid = rng.random(n) < 0.1
    with ShCtx(n, 64, 64, 4) as c:
        load(c, store, n)
        _lib.check(set_masks(c, hid, np.zeros(n, dtype=bool)), "masks")
        dev = torch.empty(n * 62, dtype=torch.float32, device="cuda")
        r = C.c_uint64(0)
        _lib.check(c.L.gsr_export_ply(c.h, KEPT, -1, C.c_void_p(dev.data_ptr()), n, C.byref(r)), "export")
        torch.cuda.synchronize()
        idx = xr.exported(store, n, hid, None, False)
        assert r.value == idx.size
        rows = dev[:idx.size * 62].cpu().numpy().reshape(idx.size, 62)
        np.testing.assert_array_equal(bits(rows[:, :3]), bits(store[0, idx, :3]))
        sh = xr.sh_values(store, n, 4, False)[idx]
        np.testing.assert_array_equal(bits(rows[:, 6:9]), bits(sh[:, 0:3]))
        np.testing.assert_array_equal(bits(rows[:, 9:54]), bits(sh[:, 3:].reshape(-1, 15, 3).transpose(0, 2, 1).reshape(-1, 45)))
        pick = np.sort(rng.choice(idx.size, 100_000, replace=False))
        sub = store[:, idx[pick]]
        xr.check_rows(rows[pick], sub, pick.size, 4, False, None, None, False, 3)
