"""Compressed PLY on the GPU (include/gsr.h "Compressed PLY"), through the C-ABI: the export rule of tests/compressed_reference for every
store format, scope, degree and order; equal bits across calls, destinations and a delete; uploads of reference-encoded files into every
store format, at an offset, in chunk-aligned pieces and from device memory; count-only mode, the capacity refusal and the argument
refusals; an export behind asynchronous edits; the Python save / parse / constructor round trip; a c3-size export and re-upload."""
import ctypes as C
import os

import numpy as np
import pytest

from godotgaussiansplatting_b200 import _lib
from godotgaussiansplatting_b200.compressed_ply import CompressedPlyFile
from tests import compressed_reference as cref
from tests import export_reference as xr
from tests.test_gpu_sh_degree import ShCtx
from tests.test_gpu_splat_export import bits, load, store_of, store_of_r, stride_of
from tests.test_gpu_splat_selection import set_masks
from tests.test_splat_export import cloud
from tests.transform_reference import sh_planes

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

U32 = np.uint32
KEPT, SELECTED = _lib.GSR_EXPORT_KEPT, _lib.GSR_EXPORT_SELECTED
STORE, MORTON = _lib.GSR_COMPRESS_STORE_ORDER, _lib.GSR_COMPRESS_MORTON


def count(c, scope=KEPT, degree=-1, order=MORTON):
    r = C.c_uint64(0)
    rc = c.L.gsr_export_compressed_ply(c.h, scope, degree, order, None, C.byref(r))
    return rc, int(r.value)


def host_file(rows, degree, alloc=np.empty):
    return dict(chunks=alloc((cref.chunk_count(rows), 18), dtype=np.float32), packed=alloc((rows, 4), dtype=U32),
                sh=alloc((rows, cref.sh_bytes(degree)), dtype=np.uint8))


def descriptor(ptrs, rows, degree, chunk_floats=18, chunk_count=None):
    return _lib.GsrCompressedPly(ptrs[0], ptrs[1], ptrs[2] if degree else None, rows,
                                 cref.chunk_count(rows) if chunk_count is None else chunk_count, degree, chunk_floats)


def export(c, scope, degree, order, stored_degree):
    """The file, into pageable host memory: dict(count, chunks, packed, sh)."""
    rc, n = count(c, scope, degree, order)
    assert rc == _lib.GSR_OK, _lib.lib().gsr_last_error()
    d = stored_degree if degree < 0 else degree
    f = host_file(n, d)
    if n:
        dst = descriptor([f[k].ctypes.data for k in ("chunks", "packed", "sh")], n, d)
        r = C.c_uint64(0)
        _lib.check(c.L.gsr_export_compressed_ply(c.h, scope, degree, order, C.byref(dst), C.byref(r)), "gsr_export_compressed_ply")
        assert r.value == n and dst.rows == n and dst.chunk_count == cref.chunk_count(n) and dst.sh_degree == d and dst.chunk_floats == 18
    f["count"] = n
    return f


def check(f, ref):
    assert f["count"] == ref["idx"].size
    np.testing.assert_array_equal(bits(f["chunks"]), bits(ref["chunks"]))
    np.testing.assert_array_equal(f["packed"], ref["packed"])
    np.testing.assert_array_equal(f["sh"], ref["sh"])


def upload(c, f, rows, degree, first=0, creation_time=0.0, chunk_floats=18):
    ch = np.ascontiguousarray(f["chunks"][:, :chunk_floats])
    src = descriptor([ch.ctypes.data, f["packed"].ctypes.data, f["sh"].ctypes.data if degree else None], rows, degree, chunk_floats)
    return c.L.gsr_upload_compressed_ply(c.h, C.byref(src), first, creation_time)


M, N = 12_000 + 45, 12_000 - 19   # max_splats and n: not multiples of 32 or 256


@pytest.mark.parametrize("bands", [1, 2, 3, 4])
@pytest.mark.parametrize("half", [False, True])
def test_rule_on_the_device(bands, half):
    rng = np.random.default_rng(bands * 10 + half)
    store = cloud(rng, bands, half, M, N)
    hid = rng.random(M) < 0.3
    sel = (rng.random(M) < 0.4) & ~hid
    sr = cref.scale_rot(store, bands, half, N)
    with ShCtx(M, 64, 64, bands, _lib.GSR_FLAG_SH_HALF if half else 0) as c:
        load(c, store, N)
        for order in (STORE, MORTON):
            check(export(c, KEPT, -1, order, bands - 1), cref.encode(store, N, bands, half, None, None, False, bands - 1, order, sr))
            assert count(c, SELECTED, -1, order) == (_lib.GSR_OK, 0)
        _lib.check(set_masks(c, hid, sel), "masks")
        for degree in range(bands):
            for scope in (KEPT, SELECTED):
                for order in (STORE, MORTON):
                    ref = cref.encode(store, N, bands, half, hid, sel, scope == SELECTED, degree, order, sr)
                    check(export(c, scope, degree, order, bands - 1), ref)


def test_destinations_calls_delete_and_refusals():
    """Equal bits across calls and device, page-locked and pageable destinations; count-only mode; a dst one row too small is refused,
    untouched; the argument refusals; after gsr_delete_hidden the STORE-order file is unchanged and its rows are gsr_export_ply's."""
    rng = np.random.default_rng(5)
    store = cloud(rng, 4, False, M, N)
    hid = rng.random(M) < 0.1
    with ShCtx(M, 64, 64, 4) as c:
        load(c, store, N)
        _lib.check(set_masks(c, hid, np.zeros(M, dtype=bool)), "masks")
        a, b = export(c, KEPT, -1, MORTON, 3), export(c, KEPT, -1, MORTON, 3)
        for k in ("chunks", "packed", "sh"):
            np.testing.assert_array_equal(bits(a[k]) if k == "chunks" else a[k], bits(b[k]) if k == "chunks" else b[k])
        n = a["count"]
        r = C.c_uint64(0)
        for alloc in ("device", "pinned"):
            if alloc == "device":
                t = dict(chunks=torch.full((cref.chunk_count(n), 18), -7.0, device="cuda"), packed=torch.zeros((n, 4), dtype=torch.int32, device="cuda"),
                         sh=torch.zeros((n, 45), dtype=torch.uint8, device="cuda"))
            else:
                t = dict(chunks=torch.zeros((cref.chunk_count(n), 18)).pin_memory(), packed=torch.zeros((n, 4), dtype=torch.int32).pin_memory(),
                         sh=torch.zeros((n, 45), dtype=torch.uint8).pin_memory())
            dst = descriptor([t[k].data_ptr() for k in ("chunks", "packed", "sh")], n, 3)
            _lib.check(c.L.gsr_export_compressed_ply(c.h, KEPT, -1, MORTON, C.byref(dst), C.byref(r)), alloc)
            torch.cuda.synchronize()
            assert r.value == n
            np.testing.assert_array_equal(bits(t["chunks"].cpu().numpy()), bits(a["chunks"]))
            np.testing.assert_array_equal(t["packed"].cpu().numpy().view(U32), a["packed"])
            np.testing.assert_array_equal(t["sh"].cpu().numpy(), a["sh"])
        # too small: refused, nothing written, the count returned and named
        small = host_file(n - 1, 3, alloc=lambda shape, dtype: np.full(shape, 7, dtype=dtype))
        dst = descriptor([small[k].ctypes.data for k in ("chunks", "packed", "sh")], n - 1, 3)
        r = C.c_uint64(0)
        assert c.L.gsr_export_compressed_ply(c.h, KEPT, -1, MORTON, C.byref(dst), C.byref(r)) == _lib.GSR_ERR_INVALID
        assert r.value == n and str(n) in _lib.lib().gsr_last_error().decode() and dst.rows == n - 1
        assert all((small[k] == 7).all() for k in small)
        # argument refusals
        r = C.c_uint64(99)
        for scope, degree, order in ((2, -1, MORTON), (KEPT, -2, MORTON), (KEPT, 4, MORTON), (KEPT, -1, 2), (KEPT, -1, -1)):
            assert c.L.gsr_export_compressed_ply(c.h, scope, degree, order, None, C.byref(r)) == _lib.GSR_ERR_INVALID
        assert r.value == 99
        assert c.L.gsr_export_compressed_ply(c.h, KEPT, -1, MORTON, None, None) == _lib.GSR_ERR_INVALID
        nul = descriptor([small["chunks"].ctypes.data, small["packed"].ctypes.data, None], n - 1, 3)
        nul.sh = None
        assert c.L.gsr_export_compressed_ply(c.h, KEPT, -1, MORTON, C.byref(nul), C.byref(r)) == _lib.GSR_ERR_INVALID
        # STORE order: the rows of gsr_export_ply (those with a finite position), unchanged by a delete
        before = export(c, KEPT, -1, STORE, 3)
        ply = np.full((N, 62), np.nan, dtype=np.float32)
        _lib.check(c.L.gsr_export_ply(c.h, KEPT, -1, C.c_void_p(ply.ctypes.data), N, C.byref(r)), "gsr_export_ply")
        rows = ply[:r.value]
        rows = rows[np.isfinite(rows[:, :3]).all(axis=1)]
        assert rows.shape[0] == before["count"]
        tab, _ = cref.decode(before["chunks"], before["packed"], before["sh"], before["count"], 18, 3)
        ch = before["chunks"][np.arange(before["count"]) // 256]
        assert (np.abs(tab[:, :3] - rows[:, :3]) <= (ch[:, 3:6] - ch[:, 0:3]) / 2046 + 1e-6).all()
        k = C.c_uint64(0)
        _lib.check(c.L.gsr_delete_hidden(c.h, C.byref(k)), "delete")
        after = export(c, KEPT, -1, STORE, 3)
        for key in ("chunks", "packed", "sh"):
            np.testing.assert_array_equal(bits(after[key]) if key == "chunks" else after[key], bits(before[key]) if key == "chunks" else before[key])


@pytest.mark.parametrize("bands", [1, 2, 3, 4])
@pytest.mark.parametrize("half", [False, True])
def test_upload_rule(bands, half):
    """Reference-encoded files of every degree, 18- and 12-float chunks, uploaded at first = 300 (whole, and as two chunk-aligned pieces
    from device memory) into a store already holding a cloud: the store rule bit for bit, the rest of the store unchanged."""
    rng = np.random.default_rng(40 + bands * 2 + half)
    n = 2000
    src = cref.random_store(rng, n, 4, False)
    sr = cref.scale_rot(src, 4, False, n)
    m = 3000
    with ShCtx(m, 64, 64, bands, _lib.GSR_FLAG_SH_HALF if half else 0) as c:
        base = cloud(rng, bands, half, m, m, specials=False)
        for degree in range(4):
            f = cref.encode(src, n, 4, False, None, None, False, degree, True, sr)
            for cf in (18, 12):
                load(c, base, m)
                table, alpha = cref.decode(np.ascontiguousarray(f["chunks"][:, :cf]), f["packed"], f["sh"], n, cf, degree)
                want = cref.store_rule(table, alpha, degree, bands, half, stride_of(m), first=300, creation_time=1.25, base=base)
                _lib.check(upload(c, f, n, degree, 300, 1.25, cf), "upload")
                np.testing.assert_array_equal(bits(store_of(c)), bits(want))
                # the same file as two chunk-aligned pieces from device memory
                load(c, base, m)
                for lo, hi in ((0, 1024), (1024, n)):
                    ch = torch.from_numpy(np.ascontiguousarray(f["chunks"][lo // 256:cref.chunk_count(hi), :cf])).cuda()
                    pk = torch.from_numpy(f["packed"][lo:hi].view(np.int32).copy()).cuda()
                    sh = torch.from_numpy(f["sh"][lo:hi].copy()).cuda() if degree else None
                    d = descriptor([ch.data_ptr(), pk.data_ptr(), sh.data_ptr() if degree else None], hi - lo, degree, cf)
                    _lib.check(c.L.gsr_upload_compressed_ply(c.h, C.byref(d), 300 + lo, 1.25), "piece")
                np.testing.assert_array_equal(bits(store_of(c)), bits(want))
        # refusals write nothing
        load(c, base, m)
        before = store_of(c)
        f = cref.encode(src, n, 4, False, None, None, False, 2, True, sr)
        ptrs = [f["chunks"].ctypes.data, f["packed"].ctypes.data, f["sh"].ctypes.data]
        bad = [descriptor(ptrs, n, 2, 16), descriptor(ptrs, n, 4), descriptor(ptrs, n, 2, chunk_count=cref.chunk_count(n) + 1),
               descriptor([None, ptrs[1], ptrs[2]], n, 2), descriptor([ptrs[0], None, ptrs[2]], n, 2)]
        nosh = descriptor(ptrs, n, 2)
        nosh.sh = None
        bad.append(nosh)
        for d in bad:
            assert c.L.gsr_upload_compressed_ply(c.h, C.byref(d), 0, 0.0) == _lib.GSR_ERR_INVALID
        assert c.L.gsr_upload_compressed_ply(c.h, C.byref(descriptor(ptrs, n, 2)), m - n + 1, 0.0) == _lib.GSR_ERR_INVALID
        assert c.L.gsr_upload_compressed_ply(c.h, None, 0, 0.0) == _lib.GSR_ERR_INVALID
        np.testing.assert_array_equal(bits(store_of(c)), bits(before))


def test_export_sees_asynchronous_edits():
    """An export enqueued right behind gsr_transform_selection and gsr_recolor_selection (no host sync between) sees both edits."""
    rng = np.random.default_rng(7)
    store = cloud(rng, 4, False, M, N, specials=False)
    with ShCtx(M, 64, 64, 4) as c:
        load(c, store, N)
        sel = rng.random(M) < 0.5
        _lib.check(set_masks(c, np.zeros(M, dtype=bool), sel), "masks")
        before = export(c, KEPT, -1, STORE, 3)
        L = (C.c_float * 12)(*[0.0, 0.0, 1.0, 1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.5, -2.0, 3.0])
        _lib.check(c.L.gsr_transform_selection(c.h, L, None), "transform")
        e = _lib.GsrColorEdit()
        e.matrix[:] = [0.5, 0, 0, 0, 0.5, 0, 0, 0, 0.5, 0.1, 0.1, 0.1]
        e.band_scale[:] = [0.0, 0.0, 0.0]
        e.opacity_scale, e.opacity_offset = 0.5, 0.0
        _lib.check(c.L.gsr_recolor_selection(c.h, C.byref(e), None), "recolor")
        got = export(c, KEPT, -1, STORE, 3)
        c.sync()
        edited = store_of(c)
        check(got, cref.encode(edited, N, 4, False, None, None, False, 3, False))
        assert not np.array_equal(got["packed"], before["packed"])


def test_python_round_trip(tmp_path):
    """export_compressed_ply().save(), CompressedPlyFile parse, the constructor with the parsed file: the new context's store is the
    store rule of the exported file."""
    from godotgaussiansplatting_b200 import camera as cam
    from godotgaussiansplatting_b200.rasterizer import GaussianSplattingRasterizer
    from godotgaussiansplatting_b200.synthetic import synthetic_ply
    n = 20_001
    for half, degree in ((False, -1), (True, 1)):
        r = GaussianSplattingRasterizer(synthetic_ply(n, 4), (160, 96), None, cam.orbit_camera(25, aspect=160 / 96), sh_half=half)
        r.init_gpu(device_ingest=True)
        r2 = None
        try:
            hid = np.zeros(n, dtype=bool)
            hid[::7] = True
            r.set_splat_masks(hid, np.zeros(n, dtype=bool))
            cp = r.export_compressed_ply(sh_degree=degree)
            d = 3 if degree < 0 else degree
            assert cp.size == n - int(hid.sum()) and cp.sh_degree == d
            path = os.path.join(tmp_path, f"c{int(half)}.ply")
            cp.save(path)
            back = CompressedPlyFile(path)
            np.testing.assert_array_equal(back.packed, cp.packed)
            r2 = GaussianSplattingRasterizer(back, (160, 96), None, cam.orbit_camera(25, aspect=160 / 96), sh_half=half)
            r2.init_gpu()
            assert r2._sh_bands == d + 1 and r2.num_splats_loaded[0] == back.size
            got = store_of_r(r2)
            table, alpha = cref.decode(back.chunks, back.packed, back.sh, back.size, 18, d)
            want = cref.store_rule(table, alpha, d, d + 1, half, got.shape[1], creation_time=float(got[0, 0, 3]))
            np.testing.assert_array_equal(bits(got[:, :back.size]), bits(want[:, :back.size]))
        finally:
            r.cleanup_gpu()
            if r2 is not None:
                r2.cleanup_gpu()


def test_c3_size_round_trip():
    """6 M splats of a degree-3 store: a Morton export into device memory and its upload into a second context.  Every position comes
    back within its chunk's half step, every alpha within 1 / 510, and the count is the host's."""
    n = 6_000_000
    rng = np.random.default_rng(9)
    store = cloud(rng, 4, False, n, n, specials=False)
    with ShCtx(n, 64, 64, 4) as c, ShCtx(n, 64, 64, 4) as c2:
        load(c, store, n)
        rows = n
        t = dict(chunks=torch.empty((cref.chunk_count(rows), 18), device="cuda"), packed=torch.empty((rows, 4), dtype=torch.int32, device="cuda"),
                 sh=torch.empty((rows, 45), dtype=torch.uint8, device="cuda"))
        dst = descriptor([t[k].data_ptr() for k in ("chunks", "packed", "sh")], rows, 3)
        r = C.c_uint64(0)
        _lib.check(c.L.gsr_export_compressed_ply(c.h, KEPT, -1, MORTON, C.byref(dst), C.byref(r)), "export")
        assert r.value == cref.exported(store, n, None, None, False).size == dst.rows
        _lib.check(c2.L.gsr_upload_compressed_ply(c2.h, C.byref(dst), 0, 0.0), "upload")
        back = store_of(c2)[:, :dst.rows]
        # the file's row order: sort the original rows the same way (the stable Morton order over the exported bounds)
        idx = cref.exported(store, n, None, None, False)
        keys = cref.morton_keys(store[0, idx, :3])
        idx = idx[np.argsort(keys, kind="stable")]
        ch = t["chunks"].cpu().numpy()[np.arange(idx.size) // 256].astype(np.float64)
        bound = (ch[:, 3:6] - ch[:, 0:3]) / np.array([2 * 2047, 2 * 1023, 2 * 2047]) * (1 + 1e-5) + 1e-6
        assert (np.abs(back[0, :, :3] - store[0, idx, :3].astype(np.float64)) <= bound).all()
        assert (np.abs(back[2, :, 2].astype(np.float64) - store[2, idx, 2]) <= 1 / 510 + 1e-7).all()
