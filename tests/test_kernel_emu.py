"""Every kernel of libgsr (ingest, projection, Onesweep sort, tile ranges, compositor), compiled for the CPU (tests/kernel_emu),
against the oracle -- bit for bit.

This is NOT a CPU path of the product (libgsr has none; see tests/test_abi.py): it is a pre-flight check of kernel LOGIC.
the five kernel files of csrc/ are compiled by g++ under a thin shim of the CUDA execution model (threads = fibers,
__syncthreads / warp collectives real, __shared__ = block-shared, __f*_rn intrinsics = one IEEE binary32 operation each), and one
persistent block works through every tile: staging, blend, tile-stop vote, quantum, spill, re-queue, resume.
It lets a kernel that has not seen a GPU yet prove its indexing and buffering before GPU minutes are spent.
What it cannot show: memory-model behaviour (fences, races between blocks) and timing.
"""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from oracle import oracle as orc
from tests.scenes import make_scene

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "kernel_emu"))
try:
    import build as _emu_build
finally:
    sys.path.pop(0)

SPEC, UNCONTRACTED = 0, 1   # composite_kernel<true> (the gsr spec) / <false> (GSR_FLAG_UNCONTRACTED_BLEND)
_L = None


def lib():
    global _L
    if _L is None:
        L = C.CDLL(_emu_build.build())
        L.emu_composite.restype = C.c_int
        L.emu_composite.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                    C.c_float, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        L.emu_tile_ranges.restype = C.c_int
        L.emu_tile_ranges.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_int, C.c_int, C.c_int32, C.c_void_p, C.c_int]
        L.emu_sort_pairs.restype = C.c_int
        L.emu_sort_pairs.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_int]
        L.emu_projection.restype = C.c_longlong
        L.emu_projection.argtypes = [C.c_void_p, C.c_ulonglong, C.c_uint, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint, C.POINTER(C.c_uint), C.POINTER(C.c_int), C.POINTER(C.c_uint),
                                     C.c_void_p, C.c_void_p, C.c_uint, C.c_uint]
        L.emu_aos_to_soa.argtypes = [C.c_void_p, C.c_ulonglong, C.c_void_p, C.c_ulonglong, C.c_ulonglong]
        L.emu_ply_to_soa.argtypes = [C.c_void_p, C.c_uint, C.c_ulonglong, C.c_float, C.c_void_p, C.c_ulonglong, C.c_ulonglong]
        L.emu_pack_rgb.argtypes = [C.c_void_p, C.c_void_p, C.c_ulonglong]
        L.emu_band_fixup.restype = C.c_int
        L.emu_band_fixup.argtypes = [C.c_int32, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
        _L = L
    return _L


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def emu_ranges(keys, T, quirks=1, sharded=0, global_last=-1, grid=7):
    keys = np.ascontiguousarray(keys, dtype=np.uint32)
    bounds = np.full((T, 2), 0xDEADBEEF, dtype=np.uint32)
    sync = np.zeros(1, dtype=np.int32)
    assert lib().emu_tile_ranges(keys.ctypes.data, keys.size, bounds.ctypes.data, T, quirks, sharded, global_last,
                                 sync.ctypes.data if sharded == 2 else None, grid) == 0
    return bounds, int(sync[0])


def emu_composite(variant, records, values, bounds, w, h, heat=0.0, target=0xFFFFFFFF, tile_begin=0, row_step=1, num_tiles=None, out=None,
                  hint=None, longest_first=False):
    """One emulated persistent CTA renders the launch.  hint: uint32[num_tiles] consumed-chunk hints (in/out, bit 31 = valid)."""
    gx, gy = (w + 15) // 16, (h + 15) // 16
    out = np.zeros((h, w, 4), dtype=np.float32) if out is None else out
    pick = np.zeros(4, dtype=np.float32)
    staged = C.c_ulonglong(0)
    vals = np.concatenate([np.asarray(values, dtype=np.uint32), np.zeros(512, dtype=np.uint32)])   # the kernels never read past a range
    recs, bnds = np.ascontiguousarray(records), np.ascontiguousarray(bounds, dtype=np.uint32)
    nt = gx * gy if num_tiles is None else num_tiles
    rc = lib().emu_composite(variant, recs.ctypes.data, vals.ctypes.data, bnds.ctypes.data, out.ctypes.data, w, h, tile_begin, row_step,
                             nt, heat, target, pick.ctypes.data, C.byref(staged), None if hint is None else hint.ctypes.data, int(longest_first))
    assert rc == 0, {1: "not every tile was rendered", 2: "tile_order_kernel did not produce a permutation"}.get(rc, rc)
    return out, int(staged.value), pick


def oracle_frame(n, seed, w, h, heat=0.0, **kw):
    splat60, vp, ub = make_scene(n, seed, w, h, **kw)
    return orc.frame(splat60, vp, orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8)), heatmap=heat, cap=40 * n)


#                n      seed w    h    heat kwargs
CASES = {
    "long_lists": (60000, 3, 320, 208, 0.0, dict(scale_boost=1.5)),     # 14 000-instance lists: many chunks, quantum, re-queues
    "ragged_heatmap": (9000, 5, 250, 130, 1.0, dict(frame=37, scale_boost=0.5)),
    "load_in": (6000, 7, 192, 160, 0.0, dict(time=0.6, scale_boost=1.0)),
    "tiny": (40, 9, 33, 17, 0.0, dict(scale_boost=-1.0)),
}


@pytest.mark.parametrize("variant", [SPEC, UNCONTRACTED], ids=["spec", "uncontracted"])
@pytest.mark.parametrize("case", list(CASES))
def test_compositor_kernels_reproduce_the_oracle(case, variant):
    """composite_kernel<true> == the oracle's gsr spec, composite_kernel<false> (GSR_FLAG_UNCONTRACTED_BLEND) == the oracle's
    uncontracted evaluation -- which tests/test_refshaders.py pins bit for bit to the reference's own shader text."""
    n, seed, w, h, heat, kw = CASES[case]
    orc.set_blend_contraction(variant == SPEC)
    try:
        fr = oracle_frame(n, seed, w, h, heat, **kw)
    finally:
        orc.set_blend_contraction(True)
    out, staged, _ = emu_composite(variant, fr.records, fr.values, fr.bounds, w, h, heat)
    np.testing.assert_array_equal(bits(out), bits(fr.rgba))
    assert staged == fr.staged


@pytest.mark.parametrize("variant", [SPEC], ids=["spec"])
def test_pick_and_row_interleave(variant):
    n, seed, w, h = 20000, 15, 320, 240
    fr = oracle_frame(n, seed, w, h, scale_boost=1.0)
    counts = fr.bounds[:, 1].astype(np.int64) - fr.bounds[:, 0]
    busy = int(np.argmax(counts))
    _, _, pick = emu_composite(variant, fr.records, fr.values, fr.bounds, w, h, target=busy)
    _, _, want = orc.render(fr.records, fr.values, fr.bounds, w, h, target_tile=busy, pick=np.zeros(4, np.float32))
    np.testing.assert_array_equal(bits(pick), bits(want))
    # cyclic tile rows (gsr_set_row_interleave): three "ranks" fill one frame
    gx, gy = (w + 15) // 16, (h + 15) // 16
    out = np.zeros((h, w, 4), dtype=np.float32)
    for rem in range(3):
        rows = len(range(rem, gy, 3))
        emu_composite(variant, fr.records, fr.values, fr.bounds, w, h, tile_begin=rem * gx, row_step=3, num_tiles=rows * gx, out=out)
    np.testing.assert_array_equal(bits(out), bits(fr.rgba))


@pytest.mark.parametrize("grid", [1, 7, 64])
def test_tile_ranges_kernel(grid):
    fr = oracle_frame(20000, 3, 320, 208, scale_boost=1.0)
    T = fr.bounds.shape[0]
    got, _ = emu_ranges(fr.keys, T, quirks=1, grid=grid)
    np.testing.assert_array_equal(got, fr.bounds)
    fixed, _ = emu_ranges(fr.keys, T, quirks=0, grid=grid)
    np.testing.assert_array_equal(fixed, orc.boundaries(fr.keys, T, quirks=False))
    # last grid tile occupied: the M-1 rule (gsplat_boundaries.glsl:47-49)
    keys = np.sort(np.concatenate([fr.keys, np.full(5, ((T - 1) << 16) | 7, dtype=np.uint32)]))
    got, _ = emu_ranges(keys, T, quirks=1, grid=grid)
    np.testing.assert_array_equal(got, orc.boundaries(keys, T, quirks=True))
    # empty list
    got, _ = emu_ranges(np.zeros(0, np.uint32), T, grid=grid)
    assert not got.any()
    # fast sharded mode: local last tile -> sync word, range end written
    got, sync = emu_ranges(fr.keys, T, quirks=1, sharded=2, grid=grid)
    last = int(fr.keys[-1] >> 16)
    assert sync == last + 1 and got[last, 1] == fr.keys.size


def test_band_fixup_kernel_blanks_only_the_owned_last_tile():
    w, h = 100, 70
    gx = (w + 15) // 16
    img = np.ones((h, w, 4), dtype=np.float32)
    L = 2 * gx + 3                                     # tile row 2, column 3
    lib().emu_band_fixup(L + 1, img.ctypes.data, w, h, 0, 5, 3, 1)     # row 2 % 3 != 1: another rank owns it
    assert (img == 1).all()
    lib().emu_band_fixup(L + 1, img.ctypes.data, w, h, 0, 5, 3, 2)
    blank = np.zeros_like(img, dtype=bool)
    blank[32:48, 48:64] = True
    assert (img[blank[..., 0]] == [0, 0, 0, 1]).all() and (img[~blank[..., 0]] == 1).all()
    T = gx * ((h + 15) // 16)
    img[:] = 1
    lib().emu_band_fixup(T, img.ctypes.data, w, h, 0, 5, 1, 0)         # last occupied tile == T-1: the other rule applies, nothing blanked
    assert (img == 1).all()


@pytest.mark.parametrize("n", [1, 31, 100, 5119, 5120, 5121, 6143, 6144, 6145, 20000, 100000])
@pytest.mark.parametrize("pairs", [True, False], ids=["pairs", "keys"])
def test_onesweep_kernels_are_a_stable_sort(n, pairs):
    """sort_hist_kernel + 4 x onesweep_kernel<512, 10>: tile = 5120 keys, ragged last tile, padding keys, look-back chain."""
    rng = np.random.default_rng(n)
    keys = rng.integers(0, 2**32, n, dtype=np.uint64).astype(np.uint32)
    if n > 1000:
        keys[: n // 2] &= np.uint32(0x00FF00FF)                      # heavy ties and two constant digits
        keys[n // 2: n // 2 + 50] = 0xFFFFFFFF                        # real keys equal to the padding key
    n_max = n + 777
    k = np.zeros(n_max, dtype=np.uint32)
    k[:n] = keys
    k[n:] = 0x12345678                                               # beyond n: must not be touched or read as data
    v = np.arange(n_max, dtype=np.uint32) if pairs else None
    assert lib().emu_sort_pairs(k.ctypes.data, v.ctypes.data if pairs else None, n, n_max, 5) == 0
    order = np.argsort(keys, kind="stable")
    np.testing.assert_array_equal(k[:n], keys[order])
    assert (k[n:] == 0x12345678).all()
    if pairs:
        np.testing.assert_array_equal(v[:n], order.astype(np.uint32))


def test_sorted_frame_through_the_emulated_kernels():
    """oracle projection -> emulated sort -> emulated ranges -> emulated compositor == the oracle frame."""
    n, w, h = 15000, 256, 144
    splat60, vp, ub = make_scene(n, 21, w, h, scale_boost=1.0)
    u = orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8))
    fr = orc.frame(splat60, vp, u)
    pr = orc.project(splat60, vp, u)
    cap = 10 * n
    k = np.zeros(cap, dtype=np.uint32)
    v = np.zeros(cap, dtype=np.uint32)
    k[: pr.duplicates], v[: pr.duplicates] = pr.keys, pr.values
    assert lib().emu_sort_pairs(k.ctypes.data, v.ctypes.data, pr.duplicates, cap, 3) == 0
    np.testing.assert_array_equal(k[: pr.duplicates], fr.keys)
    np.testing.assert_array_equal(v[: pr.duplicates], fr.values)
    bounds, _ = emu_ranges(k[: pr.duplicates], fr.bounds.shape[0])
    np.testing.assert_array_equal(bounds, fr.bounds)
    out, staged, _ = emu_composite(SPEC, pr.records, v[: pr.duplicates], bounds, w, h)
    np.testing.assert_array_equal(bits(out), bits(fr.rgba))
    assert staged == fr.staged


# ---------------------------------------------------------------------------------------------------------------- ingest + projection
def emu_upload(splat60, chunk=None):
    """gsr_upload_splats_aos: AoS -> 15 SoA planes (stride = n rounded up to 256), optionally in chunks like ply_file.gd:36-71."""
    splat60 = np.ascontiguousarray(splat60, dtype=np.float32)
    n = splat60.shape[0]
    stride = (n + 255) // 256 * 256
    soa = np.zeros((15, stride, 4), dtype=np.float32)
    step = chunk or n
    for first in range(0, n, step):
        part = np.ascontiguousarray(splat60[first:first + step])
        lib().emu_aos_to_soa(part.ctypes.data, part.shape[0], soa.ctypes.data, stride, first)
    return soa, stride


def emu_scatter(soa, stride, n, vp, ub, G, rank, first, count, seg_cap):
    """projection_scatter_kernel (group mode) of rank `rank`: its slice's pairs and records into G destination buffers."""
    vp = np.ascontiguousarray(vp, dtype=np.float32)
    recs = [np.zeros(n, dtype=orc.RECORD_DTYPE) for _ in range(G)]
    keys = [np.full(seg_cap, 0xDEADBEEF, dtype=np.uint32) for _ in range(G)]
    vals = [np.full(seg_cap, 0xDEADBEEF, dtype=np.uint32) for _ in range(G)]
    PP = C.c_void_p * G
    counts = (C.c_ulonglong * G)()
    last = C.c_uint(0)
    L = lib()
    L.emu_projection_scatter.restype = C.c_int
    L.emu_projection_scatter.argtypes = [C.c_void_p, C.c_ulonglong, C.c_uint, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_uint, C.c_uint, C.c_uint,
                                         C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    rc = L.emu_projection_scatter(soa.ctypes.data, stride, n, vp.ctypes.data, ub, G, rank, first, count, seg_cap,
                                  PP(*[r.ctypes.data for r in recs]), PP(*[k.ctypes.data for k in keys]), PP(*[v.ctypes.data for v in vals]),
                                  counts, C.byref(last))
    assert rc == 0, {1: "flag words not published", 2: "protocol words not reset"}.get(rc, rc)
    return recs, keys, vals, [int(c) for c in counts], int(last.value)


def emu_project(soa, stride, n, vp, ub, w, h, band=None, row_mod=1, row_rem=0, fast_reject=0, sh_bulk_min=0, cap=None):
    gy = (h + 15) // 16
    y0, y1 = (0, gy) if band is None else band
    cap = cap or 10 * n
    rec = np.zeros(n, dtype=orc.RECORD_DTYPE)
    keys = np.zeros(cap, dtype=np.uint32)
    vals = np.zeros(cap, dtype=np.uint32)
    vis, last, ovf = C.c_uint(0), C.c_int(0), C.c_uint(0)
    vp = np.ascontiguousarray(vp, dtype=np.float32)
    m = lib().emu_projection(soa.ctypes.data, stride, n, vp.ctypes.data, ub, y0, y1, row_mod, row_rem, fast_reject, sh_bulk_min, rec.ctypes.data,
                             keys.ctypes.data, vals.ctypes.data, cap, C.byref(vis), C.byref(last), C.byref(ovf),
                             None, None, 0, 0)
    return dict(m=int(m), keys=keys[:min(m, cap)], values=vals[:min(m, cap)], records=rec, visible=int(vis.value), last_tile=int(last.value),
                overflow=bool(ovf.value))


def assert_projection_equal(got, pr):
    assert got["m"] == pr.duplicates and got["visible"] == pr.visible and not got["overflow"]
    np.testing.assert_array_equal(got["keys"], pr.keys)
    np.testing.assert_array_equal(got["values"], pr.values)
    vis = np.unique(pr.values)
    for f in orc.RECORD_DTYPE.names:
        np.testing.assert_array_equal(bits(got["records"][f][vis]), bits(pr.records[f][vis]), err_msg=f"record field {f}")


@pytest.mark.parametrize("sh_bulk_min", [1, 12, 33], ids=["always_bulk", "default", "never_bulk"])
def test_projection_kernel(sh_bulk_min):
    """projection_kernel: TMA-staged planes, chained scan over the CTA links (closer warp + look-back), both SH paths, hybrid emit."""
    n, w, h = 20000, 320, 208
    splat60, vp, ub = make_scene(n, 3, w, h, scale_boost=1.0)
    pr = orc.project(splat60, vp, orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8)))
    soa, stride = emu_upload(splat60, chunk=777)
    got = emu_project(soa, stride, n, vp, ub, w, h, sh_bulk_min=sh_bulk_min)
    assert_projection_equal(got, pr)
    assert got["last_tile"] == pr.last_tile


def test_projection_kernel_edge_sizes_and_overflow():
    for n in (1, 31, 257, 1000):
        splat60, vp, ub = make_scene(n, 60 + n, 320, 240, scale_boost=-1.5)
        pr = orc.project(splat60, vp, orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8)))
        soa, stride = emu_upload(splat60)
        assert_projection_equal(emu_project(soa, stride, n, vp, ub, 320, 240), pr)
    # huge splats: M exceeds the capacity -> overflow flagged, the true M still counted, nothing written past the capacity
    n = 300
    splat60, vp, ub = make_scene(n, 5, 640, 480, scale_boost=3.0)
    pr = orc.project(splat60, vp, orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8)), cap=10 * n)
    assert pr.duplicates > 10 * n
    soa, stride = emu_upload(splat60)
    got = emu_project(soa, stride, n, vp, ub, 640, 480, cap=10 * n)
    assert got["overflow"] and got["m"] == pr.duplicates
    np.testing.assert_array_equal(got["keys"], pr.keys[: 10 * n])


def test_projection_kernel_band_and_cyclic_rows():
    n, w, h = 12000, 320, 240
    gx, gy = (w + 15) // 16, (h + 15) // 16
    splat60, vp, ub = make_scene(n, 8, w, h, scale_boost=1.0)
    u = orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8))
    soa, stride = emu_upload(splat60)
    # contiguous band (gsr_set_band): the oracle's band mode
    pr = orc.project(splat60, vp, u, band=(4, 9))
    got = emu_project(soa, stride, n, vp, ub, w, h, band=(4, 9))
    assert_projection_equal(got, pr)
    assert got["last_tile"] == pr.last_tile                      # exact sharded mode: the frame-global last tile
    # cyclic rows (gsr_set_row_interleave), plain and with the conservative reject + 1024-splat compaction kernel:
    # every rank emits exactly the full frame's pairs of its own rows, in the same (splat-id, row-major) order
    full = orc.project(splat60, vp, u)
    rows = (full.keys >> 16) // gx
    for fast_reject in (0, 1):
        seen = 0
        for rem in range(3):
            got = emu_project(soa, stride, n, vp, ub, w, h, row_mod=3, row_rem=rem, fast_reject=fast_reject)
            own = rows % 3 == rem
            np.testing.assert_array_equal(got["keys"], full.keys[own])
            np.testing.assert_array_equal(got["values"], full.values[own])
            assert got["last_tile"] == (int((full.keys[own] >> 16).max()) if own.any() else -1)   # LOCAL last tile
            seen += got["m"]
        assert seen == full.duplicates


def test_ingest_kernels():
    from godotgaussiansplatting_b200.synthetic import synthetic_ply_table
    n = 1000
    table = np.ascontiguousarray(synthetic_ply_table(n, 4), dtype=np.float32)
    want = orc.preprocess_ply(table, 2.5)                                            # (n, 60): util/ply_file.gd:44-69
    stride = (n + 255) // 256 * 256
    soa = np.zeros((15, stride, 4), dtype=np.float32)
    assert lib().emu_ply_to_soa(table.ctypes.data, table.shape[1], n, 2.5, soa.ctypes.data, stride, 0) == 0
    got = soa[:, :n, :].transpose(1, 0, 2).reshape(n, 60)
    np.testing.assert_array_equal(bits(got), bits(want))
    soa2, _ = emu_upload(want, chunk=130)
    np.testing.assert_array_equal(bits(soa2), bits(soa))
    for pixels in (1, 4, 1023, 4096):                                                # RGB32F packing incl. the ragged tail
        rgba = np.random.default_rng(pixels).random((pixels, 4), dtype=np.float32)
        rgb = np.zeros(3 * ((pixels + 3) // 4 * 4) + 4, dtype=np.float32)
        lib().emu_pack_rgb(rgba.ctypes.data, rgb.ctypes.data, pixels)
        np.testing.assert_array_equal(rgb[: 3 * pixels].reshape(pixels, 3), rgba[:, :3])


def test_whole_pipeline_through_the_emulated_kernels():
    """PLY vertices -> ingest -> projection -> sort -> ranges -> compositor -> RGB packing, every stage the product's kernel code."""
    from godotgaussiansplatting_b200.synthetic import synthetic_ply_table
    from godotgaussiansplatting_b200 import camera as cam
    from tests.scenes import uniforms_bytes
    n, w, h = 9000, 256, 144
    table = np.ascontiguousarray(synthetic_ply_table(n, 12), dtype=np.float32)
    table[:, 55:58] += 1.0
    c = cam.orbit_camera(40, aspect=w / h)
    vp = cam.pack_camera_push_constants(c.get_camera_transform(), c.get_camera_projection())
    ub = uniforms_bytes(c.global_position, 1.0, w, h, 10.0)
    fr = orc.frame(orc.preprocess_ply(table, 0.0), vp, orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8)))
    stride = (n + 255) // 256 * 256
    soa = np.zeros((15, stride, 4), dtype=np.float32)
    lib().emu_ply_to_soa(table.ctypes.data, table.shape[1], n, 0.0, soa.ctypes.data, stride, 0)
    pj = emu_project(soa, stride, n, vp, ub, w, h)
    cap = 10 * n
    k = np.zeros(cap, dtype=np.uint32)
    v = np.zeros(cap, dtype=np.uint32)
    k[: pj["m"]], v[: pj["m"]] = pj["keys"], pj["values"]
    lib().emu_sort_pairs(k.ctypes.data, v.ctypes.data, pj["m"], cap, 4)
    bounds, _ = emu_ranges(k[: pj["m"]], fr.bounds.shape[0])
    out, staged, _ = emu_composite(SPEC, pj["records"], v[: pj["m"]], bounds, w, h)
    assert pj["m"] == fr.duplicates and staged == fr.staged
    np.testing.assert_array_equal(k[: pj["m"]], fr.keys)
    np.testing.assert_array_equal(bounds, fr.bounds)
    np.testing.assert_array_equal(bits(out), bits(fr.rgba))
    rgb = np.zeros((h * w * 3 + 4,), dtype=np.float32)
    lib().emu_pack_rgb(out.ctypes.data, rgb.ctypes.data, w * h)
    np.testing.assert_array_equal(bits(rgb[: 3 * w * h].reshape(h, w, 3)), bits(fr.rgba[..., :3]))


@pytest.mark.parametrize("G", [2, 3, 8])
def test_scatter_projection_shards_the_splats_and_routes_pairs_to_row_owners(G):
    """Group mode (gsr_group_*, projection_scatter_kernel): every rank projects ITS slice of the splats and stores each pair / record
    into the buffers of the rank that owns the tile row (row % G).  Concatenating, per destination, the segments of the sources in
    rank order must give exactly the single-GPU emission restricted to the destination's rows -- same keys, same splat-id order --
    and the destination's record table must hold the oracle's records of every splat that touches its rows."""
    n, w, h = 12000, 320, 240
    gx, gy = (w + 15) // 16, (h + 15) // 16
    splat60, vp, ub = make_scene(n, 8, w, h, scale_boost=1.0)
    u = orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8))
    soa, stride = emu_upload(splat60)
    full = orc.project(splat60, vp, u)
    rows = (full.keys >> 16).astype(np.int64) // gx
    slice_len = ((n + G - 1) // G + 255) // 256 * 256
    seg_cap = 10 * n // G
    got_keys = [[] for _ in range(G)]
    got_vals = [[] for _ in range(G)]
    got_recs = [np.zeros(n, dtype=orc.RECORD_DTYPE) for _ in range(G)]
    lasts = []
    for r in range(G):
        first = min(r * slice_len, n)
        count = max(0, min(slice_len, n - first))
        recs, keys, vals, counts, last = emu_scatter(soa, stride, n, vp, ub, G, r, first, count, seg_cap)
        lasts.append(last)
        in_slice = (full.values >= first) & (full.values < first + count)
        for d in range(G):
            assert counts[d] == int((in_slice & (rows % G == d)).sum())           # the count published to destination d
            assert counts[d] <= seg_cap and np.all(keys[d][counts[d]:] == 0xDEADBEEF)  # nothing beyond the segment's fill
            got_keys[d].append(keys[d][:counts[d]]); got_vals[d].append(vals[d][:counts[d]])
            ids = np.unique(vals[d][:counts[d]])
            got_recs[d][ids] = recs[d][ids]
    assert max(lasts) == full.last_tile + 1   # the frame-global last occupied tile travels with the segments (exact Q10 bookkeeping)
    for d in range(G):
        own = rows % G == d
        np.testing.assert_array_equal(np.concatenate(got_keys[d]), full.keys[own])
        np.testing.assert_array_equal(np.concatenate(got_vals[d]), full.values[own])
        ids = np.unique(full.values[own])
        for f in orc.RECORD_DTYPE.names:
            np.testing.assert_array_equal(bits(got_recs[d][f][ids]), bits(full.records[f][ids]), err_msg=f"record field {f}")


@pytest.mark.parametrize("fmt", [0, 1, 2, 3, 0x100, 0x101, 0x102, 0x103])
def test_present_kernel_matches_the_oracle_conversion(fmt):
    """Scope row f3 (csrc/present.cu): RGBA32F -> GSR_OUT_* with the optional sRGB -> linear of main.gdshader:7-11, bit for bit
    against oracle.present -- incl. values above 1, exact 0 / 1 / 0.04045, a ragged pixel count, inf and negative inputs."""
    L = lib()
    L.emu_present.argtypes = [C.c_void_p, C.c_void_p, C.c_ulonglong, C.c_int]
    rng = np.random.default_rng(fmt)
    px = 1003
    rgba = (rng.random((px, 4)).astype(np.float32) ** 3) * 1.7
    rgba[:8, :3] = np.array([[0.0, 1.0, 0.04045], [0.040449999, 0.5, 2.5], [np.inf, -0.25, 1e-30], [65519.0, 65520.0, 6e-8],
                             [0.9999999, 0.0031308, 1e-5], [3e-5, 0.00196, 0.99803925], [0.5019608, 0.49803922, 0.2], [1e-40, 3.0, 0.7]], dtype=np.float32)
    rgba[:, 3] = 1.0
    want = orc.present(rgba, fmt)
    got = np.zeros_like(want)
    assert L.emu_present(rgba.ctypes.data, got.ctypes.data, px, fmt) == 0
    np.testing.assert_array_equal(got.view(np.uint8), want.view(np.uint8))


def test_compositor_ticket_order_does_not_change_pixels():
    """Longest-chain-first ticket order (tile_order_kernel): by list length on the first frame, by the consumed-chunk hints the
    compositor leaves from then on -- scheduling only: frame and staged-instance count stay bit-identical; also with cyclic rows."""
    n, seed, w, h, heat, kw = CASES["long_lists"]
    fr = oracle_frame(n, seed, w, h, heat, **kw)
    gx, gy = (w + 15) // 16, (h + 15) // 16
    T = gx * gy
    ts = np.zeros(T, dtype=np.uint32)
    orc.render(fr.records, fr.values, fr.bounds, w, h, heatmap=heat, tile_staged=ts)
    hint = np.zeros(T, dtype=np.uint32)
    for frame_no in range(3):     # frame 0: no hints -> list lengths; frames 1, 2: last frame's consumed chunks
        out, staged, _ = emu_composite(SPEC, fr.records, fr.values, fr.bounds, w, h, heat, hint=hint, longest_first=True)
        np.testing.assert_array_equal(bits(out), bits(fr.rgba))
        assert staged == fr.staged
        assert np.all(hint >> 31 == 1)                                             # every tile reported ...
        np.testing.assert_array_equal(hint & 0x7FFFFFFF, (ts.astype(np.int64) + 255) // 256)   # ... the chunks the oracle consumed
    out2 = np.zeros_like(out)
    for rem in range(3):
        rows = len(range(rem, gy, 3))
        h3 = np.zeros(rows * gx, dtype=np.uint32)
        for _ in range(2):
            emu_composite(SPEC, fr.records, fr.values, fr.bounds, w, h, heat, tile_begin=rem * gx, row_step=3, num_tiles=rows * gx, out=out2,
                          hint=h3, longest_first=True)
    np.testing.assert_array_equal(bits(out2), bits(fr.rgba))


@pytest.mark.parametrize("world", [2, 3, 8, 16])
def test_group_receive_kernels_pack_the_segments_in_source_order(world):
    """csrc/group.cu, destination side of the scatter projection: group_wait_segments_kernel (prefix of the clamped segment lengths, M,
    overflow, frame-global last tile) and gather_segments_kernel (segments packed in source order) -- incl. an empty and an
    over-full segment.  Running them here also proves their warp collectives sit outside divergent code (the emulator's collectives
    are real rendezvous: a shuffle that only some lanes reach never returns)."""
    rng = np.random.default_rng(world)
    seg_cap, capacity = 1000, 100000
    counts = rng.integers(0, seg_cap + 1, size=world).astype(np.uint32)
    counts[0] = 0
    if world > 2:
        counts[2] = seg_cap + 57          # the source sent more than its segment holds: kept = seg_cap, overflow flagged
    lasts = rng.integers(0, 500, size=world).astype(np.uint32)
    rx_k = rng.integers(0, 1 << 32, size=world * seg_cap, dtype=np.uint64).astype(np.uint32)
    rx_v = rng.integers(0, 1 << 32, size=world * seg_cap, dtype=np.uint64).astype(np.uint32)
    keys = np.zeros(capacity, dtype=np.uint32); vals = np.zeros(capacity, dtype=np.uint32)
    total, m, ovf, last = C.c_ulonglong(0), C.c_uint(0), C.c_uint(0), C.c_int(0)
    prefix = np.zeros(world + 1, dtype=np.uint32)
    L = lib()
    L.emu_group_receive.restype = C.c_int
    L.emu_group_receive.argtypes = [C.c_int, C.c_uint, C.c_uint] + [C.c_void_p] * 6 + [C.c_void_p] * 5
    rc = L.emu_group_receive(world, seg_cap, capacity, counts.ctypes.data, lasts.ctypes.data, rx_k.ctypes.data, rx_v.ctypes.data, keys.ctypes.data, vals.ctypes.data,
                             C.byref(total), C.byref(m), C.byref(ovf), C.byref(last), prefix.ctypes.data)
    assert rc == 0
    kept = np.minimum(counts, seg_cap)
    np.testing.assert_array_equal(prefix, np.concatenate([[0], np.cumsum(kept)]))
    assert total.value == int(counts.sum()) and m.value == int(kept.sum()) and ovf.value == int((counts > seg_cap).any()) and last.value == int(lasts.max())
    want_k = np.concatenate([rx_k[r * seg_cap: r * seg_cap + kept[r]] for r in range(world)])
    want_v = np.concatenate([rx_v[r * seg_cap: r * seg_cap + kept[r]] for r in range(world)])
    np.testing.assert_array_equal(keys[:m.value], want_k)
    np.testing.assert_array_equal(vals[:m.value], want_v)
