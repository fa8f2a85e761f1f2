"""Splat property selection without a GPU (include/gsr.h "Splat property selection"): the emulated select_where_kernel and
splat_histogram_kernel bit for bit against the numpy rule of tests/property_reference -- every property on float and binary16 stores of
bands 1-4, special stored words, vacant slots, a cloud below max_splats, instance ranges that start and end inside a word, filter
conjunctions, every op with hidden bits, edges of every kind with values on them, several CTAs adding into one histogram -- the
properties against their float64 meaning, the Python helper, and the NULL-context checks."""
import ctypes as C

import numpy as np
import pytest

from godotgaussiansplatting_b200 import _lib
from godotgaussiansplatting_b200.rasterizer import splat_filter
from tests import delete_reference as dref
from tests import property_reference as pref
from tests import selection_reference as sref
from tests.transform_reference import sh_planes

F32, U32 = np.float32, np.uint32
INF = np.inf
SPECIAL = np.array([0x7FC00000, 0xFFC00123, 0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x00000001, 0x807FFFFF, 0x3F800000],
                   dtype=U32)   # NaNs, +-0, +-inf, denormals, 1


def store_of(rng, bands, half, m, special=0.03):
    """A store of m slots (stride rounded up to 256): covariance words of plausible splats with random special words, opacity in
    [0, 1), DC coefficients around 0 (binary16 halves of them for a half store); a few vacant slots."""
    stride = (m + 255) // 256 * 256
    s = rng.normal(size=(3 + sh_planes(bands, half), stride, 4)).astype(F32)
    R = np.linalg.qr(rng.normal(size=(stride, 3, 3)))[0]
    sc = np.exp(rng.uniform(-4, 1, size=(stride, 3)))
    sc[rng.random(stride) < 0.2] *= np.array([30.0, 0.1, 0.1])   # needles
    S = np.einsum("nij,nj,nkj->nik", R, sc ** 2, R).astype(F32)
    s[1, :, 0], s[1, :, 1], s[1, :, 2], s[1, :, 3] = S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1]
    s[2, :, 0], s[2, :, 1] = S[:, 1, 2], S[:, 2, 2]
    s[2, :, 2] = rng.random(stride).astype(F32)
    if half:
        h = (rng.normal(size=(stride, 8)) * 0.8).astype(np.float16)
        s[3] = h.view(U32).reshape(stride, 4).view(F32)
    w = s.view(U32)
    for p in (0, 1, 2, 3):
        pick = rng.random(w[p].shape) < special
        w[p][pick] = SPECIAL[rng.integers(0, SPECIAL.size, int(pick.sum()))]
    dref.vacate_slots(s, rng.random(m) < 0.05)
    return s


def masks_of(rng, m, hidden=0.2, selected=0.3):
    hid = rng.random(m) < hidden
    return hid, (rng.random(m) < selected) & ~hid


def quantile_range(store, half, prop, rgb, rng, n):
    v = pref.values(store, half, prop, rgb)[:n]
    lo, hi = np.quantile(v[np.isfinite(v)], np.sort(rng.uniform(0.1, 0.9, 2)))
    return F32(lo), F32(hi)


# ---- select_where -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bands", [1, 2, 3, 4])
@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("prop", pref.PROPS)
def test_every_property_selects_by_the_rule(bands, half, prop):
    rng = np.random.default_rng(bands * 100 + half * 10 + prop)
    m, n = 3000 + 13, 2900 + 5                      # max_splats and the cloud: neither a multiple of 32
    store = store_of(rng, bands, half, m)
    hid, sel = masks_of(rng, m)
    rgb = (0.2, 0.6, 0.9)
    lo, hi = quantile_range(store, half, prop, rgb, rng, n)
    for op in range(4):
        f = [(prop, lo, hi, rgb)]
        want = pref.where_rule(store, half, hid, sel, 0, n, f, op)
        got = pref.emu_where(store, half, hid, sel, 0, n, f, op)
        np.testing.assert_array_equal(got, want, err_msg=f"op {op}")
        assert not got[n:].any() or op != sref.SET
    inside = pref.where_inside(store, half, 0, n, [(prop, lo, hi, rgb)])
    assert 10 < inside.sum() < n - 10


@pytest.mark.parametrize("half", [False, True])
def test_conjunctions_bounds_and_ranges(half):
    """1 to 8 filters, lo == hi, lo > hi, +-inf bounds; tested ranges that start and end inside a word; every op with hidden bits."""
    rng = np.random.default_rng(40 + half)
    m, n = 4096 + 77, 4000 + 3
    store = store_of(rng, 3, half, m)
    some = pref.values(store, half, pref.OPACITY)
    exact = F32(some[np.flatnonzero(np.isfinite(some))[7]])
    sets = [
        [(pref.OPACITY, 0.0, 0.05, (0, 0, 0))],
        [(pref.OPACITY, -INF, 0.5, (0, 0, 0)), (pref.SIZE, 0.1, INF, (0, 0, 0))],
        [(pref.SIZE, 0.0, 3.0, (0, 0, 0)), (pref.ISOTROPY, -INF, 0.3, (0, 0, 0))],
        [(pref.COLOR, 0.0, 0.2, (0.5, 0.5, 0.5)), (pref.OPACITY, 0.2, 1.0, (0, 0, 0)), (pref.VOLUME, -INF, 1.0, (0, 0, 0))],
        [(pref.OPACITY, exact, exact, (0, 0, 0))],                                             # lo == hi
        [(pref.OPACITY, 0.6, 0.4, (0, 0, 0))],                                                 # lo > hi: empty
        [(pref.OPACITY, -INF, INF, (0, 0, 0))],                                                # every non-NaN value
        [(p, -INF, INF, (0.1 * p, 0.2, 0.3)) for p in pref.PROPS] + [(pref.OPACITY, 0.1, 0.9, (0, 0, 0)),
                                                                     (pref.SIZE, 0.01, 50.0, (0, 0, 0)),
                                                                     (pref.COLOR, 0.0, 2.0, (1.0, 0.0, 0.0))],   # 8 filters
    ]
    ranges = [(0, n), (45, 1000 - 45 + 7), (33, 31), (3999, 4), (n - 5, 5), (n, 0)]
    hid, sel = masks_of(rng, m)
    for i, f in enumerate(sets):
        for j, (first, count) in enumerate(ranges):
            op = (i + j) % 4
            want = pref.where_rule(store, half, hid, sel, first, count, f, op)
            got = pref.emu_where(store, half, hid, sel, first, count, f, op)
            np.testing.assert_array_equal(got, want, err_msg=f"set {i} range {j} op {op}")
            sel = want
    assert pref.where_inside(store, half, 0, n, sets[4]).sum() >= 1
    assert pref.where_inside(store, half, 0, n, sets[5]).sum() == 0
    assert pref.where_inside(store, half, 0, n, sets[7]).sum() > 50


def test_vacant_and_nan_positions_are_never_inside():
    rng = np.random.default_rng(3)
    m = 1000
    store = store_of(rng, 1, False, m, special=0.0)
    dref.vacate_slots(store, np.arange(m) % 7 == 0)
    store[0, 3, 1] = np.nan   # a NaN y
    f = [(pref.OPACITY, -INF, INF, (0, 0, 0))]
    none = np.zeros(m, bool)
    got = pref.emu_where(store, False, none, none, 0, m, f, sref.SET)
    np.testing.assert_array_equal(got, pref.where_rule(store, False, none, none, 0, m, f, sref.SET))
    assert not got[::7].any() and not got[3] and got.sum() > 700


def test_properties_mean_what_they_say():
    """Size is the trace, volume the determinant (float64, to rounding), isotropy 1 for spheres and small for needles, colour
    distance 0 at the splat's own DC colour."""
    rng = np.random.default_rng(8)
    m = 512
    store = store_of(rng, 1, False, m, special=0.0)
    s = store.astype(np.float64)
    S = np.empty((store.shape[1], 3, 3))
    S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1] = s[1, :, 0], s[1, :, 1], s[1, :, 2], s[1, :, 3]
    S[:, 1, 2], S[:, 2, 2] = s[2, :, 0], s[2, :, 1]
    S[:, 1, 0], S[:, 2, 0], S[:, 2, 1] = S[:, 0, 1], S[:, 0, 2], S[:, 1, 2]
    ok = ~np.isnan(s[0, :, 0])
    np.testing.assert_allclose(pref.values(store, False, pref.SIZE)[ok], np.trace(S, axis1=1, axis2=2)[ok], rtol=1e-5)
    det, tr = np.linalg.det(S)[ok], np.trace(S, axis1=1, axis2=2)[ok]
    assert (np.abs(pref.values(store, False, pref.VOLUME)[ok] - det) <= 1e-5 * tr ** 3).all()   # float32 rounding, relative to t^3
    sphere = store.copy()
    sphere[1, :, :] = [2.0, 0.0, 0.0, 2.0]
    sphere[2, :, :2] = [0.0, 2.0]
    assert (pref.values(sphere, False, pref.ISOTROPY)[ok] == 1.0).all()
    needle = sphere.copy()
    needle[1, :, 0] = 1e4
    assert (pref.values(needle, False, pref.ISOTROPY)[ok] < 1e-3).all()
    dc = np.stack(pref.dc_of(store, False), 1)
    own = (F32(0.5) + dc[5] * pref.SH_C0)
    assert pref.values(store, False, pref.COLOR, tuple(float(x) for x in own))[5] == 0.0


# ---- the histogram ------------------------------------------------------------------------------------------------------------
def edges_of(kind, lo, hi, bins, rng):
    if kind == "uniform":
        return np.linspace(lo, hi, bins + 1).astype(F32)
    if kind == "log":
        return np.geomspace(max(lo, 1e-6), hi, bins + 1).astype(F32)
    e = np.unique(rng.uniform(lo, hi, size=bins + 1).astype(F32))   # irregular
    return e


def assert_hist(got, want):
    np.testing.assert_array_equal(got[0], want[0])
    assert np.array(got[1], F32).view(U32).tolist() == np.array(want[1], F32).view(U32).tolist(), (got[1], want[1])


@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("prop", pref.PROPS)
@pytest.mark.parametrize("kind", ["uniform", "log", "irregular"])
def test_histogram_is_the_rule(half, prop, kind):
    rng = np.random.default_rng(300 + half * 50 + prop * 5 + len(kind))
    m, n = 2048 + 45, 2000 + 1
    bands = 2 if half else 4
    store = store_of(rng, bands, half, m)
    hid, sel = masks_of(rng, m)
    rgb = (0.3, 0.3, 0.7)
    v = pref.values(store, half, prop, rgb)[:n]
    fin = v[np.isfinite(v)]
    lo, hi = np.quantile(fin, [0.05, 0.95])
    e = edges_of(kind, lo, hi, 37, rng)
    if prop == pref.OPACITY:   # values exactly on every edge, the last one included
        idx = rng.choice(np.flatnonzero(~np.isnan(store[0, :n, 0])), e.size, replace=False)
        store[2, idx, 2] = e
    for selected_only in (0, 1):
        for first, count in ((0, n), (37, 1500 - 37 + 9)):
            want = pref.histogram_rule(store, half, hid, sel, first, count, prop, rgb, e, selected_only)
            got = pref.emu_histogram(store, half, hid, sel, first, count, prop, rgb, e, selected_only, blocks=3, ctas=3)
            assert_hist(got, want)
    want = pref.histogram_rule(store, half, None, None, 0, n, prop, rgb, e, 0)   # masks not in use
    assert_hist(pref.emu_histogram(store, half, None, None, 0, n, prop, rgb, e, 0), want)
    c = want[0]
    assert c[:-3].sum() > 100 and c[-3] > 0 and c[-2] > 0
    if prop == pref.OPACITY:
        assert (c[:-3] > 0).all()


def test_histogram_specials_and_extremes():
    """Values below, above, NaN, +-0 and +-inf; min / max in ord order (-0 before +0); 1, 256 and 1024 bins; a saturated property."""
    rng = np.random.default_rng(77)
    m = 3000
    store = store_of(rng, 1, False, m, special=0.0)
    none = np.zeros(m, bool)
    store[0, :10, :3] = 0.0   # none of them vacant
    op = store[2, :, 2]
    op[:10] = [np.nan, -0.0, 0.0, np.inf, -np.inf, 1.0, 1e-45, -1e-45, 0.25, 0.5]
    for bins in (1, 256, 1024):
        e = np.linspace(0.0, 1.0, bins + 1).astype(F32)
        want = pref.histogram_rule(store, False, none, none, 0, m, pref.OPACITY, (0, 0, 0), e, 0)
        assert_hist(pref.emu_histogram(store, False, none, none, 0, m, pref.OPACITY, (0, 0, 0), e, 0, blocks=2, ctas=2), want)
        assert want[1] == (-np.inf, np.inf)
        assert want[0][bins + 2] >= 1 and want[0][bins] >= 2 and want[0][bins + 1] >= 1
    sub = pref.emu_histogram(store, False, none, none, 1, 2, pref.OPACITY, (0, 0, 0), np.array([0, 1], F32), 0)   # -0 and +0 only
    assert np.array(sub[1], F32).view(U32).tolist() == [0x80000000, 0]
    assert sub[0].tolist() == [2, 0, 0, 0]
    op[:] = 1.0   # a saturated property: every value in the last bin
    e = np.linspace(0.0, 1.0, 65).astype(F32)
    want = pref.histogram_rule(store, False, none, none, 0, m, pref.OPACITY, (0, 0, 0), e, 0)
    assert_hist(pref.emu_histogram(store, False, none, none, 0, m, pref.OPACITY, (0, 0, 0), e, 0, blocks=4, ctas=4), want)
    assert want[0][63] == int((~np.isnan(store[0, :m, 0])).sum()) and not want[0][:63].any()
    empty = pref.emu_histogram(store, False, none, none, 0, m, pref.OPACITY, (0, 0, 0), e, 1)   # nothing selected
    assert not empty[0].any() and empty[1] == (np.inf, -np.inf)


@pytest.mark.parametrize("blocks,ctas", [(1, 1), (5, 5), (8, 3), (6, 2)])
def test_histogram_ctas_interleaved(blocks, ctas):
    """Several CTAs at once, each with its own shared histogram, flushing into the same 64-bit counters and min / max keys."""
    rng = np.random.default_rng(blocks * 10 + ctas)
    m = 9000 + 7
    store = store_of(rng, 2, True, m)
    hid, sel = masks_of(rng, m)
    e = np.geomspace(1e-4, 50.0, 200).astype(F32)
    for prop in (pref.SIZE, pref.COLOR):
        want = pref.histogram_rule(store, True, hid, sel, 11, m - 20, prop, (0, 0, 0), e, 0)
        assert_hist(pref.emu_histogram(store, True, hid, sel, 11, m - 20, prop, (0, 0, 0), e, 0, blocks=blocks, ctas=ctas), want)


# ---- the Python helper and the NULL-context checks ------------------------------------------------------------------------------
def test_splat_filter_helper():
    f = splat_filter(_lib.GSR_PROP_COLOR_DISTANCE, 0.0, 0.25, (1.0, 0.0, 0.5))
    assert C.sizeof(_lib.GsrSplatFilter) == 24
    assert (f.property, f.lo, f.hi, list(f.rgb)) == (4, 0.0, 0.25, [1.0, 0.0, 0.5])
    g = splat_filter(_lib.GSR_PROP_OPACITY)
    assert (g.lo, g.hi, list(g.rgb)) == (-INF, INF, [0.0, 0.0, 0.0])


def test_null_context_is_refused():
    L = _lib.lib()
    f = splat_filter(_lib.GSR_PROP_OPACITY, 0.0, 1.0)
    e = (C.c_float * 2)(0.0, 1.0)
    counts = (C.c_uint64 * 4)(9, 9, 9, 9)
    mm = (C.c_float * 2)(5.0, 5.0)
    assert L.gsr_select_where(None, C.byref(f), 1, -1, 0) == _lib.GSR_ERR_INVALID
    assert L.gsr_splat_histogram(None, C.byref(f), -1, 0, e, 1, counts, mm) == _lib.GSR_ERR_INVALID
    assert list(counts) == [9, 9, 9, 9] and list(mm) == [5.0, 5.0]
