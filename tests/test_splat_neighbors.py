"""Splat neighbourhood selection without a GPU (include/gsr.h "Splat neighbourhood selection"): the emulated kernels of
csrc/neighbors.cu, with several CTAs interleaving their union-find hooks, bit for bit against the numpy brute-force rule of
tests/neighbor_reference in the mask words and the stats -- every mode under every op on clumpy clouds with hidden, vacant, NaN and
infinite splats; pairs at d2 = r2 and one ulp beyond across cell boundaries near 0, near +-1e4 and at the int64 clamp; coincident
duplicates; clusters split by hidden and vacant links; ranges inside words; forced hash collisions; a long chain; the budget at and
over its limit -- and the serial C++ grid reference against the same rule."""
import ctypes as C

import numpy as np
import pytest

from godotgaussiansplatting_b200 import _lib
from tests import neighbor_reference as nr
from tests import selection_reference as sref

F32 = np.float32
NAN, INF = np.nan, np.inf


def clumpy(rng, m, clumps=40, isolated=60, scale=10.0, spread=0.3):
    """plane0 (m, 4): clumps of 3..150 splats of a few radii, isolated splats, the rest of [0, m) vacant (NaN x)."""
    p = np.full((m, 4), 0.0, F32)
    p[:, 0] = NAN
    pts = []
    for _ in range(clumps):
        c = rng.uniform(-scale, scale, 3)
        k = int(rng.integers(3, 150))
        pts.append(c + rng.normal(size=(k, 3)) * spread * rng.uniform(0.2, 1.0))
    pts = np.concatenate(pts)[:int(0.9 * m) - isolated]
    pts = np.concatenate([pts, rng.uniform(-scale, scale, (isolated, 3))]).astype(F32)
    slots = rng.permutation(m)[:len(pts)]
    p[slots, :3] = pts
    return p


def masks(rng, m, hidden=0.08, selected=0.02):
    hid = rng.random(m) < hidden
    return hid, (rng.random(m) < selected) & ~hid


def check(plane0, hid, sel, first, count, radius, mode, threshold, ops=range(4), bucket_bits=0, ctas=4, cpp=True):
    for op in ops:
        want, wst = nr.select_rule(plane0, hid, sel, first, count, radius, mode, threshold, op)
        rc, got, gst = nr.emu_select(plane0, hid, sel, first, count, radius, mode, threshold, op, bucket_bits=bucket_bits, ctas=ctas)
        assert rc == 0
        np.testing.assert_array_equal(got, want, err_msg=f"mode {mode} op {op}")
        assert gst == wst, (mode, op, gst, wst)
        if cpp:
            rgot, rst = nr.ref_select(plane0, hid, sel, first, count, radius, mode, threshold, op)
            np.testing.assert_array_equal(rgot, want, err_msg=f"C++ reference, mode {mode} op {op}")
            assert rst == wst
    return wst


# ---- every mode under every op ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", nr.MODES)
def test_every_mode_and_op_is_the_rule(mode):
    rng = np.random.default_rng(100 + mode)
    m = 3000 + 13
    p = clumpy(rng, m)
    p[rng.choice(m, 20, replace=False), rng.integers(0, 3, 20)] = rng.choice([NAN, INF, -INF], 20)
    hid, sel = masks(rng, m)
    st = None
    for radius, thr in ((0.25, 3), (0.6, 8), (2.0, 40)):
        st = check(p, hid, sel, 0, m - 77, radius, mode, thr)
        assert st[0] > 1000
    if mode == nr.SPARSE:
        assert 0 < st[1] < st[0]
    if mode >= nr.CONNECTED:
        assert st[3] > 1 and st[4] > 1


@pytest.mark.parametrize("mode", nr.MODES)
def test_ranges_inside_words_and_forced_collisions(mode):
    rng = np.random.default_rng(200 + mode)
    m = 2000 + 5
    p = clumpy(rng, m, clumps=25, isolated=40, scale=4.0)
    hid, sel = masks(rng, m, selected=0.05)
    check(p, hid, sel, 37, 1500 - 11, 0.5, mode, 5)                    # a range that starts and ends inside a word
    check(p, hid, sel, 0, m, 0.5, mode, 5, bucket_bits=1)             # two buckets: every bucket impure
    check(p, hid, sel, 0, m, 0.5, mode, 5, bucket_bits=3, ctas=8)
    check(p, hid, sel, 64, 0, 0.5, mode, 5, cpp=False)                # an empty range: SET clears everything


# ---- the exact boundary ---------------------------------------------------------------------------------------------------------
def last_neighbour(base, r):
    """The largest float32 x > base with fl((x - base)^2) <= fl(r r)."""
    r2 = F32(r) * F32(r)
    x = F32(base) + F32(r)
    while (F32(x) - F32(base)) ** 2 > r2:
        x = np.nextafter(x, F32(-INF))
    while (F32(np.nextafter(x, F32(INF))) - F32(base)) ** 2 <= r2:
        x = np.nextafter(x, F32(INF))
    return F32(x)


@pytest.mark.parametrize("radius,bases", [
    (0.5, [0.0, -0.0, 1e-30, -0.2, 0.49999, 0.5000005, -0.5000001]),          # near 0, across the cells at 0 and +-h
    (0.01, [1e4, -1e4, 10000.0078125, -9999.99]),                             # near +-1e4
    (2.0 ** -40, [2.0 ** 22, -(2.0 ** 22), 2.0 ** 22 - 2.0 ** -1]),           # cells near 2^62
    (2.0 ** -60, [1e4, -1e4, 3.0]),                                           # cells clamped to +-2^62
])
def test_pairs_at_the_radius_and_one_ulp_beyond(radius, bases):
    pts = []
    for k, b in enumerate(bases):
        b = F32(b)
        x = last_neighbour(b, radius)
        y = F32(1000.0 * k)
        pts += [(b, y, 0.0), (x, y, 0.0),                                          # d2 <= r2: neighbours
                (b, y + 10.0, 0.0), (np.nextafter(x, F32(INF)), y + 10.0, 0.0),   # one ulp beyond
                (b, y + 20.0, 0.0), (b, y + 20.0, 0.0)]                           # coincident
        if b + 4 * radius != b:
            pts += [(b, y + 30.0, 0.0), (b, y + 30.0, x - b + b)]                 # the same gap along z
    m = len(pts) + 7
    p = np.full((m, 4), 0.0, F32)
    p[:, 0] = NAN
    p[:len(pts), :3] = np.array(pts, F32)
    hid = np.zeros(m, bool)
    sel = np.zeros(m, bool)
    sel[0] = sel[2] = True
    for mode in nr.MODES:
        check(p, hid, sel, 0, m, radius, mode, 2)
    inside, _ = nr.inside_rule(p, hid, sel, 0, m, radius, nr.SPARSE, 1)
    assert not inside[0] and not inside[1] and inside[2] and inside[3] and not inside[4]


# ---- clusters ---------------------------------------------------------------------------------------------------------------------
def chain(m, n, gap, rng):
    """n splats on a line, gap apart, in random slots; the rest vacant."""
    p = np.full((m, 4), 0.0, F32)
    p[:, 0] = NAN
    slots = rng.permutation(m)[:n]
    p[slots, 0] = (np.arange(n) * gap).astype(F32)
    p[slots, 1] = np.sin(np.arange(n)).astype(F32) * F32(0.1 * gap)
    p[slots, 2] = 0.0
    return p, slots


def test_a_long_chain_is_one_cluster():
    rng = np.random.default_rng(7)
    m = 4000 + 9
    p, slots = chain(m, 3500, 0.8, rng)
    hid = np.zeros(m, bool)
    sel = np.zeros(m, bool)
    sel[slots[-1]] = True
    for mode, thr in ((nr.CONNECTED, 1), (nr.SMALL, 3501)):
        st = check(p, hid, sel, 0, m, 1.0, mode, thr, ops=[sref.SET], ctas=8)
        assert st[3] == 1 and st[4] == 3500 and st[1] == 3500


def test_hidden_and_vacant_links_split_clusters():
    rng = np.random.default_rng(8)
    m = 1200
    p, slots = chain(m, 1000, 0.8, rng)
    hid = np.zeros(m, bool)
    hid[slots[300]] = True                  # a hidden link
    p[slots[600], :3] = NAN                 # a vacant link
    p[slots[800], 1] = INF                  # an infinite one
    sel = np.zeros(m, bool)
    sel[slots[0]] = True
    for mode in (nr.CONNECTED, nr.SMALL):
        st = check(p, hid, sel, 0, m, 1.0, mode, 250)
        assert st[3] == 4 and st[4] == 300
    inside, _ = nr.inside_rule(p, hid, sel, 0, m, 1.0, nr.CONNECTED, 1)
    assert inside.sum() == 300


# ---- the budget ---------------------------------------------------------------------------------------------------------------------
def test_budget_at_and_over_the_limit():
    rng = np.random.default_rng(9)
    m = 1500 + 3
    p = clumpy(rng, m, clumps=10, isolated=10, scale=2.0)
    hid, sel = masks(rng, m)
    _, want = nr.select_rule(p, hid, sel, 0, m, 0.7, nr.GROW, 1, sref.ADD)
    c = want[2]
    assert c > 10000
    rc, got, st = nr.emu_select(p, hid, sel, 0, m, 0.7, nr.GROW, 1, sref.ADD, limit=c)
    assert rc == 0 and st == want
    rc, got, st = nr.emu_select(p, hid, sel, 0, m, 0.7, nr.GROW, 1, sref.ADD, limit=c - 1)
    assert rc == 1 and st[2] == c
    np.testing.assert_array_equal(got, sel)   # refused: the selection is untouched


def test_candidates_follow_the_cell_rule():
    """The work measure does not depend on the bucket count, and a huge radius puts every pair into it."""
    rng = np.random.default_rng(10)
    m = 900
    p = clumpy(rng, m, clumps=8, isolated=20, scale=3.0)
    hid = np.zeros(m, bool)
    sel = np.zeros(m, bool)
    part = nr.participants(p, hid, 0, m)
    for bits in (0, 1, 2, 12):
        _, _, st = nr.emu_select(p, hid, sel, 0, m, 0.4, nr.SPARSE, 1, sref.SET, bucket_bits=bits)
        assert st[2] == nr.candidates(p[:, :3], part, 0.4)
    _, _, st = nr.emu_select(p, hid, sel, 0, m, 1e6, nr.SPARSE, 1, sref.SET)
    assert st[2] == part.sum() ** 2


def test_null_context_is_refused():
    L = _lib.lib()
    q = _lib.GsrNeighborhood(_lib.GSR_NEIGHBOR_SPARSE, 1.0, 1, -1)
    assert L.gsr_select_neighborhood(None, C.byref(q), 0, None) == _lib.GSR_ERR_INVALID
    assert C.sizeof(_lib.GsrNeighborhood) == 16 and C.sizeof(_lib.GsrNeighborhoodStats) == 40


def test_all_modes_of_the_cpp_reference_in_one_pass():
    rng = np.random.default_rng(11)
    m = 2500
    p = clumpy(rng, m)
    hid, sel = masks(rng, m)
    allm = nr.ref_all_modes(p, hid, sel, 0, m, 0.5, 4)
    for mode in nr.MODES:
        inside, st = nr.inside_rule(p, hid, sel, 0, m, 0.5, mode, 4)
        np.testing.assert_array_equal(allm[mode][0], inside)
        assert allm[mode][1] == st
