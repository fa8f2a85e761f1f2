"""Splat delete and duplicate without a GPU (include/gsr.h "Splat delete and duplicate"): the emulated compact_store_kernel, with several
CTAs interleaving through their look-backs, and its follow-up kernels bit for bit against the numpy rule; vacant slots in the emulated
projection against the same slots hidden; the remap helper and the NULL-context checks."""
import ctypes as C

import numpy as np
import pytest

from godotgaussiansplatting_b200 import _lib
from tests import delete_reference as dref
from tests.transform_reference import sh_planes

F32, U32 = np.float32, np.uint32
TILE = 256   # splats per CTA tile


def store_of(rng, planes, stride):
    """Random words with NaN, +-0 and inf sprinkled in: every one must move bit for bit."""
    s = rng.normal(size=(planes, stride, 4)).astype(F32)
    w = s.view(U32)
    special = np.array([0x7FC00000, 0x7FA00001, 0xFFC00123, 0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x00000001], dtype=U32)
    pick = rng.random(w.shape) < 0.05
    w[pick] = special[rng.integers(0, special.size, int(pick.sum()))]
    return s


def hidden_mask(kind, m, n, rng):
    h = np.zeros(m, dtype=bool)
    if kind == "none":
        pass
    elif kind == "all":
        h[:n] = True
    elif kind == "one_kept_at_end":
        h[:n - 1] = True
    elif kind == "alternating":
        h[:n:2] = True
    elif kind == "front":   # every later splat moves down by 100: each tile's destinations overlap its predecessor's sources
        h[:100] = True
    elif kind == "runs":   # runs that start and end inside tiles and cross tile boundaries
        for lo, hi in ((TILE - 40, 2 * TILE + 17), (3 * TILE + 5, 3 * TILE + 6), (5 * TILE - 1, 7 * TILE + 3)):
            h[lo:min(hi, n)] = True
    else:
        h[:] = rng.random(m) < 0.3
    h[n:] = rng.random(m - n) < 0.5   # bits above n: the delete clears them, the cloud ignores them
    return h


KINDS = ["none", "all", "one_kept_at_end", "alternating", "runs", "random"]


def assert_same(got, want):
    gs, gh, gsel, gk = got
    ws, wh, wsel, wk = want
    assert gk == wk
    np.testing.assert_array_equal(gs.view(U32), ws.view(U32))
    np.testing.assert_array_equal(gh, wh)
    np.testing.assert_array_equal(gsel, wsel)


@pytest.mark.parametrize("bands", [1, 2, 3, 4])
@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("kind", KINDS)
def test_emulated_delete_is_the_rule(bands, half, kind):
    rng = np.random.default_rng(bands * 100 + half * 10 + KINDS.index(kind))
    m, n = 8 * TILE + 45, 8 * TILE - 19           # max_splats and n not multiples of 32, n below max_splats
    stride = (m + 255) // 256 * 256
    store = store_of(rng, 3 + sh_planes(bands, half), stride)
    hid = hidden_mask(kind, m, n, rng)
    sel = (rng.random(m) < 0.4) & ~hid
    sel[n:] |= rng.random(m - n) < 0.3           # selected bits above n are dropped
    sel &= ~hid
    want = dref.delete_rule(store, hid, sel, n)
    assert_same(dref.emu_delete(store, bands, half, hid, sel, n, ctas=4), want)
    if kind == "none":
        np.testing.assert_array_equal(want[0].view(U32), store.view(U32))   # nothing moves, nothing is vacated
    if kind == "runs":   # other interleavings give the same store
        assert_same(dref.emu_delete(store, bands, half, hid, sel, n, ctas=8), want)
        assert_same(dref.emu_delete(store, bands, half, hid, sel, n, ctas=1), want)


@pytest.mark.parametrize("bands,half", [(1, False), (4, False), (4, True)])
@pytest.mark.parametrize("kind", ["front", "runs", "alternating", "random"])
@pytest.mark.parametrize("ctas", [2, 4, 8])
def test_emulated_delete_waits_for_a_slow_predecessor(bands, half, kind, ctas):
    """The in-place ordering: the first CTA of every wave is held between its first look-back and its loads for 400 scheduler rounds,
    so its successors, whose destinations overlap its sources, run as far as the kernel lets them.  They must wait in their second
    look-back until it has read its sources (a second look-back that accepted EARLY words would overwrite them first)."""
    rng = np.random.default_rng(2000 + bands * 100 + half * 10 + ctas)
    m, n = 8 * TILE + 45, 8 * TILE - 19
    store = store_of(rng, 3 + sh_planes(bands, half), (m + 255) // 256 * 256)
    hid = hidden_mask(kind, m, n, rng)
    sel = (rng.random(m) < 0.4) & ~hid
    assert_same(dref.emu_delete(store, bands, half, hid, sel, n, ctas=ctas, slow=400), dref.delete_rule(store, hid, sel, n))


@pytest.mark.parametrize("bands", [1, 2, 3, 4])
@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("kind", ["none", "one", "alternating", "runs", "random"])
def test_emulated_duplicate_is_the_rule(bands, half, kind):
    rng = np.random.default_rng(1000 + bands * 100 + half * 10 + len(kind))
    n = 4 * TILE + 13
    m = 2 * n + 7
    stride = (m + 255) // 256 * 256
    store = store_of(rng, 3 + sh_planes(bands, half), stride)
    hid = rng.random(m) < 0.2
    sel = np.zeros(m, dtype=bool)
    if kind == "one":
        sel[n - 1] = True
    elif kind == "alternating":
        sel[1:n:2] = True
    elif kind == "runs":
        sel[TILE - 3:2 * TILE + 40] = True
        sel[3 * TILE + 31:3 * TILE + 33] = True
    elif kind == "random":
        sel[:] = rng.random(m) < 0.35
    sel[n:] |= rng.random(m - n) < 0.3           # selected bits above n are not copied
    sel &= ~hid
    want = dref.duplicate_rule(store, hid, sel, n)
    got = dref.emu_duplicate(store, bands, half, hid, sel, n, m, ctas=4)
    assert_same(got, want)
    assert got[3] == int(sel[:n].sum())


def test_emulated_duplicate_that_does_not_fit_writes_nothing():
    rng = np.random.default_rng(5)
    n, m = 1000, 1500
    store = store_of(rng, 3 + sh_planes(4, False), 1536)
    hid = np.zeros(m, dtype=bool)
    sel = np.zeros(m, dtype=bool)
    sel[:501] = True
    got = dref.emu_duplicate(store, 4, False, hid, sel, n, m)
    assert got[3] == -2 - 501
    np.testing.assert_array_equal(got[0].view(U32), store.view(U32))
    np.testing.assert_array_equal(got[2], sel)
    sel[500] = False   # exactly fits
    assert_same(dref.emu_duplicate(store, 4, False, hid, sel, n, m), dref.duplicate_rule(store, hid, sel, n))


def test_delete_then_duplicate_chain():
    """A delete of a delete's result and a duplicate of it: the rules compose like the kernels."""
    rng = np.random.default_rng(9)
    m, n = 3000, 2500
    store = store_of(rng, 3 + sh_planes(3, True), 3072)
    hid = rng.random(m) < 0.25
    sel = (rng.random(m) < 0.2) & ~hid
    s1 = dref.emu_delete(store, 3, True, hid, sel, n)
    assert_same(s1, dref.delete_rule(store, hid, sel, n))
    s2 = dref.emu_duplicate(s1[0], 3, True, s1[1], s1[2], s1[3], m)
    assert_same(s2, dref.duplicate_rule(s1[0], s1[1], s1[2], s1[3]))


def test_remap_is_the_rank_rule():
    rng = np.random.default_rng(2)
    n = 777
    hid = rng.random(n) < 0.4
    r = dref.delete_remap(hid, n)
    want = np.array([-1 if hid[s] else int((~hid[:s]).sum()) for s in range(n)])
    np.testing.assert_array_equal(r, want)
    kept = np.flatnonzero(~hid)
    np.testing.assert_array_equal(r[kept], np.arange(kept.size))


# ---- vacant slots in the emulated projection -------------------------------------------------------------------------------
@pytest.mark.parametrize("bands", [1, 2, 4])
@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("cut", [False, True])
@pytest.mark.parametrize("inst", [False, True])
@pytest.mark.parametrize("ortho", [False, True])
def test_vacant_slots_are_hidden_splats_in_the_emulated_projection(bands, aa, cut, inst, ortho, monkeypatch):
    """A store with scattered vacant slots (written as a delete leaves them: plane-0 xyz the quiet NaN, every other word +0) gives
    exactly the keys, the values in emission order, V, the last tile and the records of the emitted ids of the same store with those
    slots' splats hidden (highlight off)."""
    from tests import cutout_reference as cr
    from tests import ortho_reference as oref
    from tests import test_splat_selection as tss
    from tests import variant_matrix as vm
    from tests.test_depth_order import H, W, scene
    from tests.test_instances import rigid
    splat60, vp, ub = scene()
    if ortho:
        vp, ub = oref.ortho_camera(W, H, size=2.6, near=0.5, far=4.5, frame=25)
    n = splat60.shape[0]
    rng = np.random.default_rng(bands * 16 + aa * 8 + cut * 4 + inst * 2 + ortho)
    vac = rng.random(n) < 0.3
    layout = [(3, 700, rigid(3)), (100, 999, rigid(4)), (0, 33, rigid(5))] if inst else None
    vols = vm.cutouts(splat60, cr.positions(splat60, 1.0, layout)[1]) if cut else None
    v = 0.3 if aa else 0.0
    off = ((0.0, 0.0, 0.0), 0.0)
    none = np.zeros(n, dtype=bool)
    want = tss.emu_frame(splat60, vp, ub, vac, none, off, layout, ortho, bands, v, vols)
    plain_store_of = tss.store_of

    def vacant_store_of(s60, b):
        store = plain_store_of(s60, b)
        dref.vacate_slots(store, vac)
        return store

    monkeypatch.setattr(tss, "store_of", vacant_store_of)
    recs, keys, vals, vis, last = tss.emu_frame(splat60, vp, ub, none, none, off, layout, ortho, bands, v, vols)
    np.testing.assert_array_equal(keys, want[1])
    np.testing.assert_array_equal(vals, want[2])
    assert (vis, last) == (want[3], want[4])
    ids = np.unique(vals)
    assert ids.size > 100
    np.testing.assert_array_equal(recs[ids].view(U32), want[0][ids].view(U32))


def test_null_context_is_refused():
    L = _lib.lib()
    k = C.c_uint64(7)
    assert L.gsr_delete_hidden(None, C.byref(k)) == _lib.GSR_ERR_INVALID
    assert L.gsr_duplicate_selection(None, C.byref(k)) == _lib.GSR_ERR_INVALID
    assert L.gsr_set_splat_count(None, 0) == _lib.GSR_ERR_INVALID
    assert k.value == 7
