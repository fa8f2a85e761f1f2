"""Splat export without a GPU (include/gsr.h "Splat export"): the emulated export_count_kernel and export_ply_kernel, with several CTAs
interleaving through their look-backs, against the rule -- which splats, in which order -- and against store_to_table, the float64
numpy export: positions, normals and coefficients bit for bit, opacity within 1 ulp, scales and rotations within the decomposition's
bars, including the covariances a cloud is full of.  Then determinism, the round trip through the ingest's rule and the NULL refusals."""
import ctypes as C

import numpy as np
import pytest

from godotgaussiansplatting_b200 import _lib
from godotgaussiansplatting_b200.ply_file import PlyFile, degree_properties, swizzle_splats
from tests import export_reference as xr

F32, U32 = np.float32, np.uint32
TILE = 256   # splats per CTA tile


def ply_table(rng, n):
    """n random degree-3 3DGS vertices with the scales, rotations and opacities of a trained cloud."""
    t = np.zeros((n, 62), dtype=F32)
    t[:, 0:3] = rng.normal(size=(n, 3)) * 3.0
    t[:, 6:54] = rng.normal(size=(n, 48)) * 0.5
    t[:, 54] = rng.normal(size=n) * 3.0
    t[:, 55:58] = rng.uniform(-7.0, -1.0, size=(n, 3))
    t[:, 58:62] = rng.normal(size=(n, 4))
    return t


def cloud(rng, bands, half, m, n, specials=True):
    """A store of m slots (stride a multiple of 256) with a trained-looking cloud in [0, n), special covariances and opacities at some
    slots, vacant slots and NaN positions inside [0, n), and random words above n."""
    stride = (m + 255) // 256 * 256
    store = xr.store_from_structs(swizzle_splats(ply_table(rng, m), 0.0), bands, half, stride)
    if specials:
        cases = xr.special_covariances(rng)
        slots = rng.choice(n, size=min(n, 2 * len(cases)), replace=False)
        for k, s in enumerate(slots):
            xr.put_special(store, s, cases[k % len(cases)][1])
        for k, o in enumerate((0.0, 1.0, np.nan, -0.1, 1.5, 0.5, 1e-30, 1.0 - 2.0 ** -24)):
            store[2, (7 * k + 3) % n, 2] = o
        vac = rng.random(n) < 0.05
        w = store.view(U32)
        w[:, np.flatnonzero(vac)] = 0
        w[0, np.flatnonzero(vac), :3] = xr.QNAN
        store[0, (11 * np.arange(4) + 5) % n, rng.integers(0, 3)] = np.nan   # one NaN coordinate: vacant too
        store[0, (13 * np.arange(4) + 2) % n, 0] = np.inf                    # an infinite position is exported as it is
    return store


def masks(rng, m, kind):
    if kind == "off":
        return None, None
    hid = rng.random(m) < 0.3
    sel = (rng.random(m) < 0.4) & ~hid
    return hid, sel


SCOPES = [("kept", "off"), ("kept", "on"), ("selected", "on"), ("selected", "off")]


@pytest.mark.parametrize("bands", [1, 2, 3, 4])
@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("scope,mask", SCOPES)
def test_emulated_export_is_the_rule(bands, half, scope, mask):
    """Every degree d <= the stored one, with max_splats and n not multiples of 32 and n below max_splats."""
    rng = np.random.default_rng(bands * 100 + half * 10 + SCOPES.index((scope, mask)))
    m, n = 4 * TILE + 45, 4 * TILE - 19
    store = cloud(rng, bands, half, m, n)
    hid, sel = masks(rng, m, mask)
    for degree in range(bands):
        rows = xr.emu_export(store, bands, half, hid, sel, n, scope == "selected", degree, ctas=4)
        idx = xr.check_rows(rows, store, n, bands, half, hid, sel, scope == "selected", degree)
        if scope == "selected" and mask == "off":
            assert idx.size == 0
        else:
            assert idx.size > 100
        assert xr.emu_export(store, bands, half, hid, sel, n, scope == "selected", degree, count_only=True) == idx.size


@pytest.mark.parametrize("bands,half", [(1, False), (4, False), (4, True)])
@pytest.mark.parametrize("ctas", [2, 4, 8])
def test_emulated_export_waits_for_a_slow_predecessor(bands, half, ctas):
    """The first CTA of every wave is held before it publishes its count for 400 scheduler rounds: its successors must wait in their
    look-backs, and every row still lands at its rank."""
    rng = np.random.default_rng(3000 + bands * 100 + half * 10 + ctas)
    m, n = 8 * TILE + 45, 8 * TILE - 19
    store = cloud(rng, bands, half, m, n, specials=False)
    hid, sel = masks(rng, m, "on")
    rows = xr.emu_export(store, bands, half, hid, sel, n, False, bands - 1, ctas=ctas, slow=400)
    xr.check_rows(rows, store, n, bands, half, hid, sel, False, bands - 1)
    np.testing.assert_array_equal(rows.view(U32), xr.emu_export(store, bands, half, hid, sel, n, False, bands - 1, ctas=1).view(U32))


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, TILE - 1, TILE, TILE + 1, 2 * TILE, 3 * TILE + 7])
def test_tile_boundary_counts(n):
    rng = np.random.default_rng(n)
    m = 3 * TILE + 40
    store = cloud(rng, 2, False, m, max(n, 1), specials=False)
    hid, sel = masks(rng, m, "on")
    for scope in (False, True):
        rows = xr.emu_export(store, 2, False, hid, sel, n, scope, 1, ctas=3)
        xr.check_rows(rows, store, n, 2, False, hid, sel, scope, 1)


def test_empty_results():
    rng = np.random.default_rng(4)
    m, n = 2 * TILE + 3, 2 * TILE
    store = cloud(rng, 3, True, m, n, specials=False)
    hid = np.zeros(m, dtype=bool)
    hid[:n] = True
    assert xr.emu_export(store, 3, True, hid, np.zeros(m, dtype=bool), n, False, 2).shape == (0, 41)
    assert xr.emu_export(store, 3, True, np.zeros(m, dtype=bool), np.zeros(m, dtype=bool), n, True, 2).shape == (0, 41)
    w = store.view(U32)   # every slot vacant
    w[0, :n, :3] = xr.QNAN
    assert xr.emu_export(store, 3, True, None, None, n, False, 0).shape == (0, 17)


def test_special_covariances_decompose():
    """Isotropic splats, repeated pairs, needles and discs (ratio 1e-12), zero, a slightly negative eigenvalue, 180-degree rotations
    and non-finite words, one per slot: the decomposition's bars, plus the exact outcomes the rule fixes."""
    rng = np.random.default_rng(11)
    cases = xr.special_covariances(rng)
    n = len(cases)
    store = cloud(rng, 1, False, n, n, specials=False)
    for s, (_, S) in enumerate(cases):
        xr.put_special(store, s, S)
    rows = xr.emu_export(store, 1, False, None, None, n, False, 0, ctas=1)
    xr.check_rows(rows, store, n, 1, False, None, None, False, 0)
    names = degree_properties(0)
    sc, rot = names.index("scale_0"), names.index("rot_0")
    for s, (name, S) in enumerate(cases):
        r = rows[s]
        if name == "isotropic":
            assert r[sc] == r[sc + 1] == r[sc + 2]
            np.testing.assert_array_equal(r[rot:rot + 4], [1, 0, 0, 0])
        elif name == "zero":
            np.testing.assert_array_equal(r[sc:sc + 3], np.full(3, F32(0.5 * np.log(np.finfo(np.float64).tiny))))
        elif name == "nonfinite":
            assert np.isnan(r[sc:sc + 3]).all()
            np.testing.assert_array_equal(r[rot:rot + 4], [1, 0, 0, 0])
        elif name == "slightly_negative":
            assert r[sc] == F32(0.5 * np.log(np.finfo(np.float64).tiny))


def test_opacity_rule():
    rng = np.random.default_rng(12)
    ops = np.array([0.0, 1.0, np.nan, -0.1, 1.5, 0.5, 1e-30, 0.25, 1.0 - 2.0 ** -24, 2.0 ** -149], dtype=F32)
    store = cloud(rng, 1, False, ops.size, ops.size, specials=False)
    store[2, :ops.size, 2] = ops
    rows = xr.emu_export(store, 1, False, None, None, ops.size, False, 0)
    o = rows[:, degree_properties(0).index("opacity")]
    assert o[0] == -104.0 and o[1] == 104.0
    np.testing.assert_array_equal(o[2:5].view(U32), np.zeros(3, dtype=U32))   # +0
    with np.errstate(divide="ignore", invalid="ignore"):
        want = np.log(ops.astype(np.float64)) - np.log1p(-ops.astype(np.float64))
    assert (xr.ulp_distance(o[5:], np.clip(want[5:], -104, 104).astype(F32)) <= 1).all()


def test_a_row_depends_only_on_the_splat():
    """The same splat copied to several indices (in several tiles, warps and lanes) exports identical bits, in either scope."""
    rng = np.random.default_rng(13)
    m = n = 3 * TILE + 17
    store = cloud(rng, 4, True, m, n, specials=False)
    src = [5, 300, 700]
    copies = {s: rng.choice(np.setdiff1d(np.arange(n), src), size=6, replace=False) for s in src}
    for s, dst in copies.items():
        store[:, dst] = store[:, s][:, None]
    hid = np.zeros(m, dtype=bool)
    sel = np.zeros(m, dtype=bool)
    sel[np.concatenate([[s] for s in src] + list(copies.values()))] = True
    kept = xr.emu_export(store, 4, True, hid, sel, n, False, 3)
    chosen = xr.emu_export(store, 4, True, hid, sel, n, True, 3, ctas=2)
    pos = {int(s): i for i, s in enumerate(np.flatnonzero(sel[:n]))}
    for s, dst in copies.items():
        for d in dst:
            np.testing.assert_array_equal(kept[d].view(U32), kept[s].view(U32))
            np.testing.assert_array_equal(chosen[pos[int(d)]].view(U32), kept[s].view(U32))


@pytest.mark.parametrize("bands,half", [(1, False), (2, True), (3, False), (4, False), (4, True)])
def test_round_trip_through_the_ingest(bands, half):
    """Exported rows back through the ingest's rule (swizzle_splats with PlyFile.layout()): positions and coefficients bit for bit,
    opacity within 2 ulp (exact at 0 and 1), covariance words within 1e-5 lambda_max."""
    rng = np.random.default_rng(20 + bands + 10 * half)
    n = 2 * TILE + 9
    store = cloud(rng, bands, half, n, n, specials=False)
    store[2, 0, 2], store[2, 1, 2] = 0.0, 1.0
    for s, (name, S) in enumerate(xr.special_covariances(rng)):
        if name != "nonfinite" and name != "slightly_negative":
            xr.put_special(store, 10 + s, S)
    rows = xr.emu_export(store, bands, half, None, None, n, False, bands - 1)
    ply = PlyFile.from_array(rows, degree_properties(bands - 1))
    back = xr.store_from_structs(swizzle_splats(ply.table, 0.0, ply.layout()), bands, half, store.shape[1])
    np.testing.assert_array_equal(back[0, :n, :3].view(U32), store[0, :n, :3].view(U32))
    np.testing.assert_array_equal(back[3:, :n].view(U32), store[3:, :n].view(U32))
    o, o2 = store[2, :n, 2], back[2, :n, 2]
    assert o2[0] == 0.0 and o2[1] == 1.0
    assert xr.ulp_distance(o, o2).max() <= 2
    S, S2 = xr.covariances(store, np.arange(n)), xr.covariances(back, np.arange(n))
    lmax = np.abs(np.linalg.eigvalsh(S)).max(axis=1)
    assert (np.abs(S2 - S).max(axis=(1, 2)) <= 1e-5 * lmax).all()


def test_null_context_is_refused():
    L = _lib.lib()
    r = C.c_uint64(7)
    assert L.gsr_export_ply(None, _lib.GSR_EXPORT_KEPT, -1, None, 0, C.byref(r)) == _lib.GSR_ERR_INVALID
    assert r.value == 7
