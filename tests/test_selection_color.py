"""Selection colour edits without a GPU (include/gsr.h "Splat colour edits"): the emulated recolor_selection_kernel bit for bit against the
numpy rule of tests/color_reference fed the library's own constants, the library's float64 constants against an independent numpy
derivation, the meaning of an edit for the SH colour, the color_edit() helper of the Python mirror, and the export of the edited cloud
(store_to_table) through the emulated ingest."""
import ctypes as C

import numpy as np
import pytest

from godotgaussiansplatting_b200.rasterizer import REC709_LUMA, color_edit, pack_mask, store_to_table
from godotgaussiansplatting_b200.synthetic import synthetic_ply_table
from tests import color_reference as cref
from tests import transform_reference as tref
from tests.test_selection_transform import N, STRIDE, random_store, selection

F32, U32 = np.float32, np.uint32

EDITS = {
    "identity": color_edit(),
    "gain": color_edit(gain=(1.2, 0.8, 1.05)),
    "saturation": color_edit(saturation=1.6),                 # negative off-diagonal entries
    "hue": color_edit(hue=40.0),
    "offset": cref.edit_struct([[1, 0, 0, 0.1], [0, 1, 0, -0.05], [0, 0, 1, 0.2]]),
    "bands": cref.edit_struct(band_scale=(0.0, 0.5, 1.0)),
    "opacity": color_edit(opacity=2.5, opacity_offset=-0.6),  # o in [0, 1) -> [-0.6, 1.9): both clamps
}


def special_store(bands, half, seed):
    """random_store plus opacity specials: NaN, +-0, a negative value, and values the opacity edit pushes past both clamps."""
    st = random_store(bands, half, seed=seed)
    st[2, 20, 2], st[2, 21, 2], st[2, 22, 2], st[2, 23, 2], st[2, 24, 2] = np.nan, -0.0, 0.0, -0.25, 1.0
    return st


# ---- the kernel against the rule -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("edit", list(EDITS))
@pytest.mark.parametrize("snapshot", [False, True])
@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("bands", [1, 2, 3, 4])
def test_kernel_is_the_rule(bands, half, snapshot, edit):
    k41 = cref.constants(EDITS[edit])
    store = special_store(bands, half, seed=bands)
    src = special_store(bands, half, seed=50 + bands) if snapshot else None
    for kind in ("random", "range", "all", "none"):
        sel = selection(kind, seed=bands + 3)
        got = cref.emu_recolor(store, bands, half, pack_mask(sel, N), k41, src)
        want = cref.oracle(store, bands, half, sel, k41, src)
        tref.assert_store_equal(got, want, half, f"{kind}")
        untouched = ~np.concatenate([sel, np.zeros(STRIDE - N, bool)])
        np.testing.assert_array_equal(got[:, untouched].view(U32), store[:, untouched].view(U32))   # unselected, hidden, padding
        if kind == "all":
            o = got[2, 20:25, 2]
            assert o[0].view(U32) == 0 and o[1].view(U32) == 0   # NaN and -0 opacity become +0
            if edit == "opacity":
                o = got[2, :N, 2]
                assert (o == 0.0).sum() > 10 and (o == 1.0).sum() > 10, "both opacity clamps reached"
    if half and bands > 1 and edit == "gain":
        out = cref.oracle(store, bands, half, np.ones(N, bool), k41, src)
        words = out[3:, 12:14].view(U32)
        assert ((words & 0x7FFF) == 0x7BFF).any() or ((words >> 16 & 0x7FFF) == 0x7BFF).any()   # +-65504 reached


def test_identity_keeps_every_finite_word_but_negative_zero():
    # (an infinite coefficient does not survive: 0 * inf turns the other channels of its triple NaN)
    k41 = cref.constants(EDITS["identity"])
    for bands in (1, 2, 3, 4):
        for half in (False, True):
            store = special_store(bands, half, seed=7)
            store[:, 0:30] = store[:, 100:130]   # no specials
            if half:
                store[3, 5, 0] = np.uint32(0x3C008000).view(F32)   # halves -0 and 1
            else:
                store[3, 5, 1] = -0.0
            got = cref.emu_recolor(store, bands, half, pack_mask(np.ones(N, bool), N), k41)
            want = store.copy()
            if half:
                want[3, 5, 0] = np.uint32(0x3C000000).view(F32)
            else:
                want[3, 5, 1] = 0.0
            np.testing.assert_array_equal(got.view(U32), want.view(U32))


# ---- the constants ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("edit", list(EDITS) + ["graded"])
def test_constants_are_the_numpy_derivation(edit):
    e = EDITS.get(edit) or color_edit(gain=(1.1, 0.95, 1.3), brightness=-0.07, contrast=1.4, saturation=0.6, hue=-75.0, view_dependence=0.3,
                                       opacity=0.5, opacity_offset=0.25)
    np.testing.assert_array_equal(cref.constants(e).view(U32), cref.constants_numpy(e).view(U32))


def test_identity_constants():
    A, d, Ns, s, t = cref.unpack(cref.constants(EDITS["identity"]))
    np.testing.assert_array_equal(A.view(U32), np.eye(3, dtype=F32).view(U32))
    np.testing.assert_array_equal(d.view(U32), np.zeros(3, dtype=F32).view(U32))
    for l in (1, 2, 3):
        np.testing.assert_array_equal(Ns[l].view(U32), np.eye(3, dtype=F32).view(U32))
    assert (s, t) == (1.0, 0.0)


# ---- meaning: the SH colour of the edited coefficients --------------------------------------------------------------------------
def sh_colour(c, d):
    """(m, K, 3) coefficients, (n, 3) unit directions -> (m, n, 3) float64 colour before the clamp, and per band the view-dependent
    share."""
    c = np.asarray(c, dtype=np.float64)
    K = c.shape[1]
    base = 0.5 + cref.SH_C0 * c[:, 0, :]
    shares = []
    for l in range(1, int(np.sqrt(K))):
        P = tref.sh_poly(l, d)
        shares.append(np.einsum("nj,mjc->mnc", P, c[:, l * l:l * l + 2 * l + 1, :]))
    return base[:, None, :], shares


@pytest.mark.parametrize("edit", ["gain", "saturation", "hue", "offset", "bands", "graded"])
def test_edit_meaning(edit):
    e = EDITS.get(edit) or color_edit(gain=(1.1, 0.95, 1.3), brightness=-0.07, contrast=1.4, saturation=0.6, hue=-75.0, view_dependence=0.3)
    bands = 4
    store = random_store(bands, False, seed=31)
    rows = np.arange(20, 200)   # finite coefficients only
    got = cref.emu_recolor(store, bands, False, pack_mask(np.ones(N, bool), N), cref.constants(e))
    coeffs = lambda st: st[3:, rows].transpose(1, 0, 2).reshape(rows.size, -1)[:, :48].reshape(rows.size, 16, 3)   # noqa: E731
    d = np.random.default_rng(5).normal(size=(256, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    A, b = cref.affine(e)
    scale = np.array(e.band_scale[:], dtype=np.float64)
    b0, sh0 = sh_colour(coeffs(store), d)
    b1, sh1 = sh_colour(coeffs(got), d)
    before = b0 + sum(s * x for s, x in zip(scale, sh0))
    want = before @ A.T + b
    edited = b1 + sum(sh1)
    np.testing.assert_allclose(edited, want, atol=1e-5, rtol=0)


# ---- color_edit() ---------------------------------------------------------------------------------------------------------------
def fields(e):
    return np.concatenate([np.array(e.matrix[:], F32), np.array(e.band_scale[:], F32), np.array([e.opacity_scale, e.opacity_offset], F32)])


def test_color_edit_defaults_are_the_identity():
    np.testing.assert_array_equal(fields(color_edit()).view(U32), fields(cref.edit_struct()).view(U32))


def test_saturation_zero_is_grey():
    A, b = cref.affine(color_edit(saturation=0.0))
    np.testing.assert_array_equal(A[0], A[1])
    np.testing.assert_array_equal(A[1], A[2])
    np.testing.assert_allclose(A[0], REC709_LUMA, rtol=1e-7)
    cols = np.random.default_rng(1).random((100, 3))
    g = cols @ A.T + b
    assert (g[:, 0] == g[:, 1]).all() and (g[:, 1] == g[:, 2]).all()


def test_hue_360_is_the_identity():
    A, b = cref.affine(color_edit(hue=360.0))
    np.testing.assert_allclose(A, np.eye(3), atol=1e-6)
    np.testing.assert_allclose(b, 0.0, atol=1e-6)
    A, b = cref.affine(color_edit(hue=120.0))   # a third of a turn permutes the channels
    np.testing.assert_allclose(A, np.roll(np.eye(3), 1, axis=0), atol=1e-6)


def test_color_edit_composes_in_the_documented_order():
    gain, sat, hue, con, bri = np.array([1.2, 0.9, 1.1]), 1.4, 30.0, 0.8, 0.05
    e = color_edit(gain=gain, brightness=bri, contrast=con, saturation=sat, hue=hue, view_dependence=0.25, opacity=0.7, opacity_offset=0.1)
    A, b = cref.affine(e)
    cols = np.random.default_rng(2).random((100, 3))
    luma = np.asarray(REC709_LUMA)

    def steps(x):
        x = x * gain                                                   # 1. gain
        grey = (x @ luma)[:, None]
        x = grey + sat * (x - grey)                                    # 2. saturation: lerp from the luma grey
        k, a = np.ones(3) / np.sqrt(3.0), np.deg2rad(hue)
        x = x * np.cos(a) + np.cross(k, x) * np.sin(a) + np.outer(x @ k, k) * (1 - np.cos(a))   # 3. hue about the grey axis
        x = (x - 0.5) * con + 0.5                                      # 4. contrast about 0.5
        return x + bri                                                 # 5. brightness
    np.testing.assert_allclose(cols @ A.T + b, steps(cols), atol=1e-6)
    assert list(e.band_scale) == [0.25] * 3 and (e.opacity_scale, e.opacity_offset) == (np.float32(0.7), np.float32(0.1))
    # the order matters: contrast after brightness would move the offset
    assert abs(b[0] - (0.5 * (1 - con) + bri * con)) > 1e-3


# ---- export of the edited cloud ------------------------------------------------------------------------------------------------
def emu_ingest(table62, stride):
    t = np.ascontiguousarray(table62, dtype=F32)
    soa = np.zeros((15, stride, 4), dtype=F32)
    assert cref.emu().emu_ply_to_soa(C.c_void_p(t.ctypes.data), 62, t.shape[0], C.c_float(0.0), C.c_void_p(soa.ctypes.data), stride, 0) == 0
    return soa


def test_kept_table_round_trip():
    table = synthetic_ply_table(N, 22)
    store = emu_ingest(table, STRIDE)
    rng = np.random.default_rng(6)
    hidden = rng.random(N) < 0.25
    sel = (rng.random(N) < 0.7) & ~hidden
    e = color_edit(gain=(1.3, 0.7, 1.0), saturation=1.5, hue=20.0, brightness=0.03, view_dependence=0.5, opacity=3.0, opacity_offset=-0.9)
    edited = cref.emu_recolor(store, 4, False, pack_mask(sel, N), cref.constants(e))
    keep = np.flatnonzero(~hidden)
    o = edited[2, keep, 2]
    assert (o == 0.0).any() and (o == 1.0).any(), "opacities clamped to exactly 0 and 1 are exported"
    out = store_to_table(edited, N, 4, False, hidden)
    again = emu_ingest(out, STRIDE)
    a, b = edited[:, keep], again[:, :keep.size]
    np.testing.assert_array_equal(b[3:].view(U32), a[3:].view(U32))     # DC and SH
    o, back = a[2, :, 2], b[2, :, 2]
    np.testing.assert_array_equal(back[(o == 0.0) | (o == 1.0)], o[(o == 0.0) | (o == 1.0)])   # the clamped ones exactly
    # the rest within 2 ulp: the float32 logit's rounding moves a small opacity by up to 2 of its ulps (1 for the unedited ingest)
    assert (np.abs(back.astype(np.float64) - o) <= 2.0 * np.spacing(o)).all()
