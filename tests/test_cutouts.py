"""Cutout frames (include/gsr.h gsr_set_cutouts) without a GPU: the inside test on hand-placed positions, the rule's semantics, the
emulated CUT projection kernels bit for bit against the composed reference (tests/cutout_reference), and the Python conversion of a
Godot transform into to_local."""
import numpy as np
import pytest

from godotgaussiansplatting_b200.rasterizer import cutout_to_local
from oracle import oracle as orc
from tests import cutout_reference as cr
from tests import depth_order_reference as dor
from tests import instance_reference as iref
from tests import ortho_reference as oref
from tests.test_depth_order import H, W, instances, scene
from tests.test_instances import rigid, rotation
from tests.test_orthographic import store_of
from tests.test_sh_degree import zero_splat_coeffs

F32, U32 = np.float32, np.uint32
IDENT = np.concatenate([np.eye(3), np.zeros((3, 1))], axis=1)


def bits(a):
    return np.ascontiguousarray(a).view(U32)


def uni(ub):
    return orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8))


def nxt(x, toward):
    return np.nextafter(F32(x), F32(toward))


# ---- the inside test ---------------------------------------------------------------------------------------------------------
def test_box_faces_are_inside():
    c12 = cr.volume(IDENT)[0]
    p = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, -1], [1, 1, 1], [-1, -1, -1], [nxt(1, 2), 0, 0], [0, nxt(-1, -2), 0], [0, 0, nxt(1, 2)],
                  [nxt(1, 0), nxt(-1, 0), 0]], dtype=F32)
    np.testing.assert_array_equal(cr.inside(c12, cr.BOX, p), [True, True, True, True, True, False, False, False, True])
    # a scaled, shifted box: u = p / 4 - 0.5 is exact, so its faces are at p = -2 and p = 6
    c12 = cr.volume(np.concatenate([np.eye(3) * 0.25, np.full((3, 1), -0.5)], axis=1))[0]
    p = np.array([[-2, 0, 0], [6, 6, 6], [nxt(nxt(-2, -3), -3), 0, 0], [0, nxt(6, 7), 0]], dtype=F32)   # (one float below -2 rounds to -1)
    np.testing.assert_array_equal(cr.inside(c12, cr.BOX, p), [True, True, False, False])


def test_ellipsoid_surface():
    c12 = cr.volume(IDENT)[0]
    p = np.array([[1, 0, 0], [0, -1, 0], [0, 0, 1], [0.5, 0.5, 0.5], [nxt(1, 2), 0, 0], [0.75, 0.75, 0], [0.6, 0.6, 0.5]], dtype=F32)
    np.testing.assert_array_equal(cr.inside(c12, cr.ELLIPSOID, p), [True, True, True, True, False, False, True])
    u = p.astype(np.float64)   # exact squares here: the float32 sum is the float64 one
    np.testing.assert_array_equal(cr.inside(c12, cr.ELLIPSOID, p)[:6], ((u * u).sum(1) <= 1.0)[:6])


def test_nan_is_outside_and_negative_zero_is_zero():
    c12 = cr.volume(IDENT)[0]
    p = np.array([[np.nan, 0, 0], [0, np.nan, 0], [0, 0, np.nan], [-0.0, -0.0, -0.0], [-0.0, 1, -1]], dtype=F32)
    for shape in (cr.BOX, cr.ELLIPSOID):
        np.testing.assert_array_equal(cr.inside(c12, shape, p), [False, False, False, True, shape == cr.BOX])
    # NaN outside every volume: a REMOVE set keeps it, a KEEP set drops it
    rm = [cr.volume(IDENT, cr.BOX, cr.REMOVE)]
    kp = [cr.volume(IDENT, cr.BOX, cr.KEEP)]
    assert cr.drawn_mask(rm, p[:1], p[:1])[0] and not cr.drawn_mask(kp, p[:1], p[:1])[0]


def test_singular_to_local_is_a_slab():
    slab = np.zeros((3, 4))
    slab[2, 2], slab[2, 3] = 0.5, -1.0   # u = (0, 0, z / 2 - 1): every x, y with z in [0, 4]
    c12 = cr.volume(slab)[0]
    p = np.array([[1e30, -1e30, 0], [5, 5, 4], [0, 0, nxt(4, 5)], [0, 0, -1], [np.inf, 0, 2]], dtype=F32)
    np.testing.assert_array_equal(cr.inside(c12, cr.BOX, p), [True, True, False, False, False])   # inf * 0 is NaN


# ---- the rule --------------------------------------------------------------------------------------------------------------------
def grid_positions():
    g = np.linspace(-2, 2, 21, dtype=F32)
    return np.stack(np.meshgrid(g, g, g, indexing="ij"), axis=-1).reshape(-1, 3)


def test_rule_semantics():
    p = grid_positions()
    a = cr.box([0, 0, 0], 1.0)
    b = cr.box([1, 0, 0], 1.0, cr.ELLIPSOID)
    r = cr.box([0.5, 0, 0], 0.5, cr.BOX, cr.REMOVE)
    in_a, in_b, in_r = (cr.inside(v[0], v[1], p) for v in (a, b, r))
    assert in_a.sum() and in_b.sum() and in_r.sum() and (in_a & in_b).sum() and (in_a & ~in_b).sum()
    np.testing.assert_array_equal(cr.drawn_mask([], p, p), np.ones(len(p), bool))            # no set: everything
    np.testing.assert_array_equal(cr.drawn_mask([a], p, p), in_a)                              # KEEP only
    np.testing.assert_array_equal(cr.drawn_mask([r], p, p), ~in_r)                             # REMOVE only
    np.testing.assert_array_equal(cr.drawn_mask([a, b], p, p), in_a | in_b)                    # overlapping KEEP volumes: the union
    np.testing.assert_array_equal(cr.drawn_mask([a, b, r], p, p), (in_a | in_b) & ~in_r)      # both
    r2 = cr.box([0.5, 0, 0], 0.75, cr.ELLIPSOID, cr.REMOVE)
    vols = [a, r, b, r2]
    want = cr.drawn_mask(vols, p, p)
    for perm in ([3, 2, 1, 0], [1, 3, 0, 2], [2, 0, 3, 1]):
        np.testing.assert_array_equal(cr.drawn_mask([vols[i] for i in perm], p, p), want)
    # SOURCE volumes test sp, FRAME volumes the frame-space position
    shifted = p + F32(10)
    np.testing.assert_array_equal(cr.drawn_mask([cr.box([0, 0, 0], 1.0, space=cr.SOURCE)], p, shifted), in_a)
    assert not cr.drawn_mask([cr.box([0, 0, 0], 1.0, space=cr.FRAME)], p, shifted).any()


# ---- the emulated kernels --------------------------------------------------------------------------------------------------------
def crop_set(splat60, kind, fp=None, seed=0):
    """Volumes around the cloud that cut a real share of it.  fp: frame-space positions for FRAME volumes (default: the splats')."""
    sp = np.asarray(splat60, dtype=F32)[:, 0:3]
    fp = sp if fp is None else fp[np.isfinite(fp).all(1)]
    rng = np.random.default_rng(seed)

    def vol(pts, frac, shape, action, space, rot=0.4):
        c = np.median(pts, axis=0) + rng.normal(scale=0.1, size=3) * pts.std(0)
        h = np.median(np.abs(pts - c), axis=0) * frac + 1e-3   # (the clouds have long tails: a spread of the bulk)
        R = rotation(rng.normal(size=3), rng.uniform(-rot, rot))
        A = np.diag(1.0 / h) @ R.T
        return cr.volume(np.concatenate([A, (-A @ c)[:, None]], axis=1), shape, action, space)

    if kind == "keep_box":
        return [vol(fp, 2.0, cr.BOX, cr.KEEP, cr.FRAME)]
    if kind == "remove_ellipsoid":
        return [vol(fp, 1.5, cr.ELLIPSOID, cr.REMOVE, cr.FRAME)]
    if kind == "source":
        return [vol(sp, 2.5, cr.BOX, cr.KEEP, cr.SOURCE), vol(sp, 0.8, cr.ELLIPSOID, cr.REMOVE, cr.SOURCE)]
    # mixed: two KEEP volumes, two REMOVE volumes in both spaces
    return [vol(fp, 2.5, cr.BOX, cr.KEEP, cr.FRAME), vol(sp, 0.8, cr.ELLIPSOID, cr.REMOVE, cr.SOURCE),
            vol(fp, 2.0, cr.ELLIPSOID, cr.KEEP, cr.FRAME), vol(fp, 0.6, cr.BOX, cr.REMOVE, cr.FRAME)]


def check(got, ref, vp, depth=False):
    recs, keys, vals, words, m, vis, last, ovf = got
    assert (m, vis, last) == (ref["m"], ref["visible"], ref["last_tile"])
    assert ovf == ref["overflow"]
    np.testing.assert_array_equal(keys, ref["unsorted_keys"])
    np.testing.assert_array_equal(vals, ref["unsorted_values"])
    ids = np.unique(ref["unsorted_values"])
    np.testing.assert_array_equal(bits(recs[ids].view(F32)), bits(ref["records"][ids].view(F32)))
    assert ref["mask"][ids].all()
    if depth:
        np.testing.assert_array_equal(words, dor.ord_words(dor.view_depth(ref["records"], ref["unsorted_values"], vp)))


def emu(splat60, bands, vp, ub, bulk_min, vols, v=0.0, ortho=False, inst=None, capacity=None, depth=False):
    ranges = xf = None
    if inst is not None:
        ranges = [(f, c) for f, c, _ in inst]
        xf = [iref.inverse(x) for _, _, x in inst]
    return cr.emu_project(store_of(splat60, bands), bands, vp, ub, bulk_min, splat60.shape[0], vols, v, ortho, ranges, xf, capacity,
                          depth)


def frame_positions(splat60, ub, inst):
    return cr.positions(splat60, uni(ub).model_scale, inst)[1]


def assert_cuts(ref, uncut_visible):
    """The set removed a real share of the visible splats, and not all of them."""
    assert 0.05 * uncut_visible < ref["visible"] < 0.95 * uncut_visible, (ref["visible"], uncut_visible)


@pytest.mark.parametrize("time", [10.0, 0.6], ids=["static", "load_in"])
@pytest.mark.parametrize("instanced", [False, True], ids=["default", "instances"])
@pytest.mark.parametrize("bands", [1, 2, 3, 4])
def test_emulated_projection_is_the_reference(bands, instanced, time):
    splat60, vp, ub = scene(time)
    padded = zero_splat_coeffs(splat60, bands)
    inst = instances() if instanced else None
    vols = crop_set(splat60, "mixed", frame_positions(splat60, ub, inst), seed=bands)
    ref = cr.oracle_frame(padded, vp, ub, vols, inst=inst)
    assert_cuts(ref, dor.project(padded, vp, uni(ub), inst=inst).visible)
    for bulk_min in (1, 33):
        check(emu(padded, bands, vp, ub, bulk_min, vols, inst=inst), ref, vp)


@pytest.mark.parametrize("instanced", [False, True], ids=["default", "instances"])
@pytest.mark.parametrize("mode", ["aa_0.3", "ortho", "ortho_aa_0.1"])
def test_emulated_orthographic_and_antialiased(mode, instanced):
    splat60, vp, ub = scene(seed=13)
    ortho = mode.startswith("ortho")
    v = {"aa_0.3": 0.3, "ortho_aa_0.1": 0.1}.get(mode, 0.0)
    if ortho:
        vp, _ = oref.ortho_camera(W, H, size=2.5, near=0.5, far=4.5, frame=5)
    inst = instances() if instanced else None
    for kind in ("keep_box", "remove_ellipsoid"):
        vols = crop_set(splat60, kind, frame_positions(splat60, ub, inst), seed=7)
        ref = cr.oracle_frame(splat60, vp, ub, vols, v, ortho, inst=inst)
        assert_cuts(ref, dor.project(splat60, vp, uni(ub), v, ortho, inst).visible)
        for bulk_min in (1, 33):
            check(emu(splat60, 4, vp, ub, bulk_min, vols, v, ortho, inst), ref, vp)


@pytest.mark.parametrize("space", [cr.FRAME, cr.SOURCE], ids=["frame", "source"])
def test_emulated_instances_cut_one_copy_of_a_source_splat(space):
    """Two instances draw the same source range; a FRAME volume around the first copy cuts splats of that copy only, a SOURCE volume
    cuts the same source splats in both copies."""
    splat60, vp, ub = scene(seed=21)
    inst = [(0, 1000, rigid(4, 0.3, 0.1)), (0, 1000, rigid(9, 0.3, 0.8))]
    sp, fp = cr.positions(splat60, 1.0, inst)
    w0, _ = iref.layout([(f, c) for f, c, _ in inst])
    first_copy = fp[:1000]
    pts = first_copy if space == cr.FRAME else sp[:1000]
    c, h = np.median(pts, axis=0), pts.std(0) * 0.8
    vols = [cr.box(c, h, cr.BOX, cr.REMOVE, space)]
    ref = cr.oracle_frame(splat60, vp, ub, vols, inst=inst)
    m0, m1 = ref["mask"][32 * w0[0]:32 * w0[0] + 1000], ref["mask"][32 * w0[1]:32 * w0[1] + 1000]
    if space == cr.FRAME:
        drawn = set(ref["unsorted_values"].tolist())
        one_cut = [j for j in range(1000) if not m0[j] and m1[j] and 32 * w0[1] + j in drawn]
        assert len(one_cut) > 20   # source splats whose first copy is cut and whose second copy is drawn
    else:
        np.testing.assert_array_equal(m0, m1)
        assert 100 < (~m0).sum() < 900
    for bulk_min in (1, 33):
        check(emu(splat60, 4, vp, ub, bulk_min, vols, inst=inst), ref, vp)


def test_emulated_truncated_frame_is_the_filtered_prefix():
    splat60, vp, ub = scene(seed=17)
    vols = crop_set(splat60, "remove_ellipsoid", seed=3)
    m = cr.oracle_frame(splat60, vp, ub, vols)["m"]
    cap = m // 2 + 7
    ref = cr.oracle_frame(splat60, vp, ub, vols, cap=cap)
    got = emu(splat60, 4, vp, ub, 12, vols, capacity=cap)
    check(got, ref, vp)
    assert got[7] == 1 and len(got[1]) == cap


@pytest.mark.parametrize("instanced", [False, True], ids=["default", "instances"])
def test_emulated_depth_order_words(instanced):
    splat60, vp, ub = scene(seed=19)
    inst = instances() if instanced else None
    vols = crop_set(splat60, "mixed", frame_positions(splat60, ub, inst), seed=5)
    ref = cr.oracle_frame(splat60, vp, ub, vols, inst=inst, depth_order=True)
    for bulk_min in (1, 33):
        check(emu(splat60, 4, vp, ub, bulk_min, vols, inst=inst, depth=True), ref, vp, depth=True)


def test_emulated_hand_placed_splats_on_the_faces():
    """Splats exactly on a box's faces, one float beyond, at -0 and NaN: the kernel decides as the reference predicate."""
    splat60, vp, ub = scene(seed=23, n=256)
    s = splat60.copy()
    face = [1.0, -1.0, nxt(1, 2), nxt(-1, -2), nxt(1, 0), -0.0, 0.0, np.nan]
    for i in range(256):
        s[i, 0:3] = [face[i % 8] if i % 3 == 0 else 0.25, face[(i // 8) % 8] if i % 3 == 1 else -0.25, face[(i // 3) % 8] * 0.5]
    s[:, 4] = s[:, 7] = s[:, 9] = 1e-3
    s[:, 5] = s[:, 6] = s[:, 8] = 0.0
    s[:, 10] = 0.9
    for shape in (cr.BOX, cr.ELLIPSOID):
        for action in (cr.KEEP, cr.REMOVE):
            vols = [cr.volume(np.concatenate([np.diag([1.0, 1.0, 2.0]), np.zeros((3, 1))], axis=1), shape, action)]
            ref = cr.oracle_frame(s, vp, ub, vols)
            nan_ok = np.isfinite(s[:, 0:3]).all(1)
            vis = dor.project(s, vp, uni(ub)).values
            assert len(np.unique(vis)) > 40 and (~nan_ok).sum() > 0
            check(emu(s, 4, vp, ub, 12, vols), ref, vp)


def test_keep_box_around_everything_is_the_default_kernel():
    splat60, vp, ub = scene(seed=25)
    for inst in (None, instances()):
        ranges = None if inst is None else [(f, c) for f, c, _ in inst]
        xf = None if inst is None else [iref.inverse(x) for _, _, x in inst]
        store = store_of(splat60, 4)
        everything = [cr.volume(np.concatenate([np.eye(3) * 1e-6, np.zeros((3, 1))], axis=1))]   # |u| <= 1 for |p| <= 1e6
        sixteen = everything * 8 + [cr.box([1e9, 0, 0], 1.0, cr.ELLIPSOID, cr.REMOVE, cr.SOURCE)] * 8
        want = cr.emu_project(store, 4, vp, ub, 12, splat60.shape[0], None, ranges=ranges, xf=xf)
        for vols in (everything, sixteen):
            got = cr.emu_project(store, 4, vp, ub, 12, splat60.shape[0], vols, ranges=ranges, xf=xf)
            assert got[4:] == want[4:]
            for g, w in zip(got[1:3], want[1:3]):
                np.testing.assert_array_equal(g, w)
            np.testing.assert_array_equal(bits(got[0].view(F32)), bits(want[0].view(F32)))


# ---- the Python conversion -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("basis", ["identity", "y_up_flip", "rotated"])
def test_set_cutouts_conversion_maps_the_unit_cube(basis):
    bo = {"identity": np.eye(3), "y_up_flip": np.array([[1, 0, 0], [0, 0, 1], [0, -1, 0]]),
          "rotated": rotation([0.3, 1.0, -0.2], 0.7)}[basis]
    T = np.concatenate([rotation([1.0, 2.0, 0.5], 0.9) @ np.diag([2.0, 0.5, 3.0]), np.array([[4.0], [-1.0], [2.5]])], axis=1)
    to_local = cutout_to_local(T, bo).astype(np.float64)
    Fb = np.diag([-1.0, -1.0, 1.0]) @ np.asarray(bo, dtype=np.float64).T
    corners = np.array([[x, y, z] for x in (-1, 1) for y in (-1, 1) for z in (-1, 1)], dtype=np.float64)
    world = corners @ T[:, :3].T + T[:, 3]          # Godot positions of the unit cube's corners
    frame = world @ Fb.T                            # where they sit in frame space
    u = frame @ to_local[:, :3].T + to_local[:, 3]
    np.testing.assert_allclose(u, corners, rtol=0, atol=2e-6)
    assert cutout_to_local(T, bo).dtype == np.float32
    with pytest.raises(np.linalg.LinAlgError):
        cutout_to_local(np.zeros((3, 4)), bo)
