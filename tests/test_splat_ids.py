"""Splat and instance IDs (include/gsr.h gsr_set_splat_ids) on the CPU: composite_ids_kernel<CONTRACT, MOTION> on the kernel
emulator against the ID oracle, bit for bit, in both contraction modes; rgba, depth and motion against the frames without IDs; the
tie and no-coverage rules on hand-made records; and the drawn-id -> source-splat map of GaussianSplattingRasterizer.splat_sources
against the instance reference's layout."""
import numpy as np
import pytest

from godotgaussiansplatting_b200 import _lib
from godotgaussiansplatting_b200.rasterizer import splat_sources
from oracle import oracle as orc
from tests import depth_order_reference as dor
from tests import depth_reference as dref
from tests import id_reference as idr
from tests import instance_appearance_reference as ar
from tests import instance_reference as iref
from tests import motion_reference as mref
from tests import ortho_reference as oref
from tests.scenes import make_scene

F32, U32 = np.float32, np.uint32
NO_ID = idr.NO_ID
CONTRACT = pytest.mark.parametrize("contract", [True, False], ids=["spec", "uncontracted"])


def bits(a):
    return np.ascontiguousarray(a).view(U32)


def uni(ub):
    return orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8))


def check_ids(records, values, bounds, W, H, vp, Z=None, heat=0.0, contract=True, ranges=None, motion=None):
    """Emulated kernel == oracle (rgba, depth, ids, staged); rgba and depth == the depth-compositing reference (the frame without IDs);
    an ID exactly where alpha > 0, k the instance of v's warp.  motion: None, or (prev_vp, per-record motion, instances of
    motion_reference.emu_composite_motion) -- then the motion output == the motion oracle's too.  Returns (ids, rgba)."""
    variant = 0 if contract else 1
    o_rgba, o_depth, o_ids, o_staged = idr.render_ids(records, values, bounds, W, H, vp, Z, heat, contract, ranges)
    e_rgba, e_depth, e_mo, e_ids, e_staged = idr.emu_composite_ids(variant, records, values, bounds, W, H, vp, Z, heat, ranges,
                                                                   None if motion is None else (motion[0], motion[2]))
    np.testing.assert_array_equal(e_ids, o_ids)
    np.testing.assert_array_equal(bits(e_rgba), bits(o_rgba))
    np.testing.assert_array_equal(bits(e_depth), bits(o_depth))
    assert e_staged == o_staged
    d_rgba, d_depth, d_staged = dref.render_depth(records, values, bounds, W, H, vp, Z, heat, contract)
    np.testing.assert_array_equal(bits(o_rgba), bits(d_rgba))
    np.testing.assert_array_equal(bits(o_depth), bits(d_depth))
    assert o_staged == d_staged
    if motion is not None:
        m_rgba, m_depth, m_mo, _ = mref.render_motion(records, values, bounds, W, H, vp, motion[1], Z, heat, contract)
        np.testing.assert_array_equal(bits(e_mo), bits(m_mo))
        np.testing.assert_array_equal(bits(e_rgba), bits(m_rgba))
    has = o_ids[..., 0] != NO_ID
    np.testing.assert_array_equal(has, o_rgba[..., 3] > 0)
    assert (o_ids[~has] == NO_ID).all()
    if ranges is None:
        assert (o_ids[..., 1] == NO_ID).all()
    else:
        np.testing.assert_array_equal(o_ids[has, 1], idr.warp_instances(ranges)[o_ids[has, 0] >> 5])
    assert np.isin(o_ids[has, 0], values).all()
    return o_ids, o_rgba


# ---- the depth tests' scenes, with an occluding scene depth --------------------------------------------------------------------
#                n     seed w    h    heat kwargs
CASES = {
    "ragged_heatmap": (6000, 5, 250, 130, 1.0, dict(frame=37, scale_boost=0.5)),
    "load_in": (5000, 7, 192, 160, 0.0, dict(time=0.6, scale_boost=1.0)),
    "tiny": (40, 9, 33, 17, 0.0, dict(scale_boost=-1.0)),
}


def lower_half_plane(records, values, vp, w, h):
    d = -(((vp[2] * records["pos_xy"][:, 0] + vp[6] * records["pos_xy"][:, 1]) + vp[10] * records["pos_z"]) + vp[14])
    Z = np.full((h, w), np.inf, dtype=F32)
    Z[h // 2:] = np.median(d[values])
    return Z


@CONTRACT
@pytest.mark.parametrize("plane", ["none", "half"])
@pytest.mark.parametrize("case", list(CASES))
def test_kernel_is_the_oracle(case, plane, contract):
    n, seed, w, h, heat, kw = CASES[case]
    splat60, vp, ub = make_scene(n, seed, w, h, **kw)
    fr = orc.frame(splat60, vp, uni(ub), heatmap=heat, cap=40 * n)
    Z = lower_half_plane(fr.records, fr.values, vp, w, h) if plane == "half" else None
    ids, _ = check_ids(fr.records, fr.values, fr.bounds, w, h, vp, Z, heat, contract)
    assert (ids[..., 0] != NO_ID).any()


@CONTRACT
def test_orthographic_frame(contract):
    n, w, h = 8000, 160, 120
    splat60 = make_scene(n, 4, w, h, scale_boost=0.5)[0]
    vp, ub = oref.ortho_camera(w, h, frame=30)
    fr = oref.oracle_frame(splat60, vp, ub, depth=True, contract=contract)
    ids, _ = check_ids(fr["records"], fr["values"], fr["bounds"], w, h, vp, contract=contract)
    assert (ids[..., 0] != NO_ID).sum() > w * h // 10


@CONTRACT
def test_view_depth_order(contract):
    n, w, h = 6000, 200, 150
    splat60, vp, ub = make_scene(n, 12, w, h, frame=44, scale_boost=0.5)
    fr = dor.oracle_frame(splat60, vp, ub, depth=True, contract=contract)
    check_ids(fr["records"], fr["values"], fr["bounds"], w, h, vp, contract=contract)


# ---- instances -----------------------------------------------------------------------------------------------------------------
def to_frame(t, ang=0.0):
    c, s = np.cos(ang), np.sin(ang)
    A = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]], dtype=np.float64)
    return np.concatenate([A.T.reshape(9), np.asarray(t, dtype=np.float64)]).astype(F32)


def instanced_scene(n=8000, w=200, h=150):
    """Three instances; the first and the last draw the same source range at two places that overlap on screen."""
    splat60, vp, ub = make_scene(n, 11, w, h, frame=20, scale_boost=0.5)
    ranges = [(0, 3000), (3000, 2500), (0, 3000)]
    cur = [to_frame((0.2, 0.0, 0.0)), to_frame((0.0, 0.1, 0.3), 0.1), to_frame((0.05, 0.02, 0.1), -0.05)]
    return splat60, vp, ub, ranges, cur


def source_positions_match(splat60, records, ids, ranges, cur, ms):
    """Every pixel's drawn record sits where its splat_sources splat lands under its instance's transform (the projection's own
    operations, bit for bit): the map is the layout the projection used."""
    has = ids[..., 0] != NO_ID
    v, k = ids[has, 0].astype(np.int64), ids[has, 1]
    s = splat_sources(ids, ranges)[has].astype(np.int64)
    np.testing.assert_array_equal(s, idr.sources(ids, ranges)[has])
    for kk in np.unique(k):
        sel = k == kk
        first, count = ranges[kk]
        assert ((s[sel] >= first) & (s[sel] < first + count)).all()
        xf = np.concatenate([np.asarray(cur[kk], dtype=F32), np.zeros(12, dtype=F32)])
        p = iref.frame_position(xf, splat60[s[sel], 0:3] * F32(ms))
        np.testing.assert_array_equal(bits(p[:, 0]), bits(records["pos_xy"][v[sel], 0]))
        np.testing.assert_array_equal(bits(p[:, 1]), bits(records["pos_xy"][v[sel], 1]))
        np.testing.assert_array_equal(bits(p[:, 2]), bits(records["pos_z"][v[sel]]))


@CONTRACT
def test_instances_drawing_one_source_range_twice(contract):
    splat60, vp, ub, ranges, cur = instanced_scene()
    u = uni(ub)
    W, H = u.dims[0], u.dims[1]
    xf = np.stack([iref.inverse(x) for x in cur])
    fr = iref.frame(splat60, vp, u, ranges, xf, depth=True, contract=contract)
    ids, _ = check_ids(fr.proj.records, fr.values, fr.bounds, W, H, vp, contract=contract, ranges=ranges)
    has = ids[..., 0] != NO_ID
    ks = ids[has, 1]
    assert set(np.unique(ks)) == {0, 1, 2}
    # one source splat owns pixels as instance 0 and as instance 2: same source, different drawn ids and instances
    src = splat_sources(ids, ranges)[has]
    both = np.intersect1d(src[ks == 0], src[ks == 2])
    assert both.size > 0
    s = both[0]
    v0, v2 = ids[has][(src == s) & (ks == 0), 0], ids[has][(src == s) & (ks == 2), 0]
    assert np.unique(v0).size == 1 and np.unique(v2).size == 1 and v0[0] != v2[0]
    source_positions_match(splat60, fr.proj.records, ids, ranges, cur, u.model_scale)


@CONTRACT
def test_hidden_instance_and_draw_count(contract):
    splat60, vp, ub, ranges, cur = instanced_scene()
    u = uni(ub)
    W, H = u.dims[0], u.dims[1]
    inst = [(f, c, x) for (f, c), x in zip(ranges, cur)]
    draw = 1001   # a prefix that ends inside a warp
    app = [((1.0, 0.5, 2.0), 1.0, draw), ((1.0, 1.0, 1.0), 0.0, None), ar.DEFAULT]   # a prefix, hidden, the default
    fr = ar.frame(splat60, vp, ub, inst, app, contract=contract, depth=True)
    ids, _ = check_ids(fr["records"], fr["values"], fr["bounds"], W, H, vp, contract=contract, ranges=ranges)
    has = ids[..., 0] != NO_ID
    ks = ids[has, 1]
    assert 1 not in set(np.unique(ks))                    # the hidden instance owns no pixel
    assert {0, 2} <= set(np.unique(ks))
    src = splat_sources(ids, ranges)[has]
    assert (src[ks == 0] < ranges[0][0] + draw).all()       # nor does a splat past the draw count
    assert (src[ks == 2] >= draw).any()                     # (which the default instance of the same range draws)


# ---- motion and IDs together ---------------------------------------------------------------------------------------------------
@CONTRACT
def test_motion_and_ids(contract):
    n, w, h = 9000, 250, 130
    splat60, vp, ub = make_scene(n, 5, w, h, frame=37, scale_boost=0.5)
    pvp = make_scene(16, 5, w, h, frame=35)[1]
    fr = orc.frame(splat60, vp, uni(ub), cap=1000 * n)
    m = mref.splat_motion(fr.records, vp, pvp, w, h)
    Z = lower_half_plane(fr.records, fr.values, vp, w, h)
    check_ids(fr.records, fr.values, fr.bounds, w, h, vp, Z, contract=contract, motion=(pvp, m, None))


@CONTRACT
def test_motion_and_ids_with_moving_instances(contract):
    splat60, vp, ub, ranges, cur = instanced_scene()
    u = uni(ub)
    W, H = u.dims[0], u.dims[1]
    pvp = make_scene(16, 11, W, H, frame=19)[1]
    prev = [to_frame((0.25, -0.02, 0.0)), cur[1].copy(), to_frame((0.0, 0.0, 0.1), -0.1)]
    xf = np.stack([iref.inverse(x) for x in cur])
    fr = iref.frame(splat60, vp, u, ranges, xf, depth=True, contract=contract)
    pp = mref.instance_prev_positions(splat60, ranges, prev, u.model_scale, fr.proj.drawn)
    m = mref.splat_motion(fr.proj.records, vp, pvp, W, H, pp)
    check_ids(fr.proj.records, fr.values, fr.bounds, W, H, vp, contract=contract, ranges=ranges,
              motion=(pvp, m, (splat60, splat60.shape[0], ranges, np.stack(prev), u.model_scale)))


# ---- the rules on hand-made records --------------------------------------------------------------------------------------------
def hand_made(opacities_per_tile, W=32, H=32):
    """Records centred on pixel (5 + 16 tx, 7 + 16 ty) of tile (tx, ty), the given opacities in sorted order per tile; the other
    tiles are empty.  At the centre alpha is exactly the opacity (power 0)."""
    tiles_x = (W + 15) // 16
    T = tiles_x * ((H + 15) // 16)
    recs, vals, bounds, n = [], [], np.zeros((T, 2), dtype=U32), 0
    for tile, ops in opacities_per_tile.items():
        tx, ty = tile % tiles_x, tile // tiles_x
        bounds[tile] = (n, n + len(ops))
        for op in ops:
            r = np.zeros(1, dtype=orc.RECORD_DTYPE)
            r["image_pos"] = (5 + 16 * tx, 7 + 16 * ty)
            r["conic"] = (2.0, 0.0, 2.0)
            r["color"] = (1.0, 0.5, 0.25, op)
            recs.append(r)
            vals.append(n)
            n += 1
    empty = bounds[:, 0] == bounds[:, 1]
    bounds[empty] = n
    return np.concatenate(recs), np.array(vals, dtype=U32), bounds


@CONTRACT
def test_exact_tie_replacement_and_uncovered_pixels(contract):
    W = H = 32
    vp = make_scene(16, 1, W, H)[1]
    # tile 0: alpha 0.5 then 1.0 -> w = 0.5 and 0.5, the first wins; tile 1: 0.25 then 0.5 -> w = 0.25 then 0.375, the second wins;
    # tile 2: 1.0 then 0.5 -> the second is never blended; tile 3: nothing
    recs, vals, bounds = hand_made({0: [0.5, 1.0], 1: [0.25, 0.5], 2: [1.0, 0.5]}, W, H)
    ids, rgba = check_ids(recs, vals, bounds, W, H, vp, contract=contract)
    assert tuple(ids[7, 5]) == (0, NO_ID)
    assert tuple(ids[7, 21]) == (3, NO_ID)
    assert tuple(ids[23, 5]) == (4, NO_ID)
    assert rgba[7, 5, 3] == 1.0
    assert (ids[16:, 16:] == NO_ID).all() and (rgba[16:, 16:, 3] == 0).all()   # the empty tile
    assert (ids[0, :] == NO_ID).all() and (rgba[0, :, 3] == 0).all()           # far from every splat: alpha rounds away
    assert (ids[8, 5, 0] != NO_ID) and (ids[7, 6, 0] != NO_ID)                 # the neighbours are covered


def test_splat_sources_without_instances_and_no_id():
    ids = np.array([[[7, NO_ID], [NO_ID, NO_ID]], [[123456, NO_ID], [0, NO_ID]]], dtype=U32)
    np.testing.assert_array_equal(splat_sources(ids), [[7, NO_ID], [123456, 0]])
    assert splat_sources(ids).dtype == U32
    assert _lib.GSR_NO_ID == NO_ID


def test_splat_sources_follow_the_instance_layout():
    ranges = [(100, 40), (0, 33), (7, 1), (500, 64)]
    w0, D = iref.layout(ranges)
    v = np.arange(D, dtype=U32)
    wi = idr.warp_instances(ranges)[v >> 5]
    live = np.zeros(D, dtype=bool)
    for k, (f, c) in enumerate(ranges):
        live[32 * w0[k]:32 * w0[k] + c] = True
    ids = np.stack([v[live], wi[live]], axis=-1)[None]
    src = splat_sources(ids, ranges)[0]
    expect = np.concatenate([np.arange(f, f + c) for f, c in ranges])
    np.testing.assert_array_equal(src, expect)
    np.testing.assert_array_equal(src, idr.sources(ids, ranges)[0])
