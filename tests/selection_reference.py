"""Reference implementation of splat selection (include/gsr.h "Splat selection") for the tests.

TEST INFRASTRUCTURE.  Two parts, both in numpy float32 with the library's operations and order:
  1. the selection rules: the tested position q of every source splat, pix(M, q) of tests/motion_reference, the even-odd polygon test,
     the cutout shape test of tests/cutout_reference, the ID-plane mapping of rasterizer.splat_sources, the four ops and the invariant
     selected &= ~hidden;
  2. the frame with masks, composed from the unchanged references like tests/cutout_reference.oracle_frame: the projection of the frame's
     reference at unlimited capacity, every pair of a hidden (or cutout-removed) drawn id dropped, then the highlight c' = (c * k) + h
     applied to the colour words of the selected records, then the sort, the ranges and the compositor.
"""
from __future__ import annotations

import numpy as np

from oracle import oracle as orc
from tests import cutout_reference as cr
from tests import depth_order_reference as dor
from tests import depth_reference as dref
from tests import instance_reference as iref
from tests import motion_reference as mref

F32, U32 = np.float32, np.uint32
SET, ADD, SUBTRACT, TOGGLE = range(4)
DEFAULT_STYLE = ((1.0, 0.5, 0.0), 0.5)


# ---- masks -------------------------------------------------------------------------------------------------------------------
def combine(op, selected, inside, hidden):
    """One operation's result on bool arrays: op(selected, inside) & ~hidden."""
    if op == SET:
        r = inside.copy()
    elif op == ADD:
        r = selected | inside
    elif op == SUBTRACT:
        r = selected & ~inside
    else:
        r = selected ^ inside
    return r & ~hidden


def tested_positions(splat60, model_scale, n, instance=None):
    """(sp, q, in_range) over the n source splats: sp = position * model_scale; q = sp, or A sp + t of instance = (first, count, A12);
    in_range = the splats the operation tests."""
    s = np.ascontiguousarray(splat60, dtype=F32).reshape(-1, 60)
    sp = np.zeros((n, 3), dtype=F32)
    sp[:s.shape[0]] = s[:, 0:3] * F32(model_scale)   # splats past the upload are zero, like the store
    in_range = np.ones(n, dtype=bool)
    q = sp
    if instance is not None:
        first, count, A = instance
        in_range[:] = False
        in_range[first:first + count] = True
        A = np.asarray(A, dtype=F32).reshape(12)
        with np.errstate(all="ignore"):
            q = np.stack([((A[r] * sp[:, 0] + A[3 + r] * sp[:, 1]) + A[6 + r] * sp[:, 2]) + A[9 + r] for r in range(3)], axis=1).astype(F32)
    return sp, q, in_range


def polygon_inside(px, py, xy):
    """The even-odd rule of gsr_select_polygon, float32, one rounding per operation; NaN is outside."""
    xy = np.asarray(xy, dtype=F32).reshape(-1, 2)
    px, py = np.asarray(px, dtype=F32), np.asarray(py, dtype=F32)
    inside = np.zeros(px.shape, dtype=bool)
    n = xy.shape[0]
    with np.errstate(all="ignore"):
        for i in range(n):
            a, b = xy[i - 1], xy[i]   # the edge from the previous vertex (the last connects to the first)
            straddle = (a[1] > py) != (b[1] > py)
            x = (((b[0] - a[0]) * (py - a[1])) / (b[1] - a[1])) + a[0]
            inside ^= straddle & (px < x)
    return inside


def polygon_set(splat60, n, vp32, width, height, xy, model_scale=1.0, instance=None):
    """inside of gsr_select_polygon over the n source splats."""
    _, q, in_range = tested_positions(splat60, model_scale, n, instance)
    with np.errstate(all="ignore"):
        x, y, w = mref.pix(np.asarray(vp32, dtype=F32), q[:, 0], q[:, 1], q[:, 2], width, height)
    return in_range & (w > F32(0)) & polygon_inside(x, y, xy)


def volume_set(splat60, n, c12, shape, space, model_scale=1.0, instance=None):
    """inside of gsr_select_volume over the n source splats."""
    sp, q, in_range = tested_positions(splat60, model_scale, n, instance)
    return in_range & cr.inside(c12, shape, sp if space == cr.SOURCE else q)


def id_set(ids, n, rect, ranges=None):
    """inside of gsr_select_ids: the source splats of the (h, w, 2) ID plane's pixels in rect = (x0, y0, x1, y1)."""
    x0, y0, x1, y1 = rect
    v = np.asarray(ids, dtype=U32)[y0:y1, x0:x1, 0].reshape(-1)
    v = v[v != U32(0xFFFFFFFF)].astype(np.int64)
    inside = np.zeros(n, dtype=bool)
    if ranges:
        w0, D = iref.layout(ranges)
        for k, (first, count) in enumerate(ranges):
            j = v - 32 * w0[k]
            hit = (j >= 0) & (j < count)
            inside[first + j[hit]] = True
    else:
        inside[v[v < n]] = True
    return inside


def drawn_sources(n, ranges=None):
    """The source splat of every drawn id (-1 for padding ids)."""
    if not ranges:
        return np.arange(n, dtype=np.int64)
    w0, D = iref.layout(ranges)
    src = np.full(D, -1, dtype=np.int64)
    for k, (first, count) in enumerate(ranges):
        src[32 * w0[k] + np.arange(count)] = first + np.arange(count)
    return src


def highlight(style):
    """(k, h) of gsr_set_selection_style, float32 on the host."""
    rgb, s = style
    s = F32(s)
    return F32(1.0) - s, np.asarray(rgb, dtype=F32) * s, s > F32(0)


# ---- the frame ---------------------------------------------------------------------------------------------------------------
def oracle_frame(splat60, vp32, ub, hidden, selected, style=DEFAULT_STYLE, vols=(), inst=None, heat=0.0, contract=True, scene_depth=None,
                 depth=False, v=0.0, ortho=False):
    """A whole frame with masks in use.  hidden / selected: bool arrays over the source splats; inst = [(first, count, to_frame12)]."""
    u = orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8))
    W, H = u.dims[0], u.dims[1]
    pr = dor.project(splat60, vp32, u, v, ortho, inst)
    sp, fp = cr.positions(splat60, u.model_scale, inst)
    n = np.asarray(hidden).size
    src = drawn_sources(n, None if inst is None else [(f, c) for f, c, _ in inst])
    valid = src >= 0
    hid = np.zeros(src.size, dtype=bool)
    sel = np.zeros(src.size, dtype=bool)
    hid[valid] = np.asarray(hidden)[src[valid]]
    sel[valid] = np.asarray(selected)[src[valid]]
    mask = cr.drawn_mask(list(vols), sp, fp)[:src.size] & ~hid
    records = pr.records.copy()
    k, h, on = highlight(style)
    if on:
        c = records["color"][:src.size]
        for ch in range(3):
            c[sel, ch] = (c[sel, ch] * k) + h[ch]
        records["color"][:src.size] = c
    keep = mask[pr.values.astype(np.int64)]
    keys, values = pr.keys[keep].astype(U32), pr.values[keep].astype(U32)
    m, visible = int(keys.size), int(np.unique(values).size)
    last = int((keys >> U32(16)).max()) if m else -1
    kk, vals = orc.sort_pairs(keys, values)
    T = ((W + 15) // 16) * ((H + 15) // 16)
    b = orc.boundaries(kk, T, quirks=True)
    dep = None
    if depth or scene_depth is not None:
        rgba, dep, _ = dref.render_depth(records, vals, b, W, H, vp32, scene_depth, heat, contract)
    else:
        orc.set_blend_contraction(contract)
        try:
            rgba, _, _ = orc.render(records, vals, b, W, H, heat)
        finally:
            orc.set_blend_contraction(True)
    return dict(rgba=rgba, records=records, keys=kk, values=vals, bounds=b, visible=visible, m=m, last_tile=last, depth=dep, mask=mask)


def variant_frame(fr, hidden, selected, style=DEFAULT_STYLE):
    """A case of tests/variant_matrix (a vm.Frame) drawn with masks in use: the case's composed reference (vm.reference: cutouts,
    instances and their appearance, store, bands, anti-aliasing, orthographic) at unlimited capacity, every pair of a hidden drawn id
    dropped from its emission-order pairs, the highlight applied to the selected records' colour, then the case's sort (key or view
    depth), the ranges and the case's compositor (plain, depth, or depth + motion with the case's previous frame)."""
    from tests import variant_matrix as vm
    c = fr.case
    base = vm.reference(fr)
    ranges = [(f, k) for f, k, _ in fr.inst] if fr.inst else None
    src = drawn_sources(fr.n, ranges)
    valid = src >= 0
    hid = np.zeros(src.size, dtype=bool)
    sel = np.zeros(src.size, dtype=bool)
    hid[valid] = np.asarray(hidden)[src[valid]]
    sel[valid] = np.asarray(selected)[src[valid]]
    records = base["records"].copy()
    k, h, on = highlight(style)
    if on:
        col = records["color"][:src.size]
        for ch in range(3):
            col[sel, ch] = (col[sel, ch] * k) + h[ch]
        records["color"][:src.size] = col
    keep = ~hid[base["unsorted_values"].astype(np.int64)]
    keys, values = base["unsorted_keys"][keep].astype(U32), base["unsorted_values"][keep].astype(U32)
    m, visible = int(keys.size), int(np.unique(values).size)
    last = int((keys >> U32(16)).max()) if m else -1
    if c.dord:
        kk, vals, _ = dor.sort_by_depth(keys, values, dor.ord_words(dor.view_depth(records, values, fr.vp)))
    else:
        kk, vals = orc.sort_pairs(keys, values)
    T = ((fr.w + 15) // 16) * ((fr.h + 15) // 16)
    b = orc.boundaries(kk, T, quirks=True)
    heat = 1.0 if c.heat else 0.0
    dep = mo = None
    if c.compositor == "plain":
        orc.set_blend_contraction(c.contract)
        try:
            rgba, staged, _ = orc.render(records, vals, b, fr.w, fr.h, heat)
        finally:
            orc.set_blend_contraction(True)
    elif c.compositor == "depth":
        rgba, dep, staged = dref.render_depth(records, vals, b, fr.w, fr.h, fr.vp, fr.Z, heat, c.contract)
    else:
        prev_pos = None
        if c.inst:
            prev_pos = mref.instance_prev_positions(fr.src, ranges, [x for _, _, x in fr.prev_inst], 1.0, fr.drawn)
        mv = mref.splat_motion(records, fr.vp, fr.pvp, fr.w, fr.h, prev_pos)
        rgba, dep, mo, staged = mref.render_motion(records, vals, b, fr.w, fr.h, fr.vp, mv, fr.Z, heat, c.contract)
    return dict(rgba=rgba, records=records, keys=kk, values=vals, unsorted_values=values, bounds=b, visible=visible, m=m, last_tile=last,
                staged=staged, depth=dep, motion=mo, selected_ids=np.flatnonzero(sel), hidden_ids=np.flatnonzero(hid))
