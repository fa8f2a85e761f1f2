"""Splat contribution (include/gsr.h gsr_set_splat_contribution) on the CPU: composite_contrib_kernel<CONTRACT> on the kernel emulator
against the contribution oracle, bit for bit, in both contraction modes, over several frames into one buffer with each frame's tiles
dealt to several persistent blocks; rgba and depth against the frames without the mode; the overflow rule; and the four
contribution properties of select_where_kernel and splat_histogram_kernel against their numpy restatement."""
import numpy as np
import pytest

from godotgaussiansplatting_b200.rasterizer import CONTRIBUTION_DTYPE, read_splat_contribution
from oracle import oracle as orc
from tests import contribution_reference as cref
from tests import depth_reference as dref
from tests import instance_appearance_reference as ar
from tests import instance_reference as iref
from tests.scenes import make_scene
from tests.test_splat_ids import instanced_scene, lower_half_plane, uni

F32, U32 = np.float32, np.uint32
CONTRACT = pytest.mark.parametrize("contract", [True, False], ids=["spec", "uncontracted"])


def bits(a):
    return np.ascontiguousarray(a).view(U32)


def run_frames(frames, slots, contract, ranges=None, ctas=3):
    """Every frame (records, values, bounds, W, H, vp, Z) through the emulated kernel and the oracle into one buffer each; rgba and
    depth of every emulated frame == the depth-compositing reference.  Returns the two buffers and the frame counter."""
    got, want = cref.zeros(slots), cref.zeros(slots)
    counter = np.zeros(1, dtype=U32)
    for e, (recs, vals, bnds, W, H, vp, Z) in enumerate(frames):
        rgba, depth, staged = cref.emu_composite_contrib(0 if contract else 1, got, recs, vals, bnds, W, H, vp, Z, ranges, epoch=e + 1,
                                                         ctas=ctas, frames=counter)
        d_rgba, d_depth, d_staged = dref.render_depth(recs, vals, bnds, W, H, vp, Z, 0.0, contract)
        np.testing.assert_array_equal(bits(rgba), bits(d_rgba))
        np.testing.assert_array_equal(bits(depth), bits(d_depth))
        assert staged == d_staged
        cref.accumulate(want, recs, vals, bnds, W, H, vp, Z, contract, ranges)
    cref.assert_same(got, want)
    assert int(counter[0]) == len(frames)
    return got, want


def orbit_frames(n, seed, w, h, frames, plane=False, **kw):
    out = []
    splat60 = None
    for f in frames:
        s, vp, ub = make_scene(n, seed, w, h, frame=f, **kw)
        splat60 = s if splat60 is None else splat60
        fr = orc.frame(splat60, vp, uni(ub), cap=40 * n)
        Z = lower_half_plane(fr.records, fr.values, vp, w, h) if plane else None
        out.append((fr.records, fr.values, fr.bounds, w, h, vp, Z))
    return out


@CONTRACT
@pytest.mark.parametrize("plane", ["none", "half"])
def test_kernel_is_the_oracle_over_an_orbit(plane, contract):
    n, w, h = 6000, 250, 130   # a ragged last tile column and row; tiles end in partial chunks
    frames = orbit_frames(n, 5, w, h, (30, 37, 44), plane == "half", scale_boost=0.5)
    got, _ = run_frames(frames, n, contract)
    c = read_splat_contribution(got)
    assert (c["pixels"] > 0).any() and (c["pixels"] == 0).any()
    assert (c["views"] == 3).any() and c["views"].max() <= 3
    # weight >= peak (one hit at least) wherever a splat was hit, and a hit has w > 0
    hit = c["pixels"] > 0
    assert (c["peak"][hit] > 0).all() and (c["peak"][~hit] == 0).all()
    assert (c["weight"][hit] + 2.0 ** -24 >= c["peak"][hit]).all()


@CONTRACT
def test_long_tiles_many_chunks(contract):
    n, w, h = 20000, 96, 64   # deep tiles: many 256-splat chunks and the tile-stop vote
    frames = orbit_frames(n, 3, w, h, (12, 20), scale_boost=1.0)
    run_frames(frames, n, contract, ctas=5)


@CONTRACT
def test_instances_drawing_one_source_range_twice(contract):
    splat60, vp, ub, ranges, cur = instanced_scene()
    u = uni(ub)
    W, H = u.dims[0], u.dims[1]
    xf = np.stack([iref.inverse(x) for x in cur])
    fr = iref.frame(splat60, vp, u, ranges, xf, depth=True, contract=contract)
    n = splat60.shape[0]
    got, _ = run_frames([(fr.proj.records, fr.values, fr.bounds, W, H, vp, None)], n, contract, ranges)
    # instances 0 and 2 draw [0, 3000): slots hit through both copies sum both copies' pixels, and count the frame once
    slot = cref.slot_of(ranges, len(fr.proj.records))
    w0, _ = iref.layout(ranges)
    c = read_splat_contribution(got)
    assert c["views"].max() == 1
    assert (c["pixels"][3000:5500] > 0).any() and (c["pixels"][5500:] == 0).all()
    vals = np.asarray(fr.values, dtype=U32)
    via0, via2 = slot[vals[vals < 32 * w0[1]]], slot[vals[vals >= 32 * w0[2]]]
    assert np.intersect1d(via0, via2).size > 0   # the oracle equality above covers the sum over both copies of those slots


@CONTRACT
def test_hidden_instance_and_draw_count(contract):
    splat60, vp, ub, ranges, cur = instanced_scene()
    u = uni(ub)
    W, H = u.dims[0], u.dims[1]
    inst = [(f, c, x) for (f, c), x in zip(ranges, cur)]
    draw = 1001
    app = [((1.0, 0.5, 2.0), 1.0, draw), ((1.0, 1.0, 1.0), 0.0, None), ar.DEFAULT]
    fr = ar.frame(splat60, vp, ub, inst, app, contract=contract, depth=True)
    n = splat60.shape[0]
    got, _ = run_frames([(fr["records"], fr["values"], fr["bounds"], W, H, vp, None)], n, contract, ranges)
    c = read_splat_contribution(got)
    assert (c["pixels"][3000:5500] == 0).all()   # the hidden instance's range is drawn by nobody else
    assert (c["pixels"][:3000] > 0).any()


def test_overflowed_frame_adds_nothing():
    n, w, h = 4000, 160, 120
    (recs, vals, bnds, W, H, vp, Z), = orbit_frames(n, 7, w, h, (25,), scale_boost=0.5)
    buf, counter = cref.zeros(n), np.zeros(1, dtype=U32)
    rgba, depth, _ = cref.emu_composite_contrib(0, buf, recs, vals, bnds, W, H, vp, Z, overflow=True, frames=counter)
    assert not buf.view(np.uint8).any() and counter[0] == 0
    d_rgba, d_depth, _ = dref.render_depth(recs, vals, bnds, W, H, vp, Z, 0.0, True)
    np.testing.assert_array_equal(bits(rgba), bits(d_rgba))
    # the same frame again (the re-render, same epoch) adds it once
    cref.emu_composite_contrib(0, buf, recs, vals, bnds, W, H, vp, Z, epoch=1, frames=counter)
    want = cref.accumulate(cref.zeros(n), recs, vals, bnds, W, H, vp, Z)
    cref.assert_same(buf, want)
    assert counter[0] == 1


# ---- the properties ------------------------------------------------------------------------------------------------------------
def property_setup(n=3000, m=3200, seed=3):
    rng = np.random.default_rng(seed)
    store = rng.normal(size=(15, m, 4)).astype(F32)
    store[0, n:, :3] = np.nan   # vacant slots
    buf = cref.zeros(m)
    buf["weight"] = rng.integers(0, 2 ** 34, size=m, dtype=np.uint64) * (rng.random(m) < 0.7)
    buf["pixels"] = rng.integers(0, 2 ** 26, size=m, dtype=np.uint64)
    buf["peak"] = rng.random(m).astype(F32) * (rng.random(m) < 0.8)
    buf["views"] = rng.integers(0, 400, size=m, dtype=np.uint32)
    buf["weight"][5] = (1 << 40) + 1   # needs the round to nearest
    return store, buf, rng


@pytest.mark.parametrize("half", [False, True])
def test_select_where_on_contribution(half):
    store, buf, rng = property_setup()
    m = store.shape[1]
    hidden = rng.random(m) < 0.1
    selected = rng.random(m) < 0.5
    w = read_splat_contribution(buf)["weight"]
    thr = float(np.quantile(w, 0.3))
    sets = [
        [(cref.CONTRIBUTION, -np.inf, thr, (0, 0, 0))],
        [(cref.PEAK, 0.1, 0.6, (0, 0, 0)), (cref.VIEWS, 10.0, 300.0, (0, 0, 0))],
        [(cref.PIXELS, 1e6, np.inf, (0, 0, 0)), (0, -np.inf, 0.5, (0, 0, 0)), (4, 0.0, 3.0, (0.5, 0.2, 0.1)), (1, -1.0, 5.0, (0, 0, 0))],
    ]
    for filters in sets:
        for op in range(4):
            want = cref.where_rule(store, half, hidden, selected, 0, 3000, filters, op, buf)
            got = cref.emu_where(store, half, hidden, selected, 0, 3000, filters, op, buf)
            np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("prop", cref.CONTRIB_PROPS)
def test_histogram_on_contribution(prop):
    store, buf, rng = property_setup()
    m = store.shape[1]
    hidden = rng.random(m) < 0.1
    v = cref.prop_values(store, False, prop, (0, 0, 0), buf)[:3000]
    edges = np.unique(np.quantile(v, np.linspace(0.05, 0.95, 17)).astype(F32))
    for hid in (None, hidden):
        want = cref.histogram_rule(store, False, hid, None, 0, 3000, prop, edges, buf)
        got = cref.emu_histogram(store, False, hid, 0, 3000, prop, edges, buf)
        np.testing.assert_array_equal(got[0], want[0])
        assert got[1] == want[1]


def test_read_splat_contribution():
    buf = cref.zeros(3)
    buf["weight"] = [0, 1 << 24, 3 << 23]
    buf["pixels"] = [0, 1, 2]
    buf["peak"] = [0.0, 1.0, 0.75]
    buf["views"] = [0, 1, 2]
    c = read_splat_contribution(buf.tobytes())
    np.testing.assert_array_equal(c["weight"], [0.0, 1.0, 1.5])
    np.testing.assert_array_equal(c["pixels"], [0, 1, 2])
    assert CONTRIBUTION_DTYPE.itemsize == 32
