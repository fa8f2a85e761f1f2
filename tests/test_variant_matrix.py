"""Every projection and compositor variant without a GPU: the 256 cases of tests/variant_matrix through the kernels compiled for the CPU
(tests/kernel_emu and the per-feature emulator libraries), bit for bit against the composed reference; the covering design of the table;
and the instantiations compiled into libgsr.so, which must be exactly the table's."""
import functools
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from tests import cutout_reference as cr
from tests import depth_order_reference as dor
from tests import depth_reference as dref
from tests import instance_appearance_reference as ar
from tests import motion_reference as mref
from tests import test_sh_half as shh
from tests import variant_matrix as vm
from tests.test_kernel_emu import SPEC, UNCONTRACTED, emu_composite
from tests.test_orthographic import store_of

N = 2048
SIZE, RAGGED = (128, 96), (121, 83)
F32 = np.float32
bits = vm.bits


@functools.lru_cache(maxsize=None)
def case_frame(case):
    fr = vm.frame_of(case, N, SIZE, RAGGED)
    return fr, vm.reference(fr)


def bulk_mins(i):
    """Both phase-2 paths forced on every seventh case (seven is odd: the subset takes every value of every axis), the library's
    threshold on the others."""
    return (1, 33) if i % 7 == 0 else (12,)


def emu_project(fr, bulk_min):
    """The case's projection_kernel on the CPU: (records, keys, values, depth words or None, M, V, last tile)."""
    c = fr.case
    ranges = xf = None
    if c.inst:
        ranges = [(f, k) for f, k, _ in fr.inst]
        xf = [vm.iref.inverse(x) for _, _, x in fr.inst]
    if c.half:
        return shh.emu_project(shh.store_of(fr.splat60, c.store_bands), c.bands, fr.vp, fr.ub, bulk_min, fr.n, c.v, c.ortho, fr.inst, fr.app,
                               fr.vols, c.dord)
    store = store_of(fr.splat60, c.store_bands)
    if c.inst and fr.app is not None:
        got = ar.emu_project(store, c.bands, fr.vp, fr.ub, bulk_min, fr.inst, fr.app, c.v, c.ortho, fr.vols, depth=c.dord)
    else:
        got = cr.emu_project(store, c.bands, fr.vp, fr.ub, bulk_min, fr.n, fr.vols, c.v, c.ortho, ranges, xf, depth=c.dord)
    assert got[7] == 0   # no overflow
    return got[:7]


@pytest.mark.parametrize("i", range(len(vm.CASES)), ids=vm.IDS)
def test_projection_kernel_is_the_reference(i):
    case = vm.CASES[i]
    fr, ref = case_frame(case)
    assert ref["m"] > 0 and ref["visible"] > 0
    ids = np.unique(ref["unsorted_values"])
    for bulk_min in bulk_mins(i):
        recs, keys, vals, words, m, vis, last = emu_project(fr, bulk_min)
        where = f"{case.id} bulk_min={bulk_min}"
        assert (m, vis, last) == (ref["m"], ref["visible"], ref["last_tile"]), where
        np.testing.assert_array_equal(keys, ref["unsorted_keys"], err_msg=where)
        np.testing.assert_array_equal(vals, ref["unsorted_values"], err_msg=where)
        for w in ("image_pos", "pos_xy", "conic", "pos_z", "color"):
            np.testing.assert_array_equal(bits(recs[w][ids]), bits(ref["records"][w][ids]), err_msg=f"{where}: record word {w}")
        assert (words is not None) == case.dord
        if case.dord:
            np.testing.assert_array_equal(words, dor.ord_words(dor.view_depth(ref["records"], ref["unsorted_values"], fr.vp)), err_msg=where)


@pytest.mark.parametrize("i", range(len(vm.CASES)), ids=vm.IDS)
def test_compositor_kernel_is_the_reference(i):
    case = vm.CASES[i]
    fr, ref = case_frame(case)
    heat = 1.0 if case.heat else 0.0
    variant = SPEC if case.contract else UNCONTRACTED
    args = (ref["records"], ref["values"], ref["bounds"], fr.w, fr.h)
    if case.compositor == "plain":
        rgba, staged, _ = emu_composite(variant, *args, heat)
    elif case.compositor == "depth":
        rgba, depth, staged = dref.emu_composite_depth(variant, *args, fr.vp, fr.Z, heat)
        np.testing.assert_array_equal(bits(depth), bits(ref["depth"]))
    else:
        inst = None
        if case.inst:
            inst = (fr.splat60, fr.n, [(f, k) for f, k, _ in fr.inst], np.stack([x for _, _, x in fr.prev_inst]), 1.0)
        rgba, depth, motion, staged = mref.emu_composite_motion(variant, *args, fr.vp, fr.pvp, fr.Z, heat, inst)
        np.testing.assert_array_equal(bits(depth), bits(ref["depth"]))
        np.testing.assert_array_equal(bits(motion), bits(ref["motion"]))
        assert np.abs(ref["motion"]).max() > 0
    np.testing.assert_array_equal(bits(rgba), bits(ref["rgba"]))
    assert staged == ref["staged"]


# ---- the table ---------------------------------------------------------------------------------------------------------------------
def test_one_case_per_projection_kernel_and_readable_ids():
    assert len(vm.CASES) == 256
    assert len({c.kernel for c in vm.CASES}) == 256
    assert len(set(vm.IDS)) == 256
    assert "inst-b2-ortho-aa-dord-cut-half" in vm.IDS and "flat-b4" in vm.IDS


def test_covering_design():
    """Every value of every setting meets every value of every projection axis in some case (where the setting can take it)."""
    assert vm.coverage_gaps() == []
    assert {c.compositor_kernel for c in vm.CASES} == {(k, d, m) for k in (True, False) for d, m in ((False, False), (True, False), (True, True))}
    aa = [c.v for c in vm.CASES if c.aa]
    assert set(aa) == {vm.AA_MOST, vm.AA_SOME} and aa.count(vm.AA_MOST) > aa.count(vm.AA_SOME)
    assert all(c.v == 0.0 for c in vm.CASES if not c.aa)
    # and the check sees a gap: drop one value from the cases that carry it
    thin = [c for c in vm.CASES if not (c.heat and c.half)]
    assert ("heat", True, "half", True) in vm.coverage_gaps(thin)


def test_fixtures():
    inst = vm.layout(N)
    first, count, _ = inst[2]
    assert first + count == N and first % 32                   # ends at max_splats, unaligned first
    assert inst[0][:2] == inst[3][:2]                          # a source range drawn twice
    A = inst[1][2][:9].astype(np.float64).reshape(3, 3)
    assert not np.allclose(A @ A.T, np.eye(3), atol=1e-3)      # not rigid
    app = vm.mixed_appearance(inst)
    assert any(max(t) > 1 for t, _, _ in app) and any(o == 0.5 for _, o, _ in app) and any(o == 0.0 for _, o, _ in app)
    assert any(d is not None and d % 32 for _, _, d in app)
    vols = vm.cutouts(vm.cloud(N), vm.cloud(N)[:, 0:3])
    assert {(v[1], v[2], v[3]) for v in vols} == {(cr.BOX, cr.KEEP, cr.FRAME), (cr.ELLIPSOID, cr.REMOVE, cr.SOURCE)}


# ---- the instantiations in libgsr.so -----------------------------------------------------------------------------------------------
def compiled_kernels():
    cuda_bin = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin")
    tools = [shutil.which(t) or os.path.join(cuda_bin, t) for t in ("cuobjdump", "cu++filt")]
    if not all(os.path.exists(t) for t in tools):
        pytest.skip("cuobjdump / cu++filt not available")
    from godotgaussiansplatting_b200 import build as gsr_build
    so = gsr_build.build()
    dump = subprocess.run([tools[0], "-res-usage", so], capture_output=True, text=True, check=True).stdout
    mangled = re.findall(r"Function (\S+?):", dump)
    assert mangled
    names = subprocess.run([tools[1]], input="\n".join(mangled), capture_output=True, text=True, check=True).stdout.splitlines()
    return names


def template_args(names, kernel):
    """The template argument tuples of every `kernel` instantiation: bools as bool, ints as int."""
    out = []
    for nm in names:
        m = re.search(r"::" + kernel + r"<([^>]*)>\(", nm)
        if m:
            args = []
            for a in m.group(1).split(","):
                t, v = re.fullmatch(r"\s*\((\w+)\)(-?\d+)\s*", a).groups()
                args.append(bool(int(v)) if t == "bool" else int(v))
            out.append(tuple(args))
    return out


def test_compiled_projection_and_compositor_kernels_are_the_table():
    names = compiled_kernels()
    proj = template_args(names, "projection_kernel")
    assert len(proj) == len(set(proj))
    assert set(proj) == {c.kernel for c in vm.CASES}
    defaults = [t for t in proj if not any(t[i] for i in (0, 2, 3, 4, 5, 6))]
    assert len(defaults) == 4 and len([t for t in proj if not any(t[i] for i in (2, 3, 4, 5, 6))]) == 8
    assert any("projection_sharded_kernel" in n for n in names) and any("projection_scatter_kernel" in n for n in names)
    comp = template_args(names, "composite_kernel")
    assert len(comp) == len(set(comp))
    assert set(comp) == {c.compositor_kernel for c in vm.CASES}
