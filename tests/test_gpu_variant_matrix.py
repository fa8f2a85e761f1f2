"""Every projection and compositor variant on the GPU: the 256 cases of tests/variant_matrix through the C-ABI (the dispatch and frame
arguments of gsr_api.cu, the real TMA / mbarrier byte counts and the compiled SASS of each instantiation), bit for bit against the
composed reference in RGBA, M, V, overflow, last tile, sorted keys and values, tile bounds, the records of every emitted id, the depth
output and the motion output (the latter computed from the reference's records)."""
import ctypes as C

import numpy as np
import pytest

from godotgaussiansplatting_b200 import _lib
from godotgaussiansplatting_b200.rasterizer import pack_instance_appearance
from tests import variant_matrix as vm
from tests.gsr_direct import REC_DTYPE
from tests.test_gpu_sh_degree import ShCtx, set_instances

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

N = 10240
SIZE, RAGGED = (320, 192), (321, 181)
bits = vm.bits


def flags_of(case):
    return ((_lib.GSR_FLAG_ORTHOGRAPHIC if case.ortho else 0) | (_lib.GSR_FLAG_SH_HALF if case.half else 0) |
            (0 if case.contract else _lib.GSR_FLAG_UNCONTRACTED_BLEND))


def set_cutouts(c, vols):
    arr = (_lib.GsrCutout * len(vols))()
    for k, (c12, shape, action, space) in enumerate(vols):
        arr[k].to_local[:] = [float(v) for v in np.asarray(c12, dtype=np.float32)]
        arr[k].shape, arr[k].action, arr[k].space = int(shape), int(action), int(space)
    _lib.check(c.L.gsr_set_cutouts(c.h, arr, len(vols)), "gsr_set_cutouts")


def render_case(fr):
    """Draw the case through the C-ABI.  Returns (rgba, depth or None, motion or None, stats, keys, values, bounds, records)."""
    case = fr.case
    L = _lib.lib()
    heat = 1.0 if case.heat else 0.0
    with ShCtx(fr.n, fr.w, fr.h, case.store_bands, flags_of(case), factor=16) as c:
        c.upload(fr.splat60)
        if case.store_bands != case.bands:
            _lib.check(c.degree(case.bands - 1), "gsr_set_sh_degree")
        if case.aa:
            _lib.check(L.gsr_set_antialiasing(c.h, C.c_float(case.v)), "gsr_set_antialiasing")
        if case.dord:
            _lib.check(L.gsr_set_depth_order(c.h, _lib.GSR_DEPTH_ORDER_VIEW_DEPTH), "gsr_set_depth_order")
        if case.cut:
            set_cutouts(c, fr.vols)
        if case.inst:
            set_instances(c, fr.prev_inst if fr.prev_inst is not None else fr.inst)
            if fr.app is not None:
                app = pack_instance_appearance(fr.app)
                _lib.check(L.gsr_set_instance_appearance(c.h, app, len(app)), "gsr_set_instance_appearance")
        depth = motion = None
        if case.compositor != "plain":
            Zt = None if fr.Z is None else torch.from_numpy(fr.Z).cuda()
            depth = torch.full((fr.h, fr.w), float("nan"), dtype=torch.float32, device="cuda")
            torch.cuda.synchronize()
            _lib.check(L.gsr_set_depth_compositing(c.h, None if Zt is None else C.c_void_p(Zt.data_ptr()), C.c_void_p(depth.data_ptr())),
                       "gsr_set_depth_compositing")
        if case.compositor == "motion":
            motion = torch.full((fr.h, fr.w, 2), float("nan"), dtype=torch.float32, device="cuda")
            torch.cuda.synchronize()
            _lib.check(L.gsr_set_motion_vectors(c.h, C.c_void_p(motion.data_ptr())), "gsr_set_motion_vectors")
            c.render(fr.pvp, fr.pub, heatmap=heat)   # the previous frame: another camera, other instance transforms
            if case.inst:
                set_instances(c, fr.inst)            # the same layout: the appearance stays
        rgba = c.render(fr.vp, fr.ub, heatmap=heat)
        c.sync()
        st = c.stats()
        m = int(min(st.duplicates, st.capacity))
        T = st.tiles_x * st.tiles_y
        out = dict(rgba=rgba, depth=None if depth is None else depth.cpu().numpy(), motion=None if motion is None else motion.cpu().numpy(),
                   stats=st, keys=c.copy(_lib.GSR_BUF_KEYS, m, np.uint32), values=c.copy(_lib.GSR_BUF_VALUES, m, np.uint32),
                   bounds=c.copy(_lib.GSR_BUF_BOUNDS, T * 2, np.uint32).reshape(T, 2), records=c.copy(_lib.GSR_BUF_RECORDS, fr.drawn, REC_DTYPE))
    return out


@pytest.mark.parametrize("i", range(len(vm.CASES)), ids=vm.IDS)
def test_case_is_the_reference(i):
    case = vm.CASES[i]
    fr = vm.frame_of(case, N, SIZE, RAGGED)
    ref = vm.reference(fr)
    vm.assert_both_phase2_paths(ref)
    got = render_case(fr)
    st = got["stats"]
    assert (st.duplicates, st.visible, st.last_tile, bool(st.overflow)) == (ref["m"], ref["visible"], ref["last_tile"], False)
    np.testing.assert_array_equal(got["keys"], ref["keys"])
    np.testing.assert_array_equal(got["values"], ref["values"])
    np.testing.assert_array_equal(got["bounds"], ref["bounds"])
    ids = np.unique(ref["values"])
    for w in ("image_pos", "pos_xy", "conic", "pos_z", "color"):
        np.testing.assert_array_equal(bits(got["records"][w][ids]), bits(ref["records"][w][ids]), err_msg=f"record word {w}")
    np.testing.assert_array_equal(bits(got["rgba"]), bits(ref["rgba"]))
    assert st.staged == ref["staged"]
    assert (got["depth"] is None) == (case.compositor == "plain")
    if got["depth"] is not None:
        np.testing.assert_array_equal(bits(got["depth"]), bits(ref["depth"]))
    assert (got["motion"] is None) == (case.compositor != "motion")
    if got["motion"] is not None:
        np.testing.assert_array_equal(bits(got["motion"]), bits(ref["motion"]))
        assert np.abs(ref["motion"]).max() > 0
