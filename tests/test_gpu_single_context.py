"""The single-context rule (include/gsr.h, "Single-context features") as one matrix, through the C-ABI.  While any single-context feature
is on, every call that would shard the context returns GSR_ERR_STATE and leaves the band and the frame as they were; on a context
sharded in any of the four ways, every call that would turn a feature on returns GSR_ERR_STATE while the calls that turn one off
succeed, and the same calls succeed once the sharding is undone."""
import ctypes as C

import numpy as np
import pytest

from godotgaussiansplatting_b200 import _lib
from tests import cutout_reference as cr
from tests import ortho_reference as oref
from tests.gsr_direct import Ctx
from tests.scenes import make_scene
from tests.test_gpu_cutouts import set_cut
from tests.test_gpu_instances import set_instances
from tests.test_gpu_sh_degree import ShCtx
from tests.test_instances import rigid

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

N, W, H = 4096, 320, 200
TILES_Y = (H + 15) // 16
OK, STATE = _lib.GSR_OK, _lib.GSR_ERR_STATE
INSTANCES = [(0, 2048, rigid(80)), (1024, 2048, rigid(81))]
CUTOUTS = [cr.volume(np.hstack([0.5 * np.eye(3), np.zeros((3, 1))]))]   # keep the splats inside a box of half-width 2


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


class Planes:
    """Caller-owned device planes of depth compositing and its companions."""

    def __init__(self):
        self.depth = torch.zeros((H, W), dtype=torch.float32, device="cuda")
        self.motion = torch.zeros((H, W, 2), dtype=torch.float32, device="cuda")
        self.ids = torch.zeros((H, W, 2), dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()

    def depth_on(self, c):
        return c.L.gsr_set_depth_compositing(c.h, None, C.c_void_p(self.depth.data_ptr()))

    def all_on(self, c):
        return (self.depth_on(c) or c.L.gsr_set_motion_vectors(c.h, C.c_void_p(self.motion.data_ptr()))
                or c.L.gsr_set_splat_ids(c.h, C.c_void_p(self.ids.data_ptr())))


# feature: (gsr_config.sh_bands, flags, the call that turns it on after creation or None for a store fixed at creation)
FEATURES = {
    "depth_compositing": (0, 0, lambda c, p: p.depth_on(c)),
    "depth_motion_ids": (0, 0, lambda c, p: p.all_on(c)),
    "instances": (0, 0, lambda c, p: set_instances(c, INSTANCES)),
    "store_3_bands": (3, 0, None),
    "degree_1": (0, 0, lambda c, p: c.degree(1)),
    "store_binary16": (0, _lib.GSR_FLAG_SH_HALF, None),
    "antialiasing": (0, 0, lambda c, p: c.L.gsr_set_antialiasing(c.h, C.c_float(0.3))),
    "view_depth_order": (0, 0, lambda c, p: c.L.gsr_set_depth_order(c.h, _lib.GSR_DEPTH_ORDER_VIEW_DEPTH)),
    "cutouts": (0, 0, lambda c, p: set_cut(c, CUTOUTS)),
}
EXPORTED_WITH = {"depth_compositing", "depth_motion_ids", "instances"}   # gsr_group_export accepts these; gsr_group_attach does not


@pytest.mark.parametrize("feature", list(FEATURES))
def test_a_feature_refuses_every_sharding_call(feature):
    bands, flags, turn_on = FEATURES[feature]
    splat60, vp, ub = make_scene(N, 7, W, H)
    planes = Planes()
    handles = (C.c_ubyte * 128)()
    blob = (C.c_ubyte * _lib.GSR_GROUP_BLOB_BYTES)()
    with ShCtx(N, W, H, bands, flags) as c:
        L = c.L
        c.upload(splat60)
        own = bytes(_lib.GSR_GROUP_BLOB_BYTES)   # a store fixed at creation never exports, so it cannot attach either
        if turn_on is not None:
            own = c.group_export()   # before the feature is on: the attach below is refused for the feature
            _lib.check(turn_on(c, planes), feature)
        before = c.render(vp, ub)
        assert L.gsr_set_band(c.h, 0, 3) == STATE
        assert L.gsr_set_row_interleave(c.h, 0, 2) == STATE
        assert L.gsr_peer_export_framebuffers(c.h, handles) == STATE
        assert L.gsr_peer_import_framebuffers(c.h, handles) == STATE   # zero handles: refused before they are opened
        pair = (C.c_ubyte * (2 * len(own))).from_buffer_copy(own + own)
        assert L.gsr_group_attach(c.h, 0, 2, pair) == STATE
        assert L.gsr_group_export(c.h, blob) == (OK if feature in EXPORTED_WITH else STATE)
        st = c.stats()
        assert (st.band_y0, st.band_y1) == (0, TILES_Y)
        _lib.check(L.gsr_set_band(c.h, 0, TILES_Y), "gsr_set_band: the full frame")
        _lib.check(L.gsr_set_row_interleave(c.h, 0, 1), "gsr_set_row_interleave(0, 1)")
        np.testing.assert_array_equal(bits(c.render(vp, ub)), bits(before))


def turn_on_calls(c, planes, vpp, ub):
    L = c.L
    return {
        "gsr_set_depth_compositing": lambda: planes.depth_on(c),
        "gsr_set_instances": lambda: set_instances(c, INSTANCES),
        "gsr_set_sh_degree(0)": lambda: c.degree(0),
        "gsr_set_sh_degree(1)": lambda: c.degree(1),
        "gsr_set_sh_degree(2)": lambda: c.degree(2),
        "gsr_set_antialiasing(0.3)": lambda: L.gsr_set_antialiasing(c.h, C.c_float(0.3)),
        "gsr_set_depth_order(VIEW_DEPTH)": lambda: L.gsr_set_depth_order(c.h, _lib.GSR_DEPTH_ORDER_VIEW_DEPTH),
        "gsr_set_cutouts": lambda: set_cut(c, CUTOUTS),
        "orthographic gsr_render": lambda: L.gsr_render(c.h, vpp, ub, 0.0, None),
        "orthographic gsr_render_async": lambda: L.gsr_render_async(c.h, vpp, ub, 0.0, None),
    }


def turn_off_calls(c):
    L = c.L
    return {
        "gsr_set_depth_compositing(NULL, NULL)": lambda: L.gsr_set_depth_compositing(c.h, None, None),
        "gsr_set_instances(n = 0)": lambda: set_instances(c, []),
        "gsr_set_sh_degree(-1)": lambda: c.degree(-1),
        "gsr_set_sh_degree(3)": lambda: c.degree(3),
        "gsr_set_antialiasing(0)": lambda: L.gsr_set_antialiasing(c.h, C.c_float(0.0)),
        "gsr_set_depth_order(KEY16)": lambda: L.gsr_set_depth_order(c.h, _lib.GSR_DEPTH_ORDER_KEY16),
        "gsr_set_cutouts(n = 0)": lambda: L.gsr_set_cutouts(c.h, None, 0),
    }


def test_a_sharded_context_refuses_every_feature():
    splat60, _, _ = make_scene(N, 7, W, H)
    vp, ub = oref.ortho_camera(W, H, size=2.6, near=0.5, far=4.5, frame=25)
    vpp = np.ascontiguousarray(vp, dtype=np.float32).ctypes.data_as(C.POINTER(C.c_float))
    planes = Planes()
    handles = (C.c_ubyte * 128)()
    with ShCtx(N, W, H, 0, _lib.GSR_FLAG_ORTHOGRAPHIC) as c, Ctx(N, W, H) as peer:
        L = c.L
        c.upload(splat60)

        def attach():   # a shard group of two contexts on one device, in this process
            blobs = c.group_export() + peer.group_export()
            c.group_attach(0, 2, blobs)
            peer.group_attach(1, 2, blobs)
            return OK

        def detach():
            return L.gsr_group_detach(c.h) or L.gsr_group_detach(peer.h)

        states = {
            "partial band": (lambda: L.gsr_set_band(c.h, 0, 3), lambda: L.gsr_set_band(c.h, 0, TILES_Y)),
            "row interleave": (lambda: L.gsr_set_row_interleave(c.h, 0, 2), lambda: L.gsr_set_row_interleave(c.h, 0, 1)),
            "peer framebuffers": (lambda: L.gsr_peer_export_framebuffers(c.h, handles), lambda: L.gsr_resize(c.h, W, H)),
            "shard group": (attach, detach),   # no frame is rendered while it is attached
        }
        on, off = turn_on_calls(c, planes, vpp, ub), turn_off_calls(c)
        for state, (setup, undo) in states.items():
            _lib.check(setup(), state)
            for name, call in on.items():
                assert call() == STATE, f"{name} with {state}"
            for name, call in off.items():
                assert call() == OK, f"{name} with {state}"
            _lib.check(undo(), f"undo {state}")
            for name, call in on.items():
                assert call() == OK, f"{name} after {state}"
            for name, call in off.items():
                assert call() == OK, f"{name} after {state}"
            c.sync()
