"""Worker of tests/test_gpu_splat_delete.py: a shard group of 2 contexts in ONE process on ONE GPU (as tests/group_inprocess_worker.py
builds it) on a store with vacant slots, written as gsr_delete_hidden leaves them.  The group's scatter projection must cull a vacant
slot like the single-context projection: rank 0's frames equal the single-context frames of the same store bit for bit, every rank's
sorted pairs are the single-context pairs of the tile rows it owns, the ranks' V add up to the single context's and every rank has its
last tile; and the single-context frame equals the frame of the original store with those slots' splats hidden.
CUDA_DEVICE_MAX_CONNECTIONS is raised by the caller (see tests/group_inprocess_worker.py)."""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from godotgaussiansplatting_b200 import _lib  # noqa: E402
from godotgaussiansplatting_b200.rasterizer import pack_mask  # noqa: E402
from tests.delete_reference import vacate_slots  # noqa: E402
from tests.gsr_direct import Ctx  # noqa: E402
from tests.scenes import make_scene  # noqa: E402

G, N, W, H = 2, 30000, 640, 360


def pinned(shape):
    import torch
    return torch.zeros(shape, dtype=torch.float32).pin_memory()


def vacant_store(c, vac):
    """Upload's store of c with the slots of `vac` made vacant, written back with gsr_restore_splat_store."""
    nbytes = int(c.L.gsr_splat_store_bytes(c.h))
    store = c.copy(_lib.GSR_BUF_SPLATS, nbytes // 4, np.float32).reshape(-1, (N + 255) // 256 * 256, 4)
    vacate_slots(store, vac)
    _lib.check(c.L.gsr_restore_splat_store(c.h, C.c_void_p(store.ctypes.data)), "gsr_restore_splat_store")
    c.sync()


def main():
    gx = (W + 15) // 16
    frames = [make_scene(N, 41, W, H, frame=f) for f in (0, 90, 200)]
    splat60 = frames[0][0]
    vac = np.random.default_rng(12).random(N) < 0.3
    single, hidden = Ctx(N, W, H), Ctx(N, W, H)
    ctxs = [Ctx(N, W, H) for _ in range(G)]
    try:
        for c in [single, hidden] + ctxs:
            c.upload(splat60)
        for c in [single] + ctxs:
            vacant_store(c, vac)
        hw, sw = pack_mask(vac, N), pack_mask(np.zeros(N, dtype=bool), N)
        u32p = C.POINTER(C.c_uint32)
        _lib.check(hidden.L.gsr_set_splat_masks(hidden.h, hw.ctypes.data_as(u32p), sw.ctypes.data_as(u32p), hw.size), "masks")
        blobs = b"".join(c.group_export() for c in ctxs)
        for r, c in enumerate(ctxs):
            c.group_attach(r, G, blobs)
        hosts = [pinned((H, W, 4)) for _ in frames]
        for k, (_, vp, ub) in enumerate(frames):
            for c in ctxs:
                c.render_async(vp, ub)
            ctxs[0].readback_async(hosts[k].data_ptr())
        for c in ctxs:
            c.sync()
        for k, (_, vp, ub) in enumerate(frames):
            want = single.render(vp, ub)
            st = single.stats()
            assert st.visible > 1000 and st.visible < N - 5000, st.visible
            assert np.array_equal(hidden.render(vp, ub).view(np.uint32), want.view(np.uint32)), f"frame {k}: vacant != hidden"
            assert np.array_equal(hosts[k].numpy().view(np.uint32), want.view(np.uint32)), f"frame {k}: group frame != single-context frame"
        t = single.taps()   # the last frame: the group's pairs, V and last tile
        rows = (t["keys"] >> 16) // gx
        vis = 0
        for r, c in enumerate(ctxs):
            g = c.taps()
            sel = rows % G == r
            assert np.array_equal(g["keys"], t["keys"][sel]), f"rank {r}: keys differ"
            assert np.array_equal(g["values"], t["values"][sel]), f"rank {r}: values differ"
            assert g["stats"].last_tile == t["stats"].last_tile, f"rank {r}: last tile {g['stats'].last_tile} != {t['stats'].last_tile}"
            vis += g["stats"].visible
        assert vis == t["stats"].visible, (vis, t["stats"].visible)
        print(f"GROUP_VACANCY_OK M={t['stats'].duplicates} V={vis}", flush=True)
    finally:
        for c in [single, hidden] + ctxs:
            c.close()


if __name__ == "__main__":
    main()
