"""Dump the compositor's schedule trace for one c3 frame: python ubench/trace_compositor.py [frame] [out.npy] (default trace.npy)"""
import ctypes as C, os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench
from godotgaussiansplatting_b200 import _lib
from godotgaussiansplatting_b200.camera import default_camera
from godotgaussiansplatting_b200.ply_file import PlyFile
from godotgaussiansplatting_b200.rasterizer import GaussianSplattingRasterizer, RenderTexture
wl = dict(bench.WORKLOADS["c3"])
stub = PlyFile(); stub.size = wl["n"]
r = GaussianSplattingRasterizer(stub, (wl["w"], wl["h"]), RenderTexture(), default_camera())
r.init_gpu(load=False)
for lo, s60 in bench.scene_chunks(wl):
    r.upload_splats(s60, lo)
L = _lib.lib()
_lib.check(L.gsr_debug_enable_trace(r._ctx, 200000), "trace")
frames = bench.frame_params(wl, 8, first=int(sys.argv[1]) if len(sys.argv) > 1 else 50)
for vp, ub in frames:
    r.render_raw(vp, ub, 0.0, None, asynchronous=False)
r.sync()
n = r.debug_copy(_lib.GSR_BUF_COMPOSITOR_TRACE_COUNT, 1, np.uint32)[0]
tr = r.debug_copy(_lib.GSR_BUF_COMPOSITOR_TRACE, 200000 * 4, np.uint64).reshape(-1, 4)[:n]
st = r.stats()
np.save(sys.argv[2] if len(sys.argv) > 2 else "trace.npy", tr)
print("items", n, "render ms", st.stage_ms[3], "C", st.staged)
# item = {tile << 32 | SM id, start ns, end ns, consumed chunks << 32 | list chunks << 1 | 1}
t0 = tr[:, 1].astype(np.float64); t1 = tr[:, 2].astype(np.float64)
cons = (tr[:, 3] >> 32).astype(np.int64)
busy = cons > 0
base = t0.min()
print("span us", (t1.max() - base) / 1e3, "busy tiles", int(busy.sum()), "chunks", int(cons.sum()),
      "mean us/chunk/CTA", float(((t1 - t0)[busy]).sum() / max(cons.sum(), 1) / 1e3))
sm = (tr[:, 0] & 0xffffffff).astype(np.int64)
last = np.array([t1[busy & (sm == s)].max() if (busy & (sm == s)).any() else base for s in np.unique(sm)])
print("per-SM last busy end us: min/median/max", (last.min() - base) / 1e3, (np.median(last) - base) / 1e3, (last.max() - base) / 1e3)
