"""Cost and use of splat contribution (gsr_set_splat_contribution) on a workload of bench.py (c3 by default), in one process:
  1. orbit frames alternating round by round between
       depth     depth compositing, no scene depth
       contrib   depth compositing + splat contribution
     the medians and spread of the compositor stage ('Render' of gsr_get_frame_history: tile order + compositor) and of the frame
     time (host wall time per frame, frames enqueued back to back);
  2. gsr_select_where and gsr_splat_histogram on the contribution properties;
  3. as information: the share of slots with pixels == 0 after a 360-frame orbit, and the frame difference (max abs, PSNR over rgb)
     at four orbit views after hiding the lowest 10 / 30 / 50 % of the splats by GSR_PROP_CONTRIBUTION.
    python ubench/splat_contribution.py [frames per case and round] [rounds] [workload]"""
import ctypes as C
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from godotgaussiansplatting_b200 import _lib  # noqa: E402
from godotgaussiansplatting_b200.rasterizer import read_splat_contribution, splat_filter  # noqa: E402
from tests.gsr_direct import Ctx  # noqa: E402

F = int(sys.argv[1]) if len(sys.argv) > 1 else 120
ROUNDS = int(sys.argv[2]) if len(sys.argv) > 2 else 4
wl = dict(bench.WORKLOADS[sys.argv[3] if len(sys.argv) > 3 else "c3"])
n, w, h = wl["n"], wl["w"], wl["h"]

try:
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                         timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    gpu = "unknown"
print(f"GPU: {gpu}; workload {wl['desc']}; {F} frames per case per round, {ROUNDS} rounds", flush=True)

ctx = Ctx(n, w, h)
for lo, blk in bench.raw_chunks(wl):
    ctx.upload_ply_raw(blk, first=lo)
ORBIT = 360
frames = bench.frame_params(wl, max(F + 10, ORBIT))
L = ctx.L
depth_out = torch.empty((h, w), dtype=torch.float32, device="cuda")
acc = torch.zeros(32 * n, dtype=torch.uint8, device="cuda")
torch.cuda.synchronize()
_lib.check(L.gsr_set_depth_compositing(ctx.h, None, C.c_void_p(depth_out.data_ptr())), "gsr_set_depth_compositing")
CASES = ("depth", "contrib")


def set_contrib(on):
    _lib.check(L.gsr_set_splat_contribution(ctx.h, C.c_void_p(acc.data_ptr()) if on else None, n if on else 0), "gsr_set_splat_contribution")


def history(k):
    buf = (_lib.GsrFrameRecord * k)()
    got = C.c_uint32(0)
    _lib.check(L.gsr_get_frame_history(ctx.h, k, buf, C.byref(got)), "gsr_get_frame_history")
    return np.array([buf[i].stage_ms[3] for i in range(got.value)])


def run(name):
    set_contrib(name == "contrib")
    for i in range(10):
        ctx.render_async(*frames[i])
    ctx.sync()
    t0 = time.perf_counter()
    for i in range(10, 10 + F):
        ctx.render_async(*frames[i])
    ctx.sync()
    return history(F), (time.perf_counter() - t0) * 1e3 / F


# ---- 1. the mode's cost ------------------------------------------------------------------------------------------------------
comp = {k: [] for k in CASES}
frame_ms = {k: [] for k in CASES}
for r in range(ROUNDS):
    for name in CASES:
        m, f = run(name)
        comp[name].append(np.median(m))
        frame_ms[name].append(f)
    print(f"round {r}: " + "  ".join(f"{k} {comp[k][-1]:.4f} ms / frame {frame_ms[k][-1]:.4f} ms" for k in CASES), flush=True)
print(f"median (min..max) of the {ROUNDS} round medians; compositor stage = tile order + compositor")
for name in CASES:
    c, f = np.array(comp[name]), np.array(frame_ms[name])
    print(f"  {name:8s} compositor {np.median(c):.4f} ms ({c.min():.4f}..{c.max():.4f})  frame {np.median(f):.4f} ms ({f.min():.4f}..{f.max():.4f})",
          flush=True)

# ---- 3a. a 360-frame orbit into a zeroed buffer --------------------------------------------------------------------------------
set_contrib(True)
_lib.check(L.gsr_reset_splat_contribution(ctx.h), "gsr_reset_splat_contribution")
for i in range(ORBIT):
    ctx.render_async(*frames[i])
ctx.sync()
got = C.c_uint32(0)
_lib.check(L.gsr_splat_contribution_frames(ctx.h, C.byref(got)), "gsr_splat_contribution_frames")
c = read_splat_contribution(acc)
print(f"orbit: {got.value} frames accumulated; slots with pixels == 0: {np.mean(c['pixels'] == 0) * 100:.2f} % of {n}; "
      f"median views {np.median(c['views']):.0f}", flush=True)

# ---- 2. the property calls -----------------------------------------------------------------------------------------------------
def timed(fn, reps=20):
    fn()
    ctx.sync()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    ctx.sync()
    return (time.perf_counter() - t0) * 1e3 / reps


thr = [float(np.quantile(c["weight"], q)) for q in (0.1, 0.3, 0.5)]
edges = np.unique(np.quantile(c["weight"], np.linspace(0, 1, 257))).astype(np.float32)
counts = np.zeros(edges.size + 2, dtype=np.uint64)
mm = np.zeros(2, dtype=np.float32)
fp = C.POINTER(C.c_float)


def where(filters):
    arr = (_lib.GsrSplatFilter * len(filters))(*filters)
    _lib.check(L.gsr_select_where(ctx.h, arr, len(filters), -1, _lib.GSR_SELECT_SET), "gsr_select_where")


def hist(prop):
    f = splat_filter(prop)
    _lib.check(L.gsr_splat_histogram(ctx.h, C.byref(f), -1, _lib.GSR_HISTOGRAM_KEPT, edges.ctypes.data_as(fp), edges.size - 1,
                                     counts.ctypes.data_as(C.POINTER(C.c_uint64)), mm.ctypes.data_as(fp)), "gsr_splat_histogram")


print(f"select_where CONTRIBUTION <= q30: {timed(lambda: where([splat_filter(_lib.GSR_PROP_CONTRIBUTION, -np.inf, thr[1])])):.3f} ms")
print(f"select_where CONTRIBUTION + OPACITY: "
      f"{timed(lambda: where([splat_filter(_lib.GSR_PROP_CONTRIBUTION, -np.inf, thr[1]), splat_filter(_lib.GSR_PROP_OPACITY, 0.0, 0.5)])):.3f} ms")
print(f"splat_histogram CONTRIBUTION, {edges.size - 1} quantile bins (synchronises): {timed(lambda: hist(_lib.GSR_PROP_CONTRIBUTION)):.3f} ms")
print(f"splat_histogram VIEWS: {timed(lambda: hist(_lib.GSR_PROP_VIEWS)):.3f} ms", flush=True)

# ---- 3b. pruning by contribution (the orbit's buffer; the comparison frames are rendered with the mode off) --------------------
set_contrib(False)
views = [frames[i] for i in (0, 90, 180, 270)]
base = [ctx.render(*v)[..., :3].astype(np.float64) for v in views]
for q, t in zip((10, 30, 50), thr):
    set_contrib(True)
    where([splat_filter(_lib.GSR_PROP_CONTRIBUTION, -np.inf, t)])
    _lib.check(L.gsr_hide_selection(ctx.h), "gsr_hide_selection")
    set_contrib(False)
    hid = C.c_uint64(0)
    sel = C.c_uint64(0)
    _lib.check(L.gsr_splat_mask_counts(ctx.h, C.byref(sel), C.byref(hid)), "gsr_splat_mask_counts")
    errs, psnr = [], []
    for v, b in zip(views, base):
        d = ctx.render(*v)[..., :3].astype(np.float64) - b
        errs.append(np.abs(d).max())
        mse = float(np.mean(d * d))
        psnr.append(np.inf if mse == 0 else 10 * np.log10(1.0 / mse))
    print(f"hide the lowest {q} % by CONTRIBUTION ({hid.value} hidden): max abs {max(errs):.4f}, PSNR min {min(psnr):.2f} dB, "
          f"mean {np.mean(psnr):.2f} dB over 4 views", flush=True)
    _lib.check(L.gsr_unhide_all(ctx.h), "gsr_unhide_all")
ctx.close()
