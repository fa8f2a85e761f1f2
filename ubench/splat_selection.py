"""Cost of splat selection (gsr_select_*) at c3: orbit frames alternating round by round between
    none          no masks (the default kernels)
    empty         masks in use, nothing selected or hidden (the CUT = true kernels)
    hidden30      30 % of the splats hidden
    selected10    10 % selected, highlighted at the default style
and the time per operation (host wall time of 50 back-to-back calls ending in a synchronise) of a 4- and a 64-vertex polygon, a volume,
select_ids over the full frame, select_all and hide_selection, and the frame time with front / back overlap with and without a
4-vertex lasso preview before every frame.  Reports medians with the card's name and power limit.
    python ubench/splat_selection.py [frames per case and round] [rounds] [workload]"""
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
from godotgaussiansplatting_b200.rasterizer import pack_mask  # noqa: E402
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
frames = bench.frame_params(wl, F + 10)
U32P = C.POINTER(C.c_uint32)
FP = C.POINTER(C.c_float)
rng = np.random.default_rng(1)
hid30 = rng.random(n) < 0.3
sel10 = (rng.random(n) < 0.1)
MASKS = {"empty": (np.zeros(n, bool), np.zeros(n, bool)), "hidden30": (hid30, np.zeros(n, bool)), "selected10": (np.zeros(n, bool), sel10)}
CASES = ("none", "empty", "hidden30", "selected10")


def set_case(name):
    if name == "none":
        _lib.check(ctx.L.gsr_clear_splat_masks(ctx.h), "gsr_clear_splat_masks")
        return
    hm, sm = (pack_mask(m, n) for m in MASKS[name])
    _lib.check(ctx.L.gsr_set_splat_masks(ctx.h, hm.ctypes.data_as(U32P), sm.ctypes.data_as(U32P), hm.size), "gsr_set_splat_masks")


def run(name):
    set_case(name)
    for i in range(10):
        ctx.render_async(*frames[i])
    ctx.sync()
    t0 = time.perf_counter()
    for i in range(10, 10 + F):
        ctx.render_async(*frames[i])
    ctx.sync()
    return (time.perf_counter() - t0) * 1e3 / F


frame_ms = {k: [] for k in CASES}
for r in range(ROUNDS):
    for name in CASES:
        frame_ms[name].append(run(name))
    print(f"round {r}: " + "  ".join(f"{k} {frame_ms[k][-1]:.4f} ms" for k in CASES), flush=True)
base = np.median(frame_ms["none"])
print(f"frame time, median over {ROUNDS} rounds of {F} frames (host wall time per frame, back to back)")
for name in CASES:
    m = np.median(frame_ms[name])
    print(f"  {name:11s} {m:.4f} ms ({100 * (m / base - 1):+6.1f} %)", flush=True)

# ---- a lasso preview before every frame, with front / back overlap (gsr_debug_pipeline(ctx, 1)) ----
quad = np.array([[w * 0.2, h * 0.2], [w * 0.8, h * 0.2], [w * 0.8, h * 0.8], [w * 0.2, h * 0.8]], dtype=np.float32)


def run_overlap(lasso):
    _lib.check(ctx.L.gsr_select_all(ctx.h, _lib.GSR_SELECT_SUBTRACT), "in use")
    t0 = 0.0
    for i in range(10 + F):
        if i == 10:
            ctx.sync()
            t0 = time.perf_counter()
        if lasso:
            vpi = np.ascontiguousarray(frames[i][0], dtype=np.float32)
            _lib.check(ctx.L.gsr_select_polygon(ctx.h, vpi.ctypes.data_as(FP), 1.0, -1, quad.ctypes.data_as(FP), 4, _lib.GSR_SELECT_SET), "lasso")
        ctx.render_async(*frames[i])
    ctx.sync()
    return (time.perf_counter() - t0) * 1e3 / F


_lib.check(ctx.L.gsr_debug_pipeline(ctx.h, 1), "gsr_debug_pipeline")
ov = {"overlap, masks in use": [], "overlap, lasso before every frame": []}
for r in range(ROUNDS):
    ov["overlap, masks in use"].append(run_overlap(False))
    ov["overlap, lasso before every frame"].append(run_overlap(True))
_lib.check(ctx.L.gsr_debug_pipeline(ctx.h, -1), "gsr_debug_pipeline")
print(f"with front / back overlap, median over {ROUNDS} rounds of {F} frames")
for name, v in ov.items():
    print(f"  {name:34s} {np.median(v):.4f} ms", flush=True)

# ---- operations ----
vp = np.ascontiguousarray(frames[0][0], dtype=np.float32)
ids = torch.zeros((h, w, 2), dtype=torch.int32, device="cuda")
depth = torch.zeros((h, w), dtype=torch.float32, device="cuda")
torch.cuda.synchronize()
_lib.check(ctx.L.gsr_set_depth_compositing(ctx.h, None, C.c_void_p(depth.data_ptr())), "depth")
_lib.check(ctx.L.gsr_set_splat_ids(ctx.h, C.c_void_p(ids.data_ptr())), "ids")
ctx.render_async(*frames[0])
ctx.sync()
t = np.linspace(0, 2 * np.pi, 64, endpoint=False)
lasso = np.stack([w * (0.5 + 0.3 * np.cos(t) * (1 + 0.2 * np.sin(5 * t))), h * (0.5 + 0.3 * np.sin(t))], axis=1).astype(np.float32)
vol = (_lib.GsrCutout * 1)()
vol[0].to_local[:] = [2, 0, 0, 0, 2, 0, 0, 0, 2, 0, 0, -5]
vol[0].shape, vol[0].action, vol[0].space = _lib.GSR_CUTOUT_ELLIPSOID, 0, _lib.GSR_CUTOUT_FRAME
OPS = {
    "polygon4": lambda: ctx.L.gsr_select_polygon(ctx.h, vp.ctypes.data_as(FP), 1.0, -1, quad.ctypes.data_as(FP), 4, _lib.GSR_SELECT_TOGGLE),
    "polygon64": lambda: ctx.L.gsr_select_polygon(ctx.h, vp.ctypes.data_as(FP), 1.0, -1, lasso.ctypes.data_as(FP), 64, _lib.GSR_SELECT_TOGGLE),
    "volume": lambda: ctx.L.gsr_select_volume(ctx.h, vol, 1.0, -1, _lib.GSR_SELECT_TOGGLE),
    "select_ids": lambda: ctx.L.gsr_select_ids(ctx.h, C.c_void_p(ids.data_ptr()), 0, 0, w, h, _lib.GSR_SELECT_TOGGLE),
    "select_all": lambda: ctx.L.gsr_select_all(ctx.h, _lib.GSR_SELECT_TOGGLE),
    "hide_selection": lambda: ctx.L.gsr_hide_selection(ctx.h),
}
op_us = {k: [] for k in OPS}
for r in range(ROUNDS):
    for name, fn in OPS.items():
        _lib.check(fn(), name)
        ctx.sync()
        t0 = time.perf_counter()
        for _ in range(50):
            _lib.check(fn(), name)
        ctx.sync()
        op_us[name].append((time.perf_counter() - t0) * 1e6 / 50)
print("time per operation, median over rounds of 50 back-to-back calls (host wall time, includes the launch)")
for name in OPS:
    print(f"  {name:15s} {np.median(op_us[name]):9.1f} us", flush=True)
ctx.close()
