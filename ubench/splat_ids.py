"""Cost of splat IDs (gsr_set_splat_ids) at c3 with moving instances: orbit frames of the cloud drawn as 8 instances whose transforms
change every frame, alternating round by round between
    depth         depth compositing, no scene depth
    ids           depth compositing + splat IDs
    motion_ids    depth compositing + motion vectors + splat IDs
Reports the medians of the compositor stage ('Render' of gsr_get_frame_history: tile order + compositor) and of the frame time.
    python ubench/splat_ids.py [frames per case and round] [rounds] [workload]"""
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
print(f"GPU: {gpu}; workload {wl['desc']} as 8 moving instances; {F} frames per case per round, {ROUNDS} rounds", flush=True)

ctx = Ctx(n, w, h)
for lo, blk in bench.raw_chunks(wl):
    ctx.upload_ply_raw(blk, first=lo)
frames = bench.frame_params(wl, F + 10)
K = 8
step = n // K
ranges = [(k * step, step if k < K - 1 else n - k * step) for k in range(K)]


def set_instances(f):
    arr = (_lib.GsrInstance * K)()
    for k, (first, count) in enumerate(ranges):
        arr[k].first, arr[k].count = first, count
        d = 0.002 * f * ((k % 3) - 1)
        arr[k].to_frame[:] = [1, 0, 0, 0, 1, 0, 0, 0, 1, d, 0.5 * d, 0.0]
    _lib.check(ctx.L.gsr_set_instances(ctx.h, arr, K), "gsr_set_instances")


depth_out = torch.empty((h, w), dtype=torch.float32, device="cuda")
motion_out = torch.empty((h, w, 2), dtype=torch.float32, device="cuda")
ids_out = torch.empty((h, w, 2), dtype=torch.int32, device="cuda")
torch.cuda.synchronize()
_lib.check(ctx.L.gsr_set_depth_compositing(ctx.h, None, C.c_void_p(depth_out.data_ptr())), "gsr_set_depth_compositing")
CASES = ("depth", "ids", "motion_ids")


def set_splat_ids(address):
    return ctx.L.gsr_set_splat_ids(ctx.h, None if address is None else C.c_void_p(address))


def history(k):
    buf = (_lib.GsrFrameRecord * k)()
    got = C.c_uint32(0)
    _lib.check(ctx.L.gsr_get_frame_history(ctx.h, k, buf, C.byref(got)), "gsr_get_frame_history")
    return np.array([buf[i].stage_ms[3] for i in range(got.value)])


def run(name):
    _lib.check(set_splat_ids(None), "gsr_set_splat_ids")   # (first: motion may not take a plane the IDs hold)
    _lib.check(ctx.L.gsr_set_motion_vectors(ctx.h, C.c_void_p(motion_out.data_ptr() if name == "motion_ids" else None)),
               "gsr_set_motion_vectors")
    _lib.check(set_splat_ids(ids_out.data_ptr() if name != "depth" else None), "gsr_set_splat_ids")
    for i in range(10):
        set_instances(i)
        ctx.render_async(*frames[i])
    ctx.sync()
    t0 = time.perf_counter()
    for i in range(10, 10 + F):
        set_instances(i)
        ctx.render_async(*frames[i])
    ctx.sync()
    return history(F), (time.perf_counter() - t0) * 1e3 / F


comp = {k: [] for k in CASES}
frame_ms = {k: [] for k in CASES}
for r in range(ROUNDS):
    for name in CASES:
        m, f = run(name)
        comp[name].append(m)
        frame_ms[name].append(f)
    print(f"round {r}: " + "  ".join(f"{k} {np.median(comp[k][-1]):.4f} ms / frame {frame_ms[k][-1]:.4f} ms" for k in CASES), flush=True)

base_c, base_f = np.median(np.concatenate(comp["depth"])), np.median(frame_ms["depth"])
print(f"median over {ROUNDS} x {F} frames (compositor stage = tile order + compositor; frame = host wall time per frame, back to back)")
for name in CASES:
    mc, mf = np.median(np.concatenate(comp[name])), np.median(frame_ms[name])
    print(f"  {name:10s} compositor {mc:.4f} ms ({100 * (mc / base_c - 1):+6.1f} %)  frame {mf:.4f} ms ({100 * (mf / base_f - 1):+6.1f} %)", flush=True)
_lib.check(set_splat_ids(None), "gsr_set_splat_ids")
_lib.check(ctx.L.gsr_set_motion_vectors(ctx.h, None), "gsr_set_motion_vectors")
ctx.close()
