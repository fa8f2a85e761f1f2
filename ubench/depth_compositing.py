"""Cost of depth compositing (gsr_set_depth_compositing) at c3: the compositor stage ('Render' of gsr_get_frame_history: tile order +
compositor) of orbit frames for four cases, alternated round by round in one process:
    off        the default frame
    on         depth compositing, no scene depth
    on_half    a scene-depth plane at depth 0 over the lower half of the frame (everything there is hidden)
    on_front   a scene-depth plane at depth 0 over the whole frame (every tile ends after its first chunk)
    python ubench/depth_compositing.py [frames per case and round] [rounds] [workload]"""
import ctypes as C
import os
import subprocess
import sys

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
print(f"GPU: {gpu}; workload {wl['desc']}; {F} frames per case per round, {ROUNDS} rounds", flush=True)

ctx = Ctx(n, w, h)
for lo, blk in bench.raw_chunks(wl):
    ctx.upload_ply_raw(blk, first=lo)
frames = bench.frame_params(wl, F + 10)
depth_out = torch.empty((h, w), dtype=torch.float32, device="cuda")
half = torch.full((h, w), float("inf"), dtype=torch.float32, device="cuda")
half[h // 2:] = 0.0
front = torch.zeros((h, w), dtype=torch.float32, device="cuda")
torch.cuda.synchronize()
CASES = {"off": None, "on": (None, depth_out), "on_half": (half, depth_out), "on_front": (front, depth_out)}


def set_case(name):
    z, d = CASES[name] or (None, None)
    _lib.check(ctx.L.gsr_set_depth_compositing(ctx.h, C.c_void_p(None if z is None else z.data_ptr()), C.c_void_p(None if d is None else d.data_ptr())),
               "gsr_set_depth_compositing")


def history(k):
    buf = (_lib.GsrFrameRecord * k)()
    got = C.c_uint32(0)
    _lib.check(ctx.L.gsr_get_frame_history(ctx.h, k, buf, C.byref(got)), "gsr_get_frame_history")
    return np.array([buf[i].stage_ms[3] for i in range(got.value)]), np.array([buf[i].staged for i in range(got.value)])


def run(name):
    set_case(name)
    for i in range(10):
        ctx.render_async(*frames[i])
    ctx.sync()
    for i in range(10, 10 + F):
        ctx.render_async(*frames[i])
    ctx.sync()
    return history(F)


ms = {k: [] for k in CASES}
staged = {k: [] for k in CASES}
for r in range(ROUNDS):
    for name in CASES:
        m, s = run(name)
        ms[name].append(m)
        staged[name].append(s)
    print(f"round {r}: " + "  ".join(f"{k} {np.median(ms[k][-1]):.4f} ms" for k in CASES), flush=True)

base = np.median(np.concatenate(ms["off"]))
print(f"compositor stage (tile order + compositor), median over {ROUNDS} x {F} frames; spread = min..max of the per-round medians")
for name in CASES:
    allm = np.concatenate(ms[name])
    rounds = [np.median(x) for x in ms[name]]
    print(f"  {name:9s} {np.median(allm):.4f} ms  ({100 * (np.median(allm) / base - 1):+6.1f} % vs off)  spread {min(rounds):.4f}..{max(rounds):.4f}  "
          f"staged C {np.median(np.concatenate(staged[name])) / 1e6:.2f} M", flush=True)
set_case("off")
ctx.close()
