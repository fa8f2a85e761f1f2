"""Cost of depth-ordered frames (gsr_set_depth_order) at c3: the projection stage ('Projection' of gsr_get_frame_history: clear +
projection), the sort, the compositor ('Render') and the whole frame (sum of the stages) of the c3 orbit frames for the two modes,
alternated round by round on one context:
    key16   the default: pairs sorted by tile << 16 | 16-bit depth (4 passes over 32 bits)
    view    GSR_DEPTH_ORDER_VIEW_DEPTH: the projection also writes every pair's depth word; (tile, depth word) sorted in 6 passes
M (pairs) and C (staged splats) are printed with each mode: the pairs are the same, C may differ a little because the order inside a
tile decides when a pixel saturates.
    python ubench/depth_order.py [frames per case and round] [rounds] [workload]"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from godotgaussiansplatting_b200 import _lib  # noqa: E402
from godotgaussiansplatting_b200.synthetic import synthetic_ply_chunks  # noqa: E402
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

c = Ctx(n, w, h)
for lo, blk in synthetic_ply_chunks(n, wl["seed"]):
    c.upload_ply_raw(blk, first=lo)
FRAMES = bench.frame_params(wl, F + 10)
CASES = {"key16": _lib.GSR_DEPTH_ORDER_KEY16, "view": _lib.GSR_DEPTH_ORDER_VIEW_DEPTH}


def history(k):
    buf = (_lib.GsrFrameRecord * k)()
    got = C.c_uint32(0)
    _lib.check(c.L.gsr_get_frame_history(c.h, k, buf, C.byref(got)), "gsr_get_frame_history")
    st = np.array([[buf[i].stage_ms[j] for j in range(5)] for i in range(got.value)])
    return st, np.array([buf[i].duplicates for i in range(got.value)]), np.array([buf[i].staged for i in range(got.value)])


def run(mode):
    _lib.check(c.L.gsr_set_depth_order(c.h, mode), "gsr_set_depth_order")
    for i in range(10):
        c.render_async(*FRAMES[i])
    c.sync()
    for i in range(10, 10 + F):
        c.render_async(*FRAMES[i])
    c.sync()
    return history(F)


COLS = {"projection": 0, "sort": 1, "compositor": 3, "frame": 4}
stages = {k: [] for k in CASES}
pairs = {k: [] for k in CASES}
staged = {k: [] for k in CASES}
for r in range(ROUNDS):
    for name, v in CASES.items():
        st, m, cc = run(v)
        stages[name].append(st)
        pairs[name].append(m)
        staged[name].append(cc)
    print(f"round {r}: " + "  ".join(f"{k} {np.median(stages[k][-1][:, 0]):.4f}/{np.median(stages[k][-1][:, 4]):.4f} ms" for k in CASES), flush=True)

print(f"median over {ROUNDS} x {F} frames; spread = min..max of the per-round medians")
base = {col: np.median(np.concatenate(stages["key16"])[:, j]) for col, j in COLS.items()}
for name in CASES:
    line = [f"  {name:5s}"]
    for col, j in COLS.items():
        allv = np.concatenate(stages[name])[:, j]
        rounds = [np.median(s[:, j]) for s in stages[name]]
        line.append(f"{col} {np.median(allv):.4f} ms ({100 * (np.median(allv) / base[col] - 1):+6.1f} %) spread {min(rounds):.4f}..{max(rounds):.4f}")
    line.append(f"M {np.median(np.concatenate(pairs[name])) / 1e6:.2f} M  C {np.median(np.concatenate(staged[name])) / 1e6:.2f} M")
    print("   ".join(line), flush=True)
c.close()
