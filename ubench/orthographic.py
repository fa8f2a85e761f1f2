"""Cost of the orthographic projection path (GSR_FLAG_ORTHOGRAPHIC) at c3: the projection stage ('Projection' of gsr_get_frame_history:
clear + projection), the sort, the compositor ('Render') and the whole frame (sum of the stages) of orbit frames for two cases,
alternated round by round on one flagged context:
    perspective    the c3 orbit camera (fov 75), packed the reference's way: the perspective path
    orthographic   the same orbit poses with an orthographic projection whose size gives the cloud the perspective camera's screen
                   height at the orbit radius (2 * 2.5 * tan(37.5 deg) = 3.84 units), near / far = 1 / 4 framing the unit-ball cloud
The projection column is the cost of the path.  The other columns compare two different pictures: M (pairs) and C (staged splats)
differ, and they are printed with them.
    python ubench/orthographic.py [frames per case and round] [rounds] [workload]"""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from godotgaussiansplatting_b200 import _lib  # noqa: E402
from godotgaussiansplatting_b200 import camera as cam  # noqa: E402
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

SIZE = 2.0 * 2.5 * math.tan(math.radians(75.0 / 2.0))
NEAR, FAR = 1.0, 4.0


def ortho_frames(k):
    out = []
    for f, (_, ub) in enumerate(bench.frame_params(wl, k)):
        c = cam.orbit_camera(f % 360, aspect=w / h)
        c.projection, c.size, c.near, c.far = cam.PROJECTION_ORTHOGONAL, SIZE, NEAR, FAR
        out.append((cam.pack_camera_push_constants(c.get_camera_transform(), c.get_camera_projection(), keep_w_row=True), ub))
    return out


c = Ctx(n, w, h, flags=_lib.GSR_FLAG_ORTHOGRAPHIC)
for lo, blk in synthetic_ply_chunks(n, wl["seed"]):
    c.upload_ply_raw(blk, first=lo)
FRAMES = {"perspective": bench.frame_params(wl, F + 10), "orthographic": ortho_frames(F + 10)}


def history(k):
    buf = (_lib.GsrFrameRecord * k)()
    got = C.c_uint32(0)
    _lib.check(c.L.gsr_get_frame_history(c.h, k, buf, C.byref(got)), "gsr_get_frame_history")
    st = np.array([[buf[i].stage_ms[j] for j in range(5)] for i in range(got.value)])
    return st, np.array([buf[i].duplicates for i in range(got.value)]), np.array([buf[i].staged for i in range(got.value)])


def run(name):
    frames = FRAMES[name]
    for i in range(10):
        c.render_async(*frames[i])
    c.sync()
    for i in range(10, 10 + F):
        c.render_async(*frames[i])
    c.sync()
    return history(F)


COLS = {"projection": 0, "sort": 1, "compositor": 3, "frame": 4}
stages = {k: [] for k in FRAMES}
pairs = {k: [] for k in FRAMES}
staged = {k: [] for k in FRAMES}
for r in range(ROUNDS):
    for name in FRAMES:
        st, m, cc = run(name)
        stages[name].append(st)
        pairs[name].append(m)
        staged[name].append(cc)
    print(f"round {r}: " + "  ".join(f"{k} {np.median(stages[k][-1][:, 0]):.4f}/{np.median(stages[k][-1][:, 4]):.4f} ms" for k in FRAMES), flush=True)

print(f"median over {ROUNDS} x {F} frames; spread = min..max of the per-round medians; orthographic size {SIZE:.3f}, near {NEAR}, far {FAR}")
base = {col: np.median(np.concatenate(stages["perspective"])[:, j]) for col, j in COLS.items()}
for name in FRAMES:
    line = [f"  {name:12s}"]
    for col, j in COLS.items():
        allv = np.concatenate(stages[name])[:, j]
        rounds = [np.median(s[:, j]) for s in stages[name]]
        line.append(f"{col} {np.median(allv):.4f} ms ({100 * (np.median(allv) / base[col] - 1):+6.1f} %) spread {min(rounds):.4f}..{max(rounds):.4f}")
    line.append(f"M {np.median(np.concatenate(pairs[name])) / 1e6:.2f} M  C {np.median(np.concatenate(staged[name])) / 1e6:.2f} M")
    print("   ".join(line), flush=True)
c.close()
