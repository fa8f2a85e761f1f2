"""Cost of cutout sets (gsr_set_cutouts) at c3: the projection stage ('Projection' of gsr_get_frame_history: clear + projection), the
sort, the compositor ('Render') and the whole frame (sum of the stages) of the c3 orbit frames, the cases alternated round by round on one
context:
    none       no set: the default kernels
    keep_all   one KEEP box that contains every splat (every lane runs one inside test)
    sixteen    sixteen KEEP boxes, only the last of which contains the splats (every lane runs all sixteen tests: the worst set that
               removes nothing)
    crop_half  one KEEP box around the bulk of the cloud that keeps about half of the splats
M (pairs) and V (visible splats) are printed with each case.
    python ubench/cutouts.py [frames per case and round] [rounds] [workload]"""
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

# the stored positions (plane 0 of GSR_BUF_SPLATS: x, y, z, creation time), model scale 1
stride = (n + 255) // 256 * 256
pos = c.copy(_lib.GSR_BUF_SPLATS, 4 * stride, np.float32).reshape(stride, 4)[:n, :3].astype(np.float64)
centre = np.median(pos, axis=0)
spread = np.median(np.abs(pos - centre), axis=0)


def box(c0, half):
    v = _lib.GsrCutout()
    A = np.diag(1.0 / np.asarray(half, dtype=np.float64))
    v.to_local[:] = [float(x) for x in np.concatenate([A, (-A @ c0)[:, None]], axis=1).T.reshape(12)]
    v.shape, v.action, v.space = _lib.GSR_CUTOUT_BOX, _lib.GSR_CUTOUT_KEEP, _lib.GSR_CUTOUT_FRAME
    return v


def inside_fraction(k):
    return float((np.abs(pos[::16] - centre) <= k * spread).all(axis=1).mean())


lo_k, hi_k = 0.1, 50.0   # the box scale that keeps half of the cloud
for _ in range(40):
    mid = 0.5 * (lo_k + hi_k)
    lo_k, hi_k = (mid, hi_k) if inside_fraction(mid) < 0.5 else (lo_k, mid)
everything = box(np.zeros(3), np.full(3, 1e6))
nowhere = box(np.full(3, 1e9), np.ones(3))
CASES = {"none": [], "keep_all": [everything], "sixteen": [nowhere] * 15 + [everything], "crop_half": [box(centre, hi_k * spread)]}


def history(k):
    buf = (_lib.GsrFrameRecord * k)()
    got = C.c_uint32(0)
    _lib.check(c.L.gsr_get_frame_history(c.h, k, buf, C.byref(got)), "gsr_get_frame_history")
    st = np.array([[buf[i].stage_ms[j] for j in range(5)] for i in range(got.value)])
    return st, np.array([buf[i].duplicates for i in range(got.value)]), np.array([buf[i].visible for i in range(got.value)])


def run(vols):
    arr = (_lib.GsrCutout * max(1, len(vols)))(*vols)
    _lib.check(c.L.gsr_set_cutouts(c.h, arr, len(vols)), "gsr_set_cutouts")
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
visible = {k: [] for k in CASES}
for r in range(ROUNDS):
    for name, vols in CASES.items():
        st, m, vis = run(vols)
        stages[name].append(st)
        pairs[name].append(m)
        visible[name].append(vis)
    print(f"round {r}: " + "  ".join(f"{k} {np.median(stages[k][-1][:, 0]):.4f}/{np.median(stages[k][-1][:, 4]):.4f} ms" for k in CASES), flush=True)

print(f"median over {ROUNDS} x {F} frames; spread = min..max of the per-round medians")
base = {col: np.median(np.concatenate(stages["none"])[:, j]) for col, j in COLS.items()}
for name in CASES:
    line = [f"  {name:9s}"]
    for col, j in COLS.items():
        allv = np.concatenate(stages[name])[:, j]
        rounds = [np.median(s[:, j]) for s in stages[name]]
        line.append(f"{col} {np.median(allv):.4f} ms ({100 * (np.median(allv) / base[col] - 1):+6.1f} %) spread {min(rounds):.4f}..{max(rounds):.4f}")
    line.append(f"M {np.median(np.concatenate(pairs[name])) / 1e6:.2f} M  V {np.median(np.concatenate(visible[name])) / 1e6:.2f} M")
    print("   ".join(line), flush=True)
c.close()
