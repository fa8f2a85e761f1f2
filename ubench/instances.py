"""Cost of splat instances (gsr_set_instances) at c3: the projection stage ('Projection' of gsr_get_frame_history: clear + instance
prepare + projection) and the whole frame (sum of the stages) of orbit frames for four cases, alternated round by round in one process:
    off        the default frame
    identity   one identity instance over all N splats: the same picture, so the difference is the pure overhead of the instanced path
    rigid8     8 instances of N/8 splats, each with its own rigid transform (rotation about the cloud's centre + a shift)
    copies4    4 copies of the first N/4 splats side by side (D = N)
The transforms are set again before every frame, as a host that moves its objects would (the transform-only path).
    python ubench/instances.py [frames per case and round] [rounds] [workload]"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

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


def rotation(axis, angle):
    a = np.asarray(axis, dtype=np.float64)
    a = a / np.linalg.norm(a)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(angle) * K + (1 - np.cos(angle)) * (K @ K)


def to_frame(A, t):
    return [float(v) for v in np.concatenate([np.asarray(A).T.reshape(9), np.asarray(t)])]


centre = np.array([0.0, 0.0, 2.5])   # the orbit's centre (frame space)
rng = np.random.default_rng(0)
rigid = []
for k in range(8):
    R = rotation(rng.normal(size=3), rng.uniform(-0.3, 0.3))
    rigid.append(to_frame(R, centre - R @ centre + rng.uniform(-0.2, 0.2, size=3)))
q = n // 4
CASES = {
    "off": [],
    "identity": [(0, n, to_frame(np.eye(3), np.zeros(3)))],
    "rigid8": [(k * (n // 8), n // 8 if k < 7 else n - 7 * (n // 8), rigid[k]) for k in range(8)],
    "copies4": [(0, q, to_frame(np.eye(3), [dx, dy, 0.0])) for dx, dy in ((-0.4, -0.3), (0.4, -0.3), (-0.4, 0.3), (0.4, 0.3))],
}


def set_case(name):
    inst = CASES[name]
    arr = (_lib.GsrInstance * max(1, len(inst)))()
    for k, (first, count, xf) in enumerate(inst):
        arr[k].first, arr[k].count = first, count
        arr[k].to_frame[:] = xf
    _lib.check(ctx.L.gsr_set_instances(ctx.h, arr, len(inst)), "gsr_set_instances")


def history(k):
    buf = (_lib.GsrFrameRecord * k)()
    got = C.c_uint32(0)
    _lib.check(ctx.L.gsr_get_frame_history(ctx.h, k, buf, C.byref(got)), "gsr_get_frame_history")
    return np.array([buf[i].stage_ms[0] for i in range(got.value)]), np.array([buf[i].stage_ms[4] for i in range(got.value)])


def run(name):
    for i in range(10):
        set_case(name)
        ctx.render_async(*frames[i])
    ctx.sync()
    for i in range(10, 10 + F):
        set_case(name)
        ctx.render_async(*frames[i])
    ctx.sync()
    return history(F)


proj = {k: [] for k in CASES}
total = {k: [] for k in CASES}
for r in range(ROUNDS):
    for name in CASES:
        p, t = run(name)
        proj[name].append(p)
        total[name].append(t)
    print(f"round {r}: " + "  ".join(f"{k} {np.median(proj[k][-1]):.4f}/{np.median(total[k][-1]):.4f} ms" for k in CASES), flush=True)

base_p, base_t = np.median(np.concatenate(proj["off"])), np.median(np.concatenate(total["off"]))
print(f"projection stage / frame (sum of stages), median over {ROUNDS} x {F} frames; spread = min..max of the per-round medians")
for name in CASES:
    p, t = np.concatenate(proj[name]), np.concatenate(total[name])
    rp, rt = [np.median(x) for x in proj[name]], [np.median(x) for x in total[name]]
    print(f"  {name:9s} projection {np.median(p):.4f} ms ({100 * (np.median(p) / base_p - 1):+6.1f} %) spread {min(rp):.4f}..{max(rp):.4f}   "
          f"frame {np.median(t):.4f} ms ({100 * (np.median(t) / base_t - 1):+6.1f} %) spread {min(rt):.4f}..{max(rt):.4f}", flush=True)
set_case("off")
ctx.close()
