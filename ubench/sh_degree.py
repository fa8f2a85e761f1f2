"""Cost of the SH degree (gsr_config.sh_bands, gsr_set_sh_degree) at c3: the projection stage ('Projection' of gsr_get_frame_history: clear +
projection) and the whole frame (sum of the stages) of orbit frames for seven cases, alternated round by round in one process:
    default     the default context (4 bands stored, degree 3 rendered)
    store1..3   a context that stores 1, 2 or 3 bands (64 / 96 / 160 B per splat) of synthetic_ply_table(..., sh_degree = bands - 1)
    deg0..2     the default context rendered at degree 0, 1 or 2 (gsr_set_sh_degree)
The degree-d clouds are the same splats (seed of the workload) with the coefficients above d set to zero.
    python ubench/sh_degree.py [frames per case and round] [rounds] [workload]"""
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


class BandsCtx(Ctx):
    def __init__(self, bands):
        self.L = _lib.lib()
        self.h = C.c_void_p()
        _lib.check(self.L.gsr_create(C.byref(_lib.GsrConfig(0, 0, n, 10, bands)), C.byref(self.h)), "gsr_create")
        self.max_splats, self.w, self.hgt = n, w, h
        _lib.check(self.L.gsr_resize(self.h, w, h), "gsr_resize")


ctxs = {}
for bands in (0, 1, 2, 3):
    c = BandsCtx(bands)
    for lo, blk in synthetic_ply_chunks(n, wl["seed"], sh_degree=(bands or 4) - 1):
        c.upload_ply_raw(blk, first=lo)
    ctxs[bands] = c
frames = bench.frame_params(wl, F + 10)
stride = (n + 255) // 256 * 256
CASES = {"default": (0, -1), "store1": (1, -1), "store2": (2, -1), "store3": (3, -1), "deg0": (0, 0), "deg1": (0, 1), "deg2": (0, 2)}


def history(c, k):
    buf = (_lib.GsrFrameRecord * k)()
    got = C.c_uint32(0)
    _lib.check(c.L.gsr_get_frame_history(c.h, k, buf, C.byref(got)), "gsr_get_frame_history")
    return np.array([buf[i].stage_ms[0] for i in range(got.value)]), np.array([buf[i].stage_ms[4] for i in range(got.value)])


def run(name):
    bands, degree = CASES[name]
    c = ctxs[bands]
    _lib.check(c.L.gsr_set_sh_degree(c.h, degree), "gsr_set_sh_degree")
    for i in range(10):
        c.render_async(*frames[i])
    c.sync()
    for i in range(10, 10 + F):
        c.render_async(*frames[i])
    c.sync()
    return history(c, F)


proj = {k: [] for k in CASES}
total = {k: [] for k in CASES}
for r in range(ROUNDS):
    for name in CASES:
        p, t = run(name)
        proj[name].append(p)
        total[name].append(t)
    print(f"round {r}: " + "  ".join(f"{k} {np.median(proj[k][-1]):.4f}/{np.median(total[k][-1]):.4f} ms" for k in CASES), flush=True)

base_p, base_t = np.median(np.concatenate(proj["default"])), np.median(np.concatenate(total["default"]))
print(f"projection stage / frame (sum of stages), median over {ROUNDS} x {F} frames; spread = min..max of the per-round medians")
for name in CASES:
    bands, degree = CASES[name]
    soa = 16 * (3 + (3 * (bands or 4) ** 2 + 3) // 4) * stride
    p, t = np.concatenate(proj[name]), np.concatenate(total[name])
    rp, rt = [np.median(x) for x in proj[name]], [np.median(x) for x in total[name]]
    print(f"  {name:8s} soa {soa / 1e9:.3f} GB  projection {np.median(p):.4f} ms ({100 * (np.median(p) / base_p - 1):+6.1f} %) spread {min(rp):.4f}..{max(rp):.4f}   "
          f"frame {np.median(t):.4f} ms ({100 * (np.median(t) / base_t - 1):+6.1f} %) spread {min(rt):.4f}..{max(rt):.4f}", flush=True)
for c in ctxs.values():
    c.close()
