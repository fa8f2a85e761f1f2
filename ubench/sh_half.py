"""Cost and precision of the binary16 SH store (GSR_FLAG_SH_HALF) at c3: the projection stage ('Projection' of gsr_get_frame_history: clear +
projection) and the whole frame (sum of the stages) of orbit frames for five cases, alternated round by round in one process:
    float4      the default context: 4 bands stored as float32 (240 B per splat)
    half4       4 bands stored as binary16 (144 B per splat)
    float3      3 bands stored as float32 (160 B per splat) of the degree-2 cloud
    half3       3 bands stored as binary16 (112 B per splat) of the degree-2 cloud
    half4_deg2  the half4 context rendered at degree 2 (gsr_set_sh_degree)
Then the precision cost: max and mean |dRGBA| between the half4 frame and the float4 frame of the same (unrounded) cloud.
    python ubench/sh_half.py [frames per case and round] [rounds] [workload]"""
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


class StoreCtx(Ctx):
    def __init__(self, bands, flags):
        self.L = _lib.lib()
        self.h = C.c_void_p()
        _lib.check(self.L.gsr_create(C.byref(_lib.GsrConfig(0, flags, n, 10, bands)), C.byref(self.h)), "gsr_create")
        self.max_splats, self.w, self.hgt = n, w, h
        _lib.check(self.L.gsr_resize(self.h, w, h), "gsr_resize")


HALF = _lib.GSR_FLAG_SH_HALF
STORES = {"float4": (4, 0), "half4": (4, HALF), "float3": (3, 0), "half3": (3, HALF)}
ctxs = {}
for name, (bands, flags) in STORES.items():
    c = StoreCtx(bands, flags)
    for lo, blk in synthetic_ply_chunks(n, wl["seed"], sh_degree=bands - 1):
        c.upload_ply_raw(blk, first=lo)
    ctxs[name] = c
frames = bench.frame_params(wl, F + 10)
stride = (n + 255) // 256 * 256
CASES = {"float4": ("float4", -1), "half4": ("half4", -1), "float3": ("float3", -1), "half3": ("half3", -1), "half4_deg2": ("half4", 2)}


def store_bytes(name):
    bands, flags = STORES[name]
    p = (3 * bands * bands + 7) // 8 if flags & HALF else (3 * bands * bands + 3) // 4
    return 16 * (3 + p) * stride


def history(c, k):
    buf = (_lib.GsrFrameRecord * k)()
    got = C.c_uint32(0)
    _lib.check(c.L.gsr_get_frame_history(c.h, k, buf, C.byref(got)), "gsr_get_frame_history")
    return np.array([buf[i].stage_ms[0] for i in range(got.value)]), np.array([buf[i].stage_ms[4] for i in range(got.value)])


def run(name):
    store, degree = CASES[name]
    c = ctxs[store]
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

base_p, base_t = np.median(np.concatenate(proj["float4"])), np.median(np.concatenate(total["float4"]))
print(f"projection stage / frame (sum of stages), median over {ROUNDS} x {F} frames; spread = min..max of the per-round medians")
for name in CASES:
    p, t = np.concatenate(proj[name]), np.concatenate(total[name])
    rp, rt = [np.median(x) for x in proj[name]], [np.median(x) for x in total[name]]
    print(f"  {name:10s} store {store_bytes(CASES[name][0]) / 1e9:.3f} GB  projection {np.median(p):.4f} ms ({100 * (np.median(p) / base_p - 1):+6.1f} %) "
          f"spread {min(rp):.4f}..{max(rp):.4f}   frame {np.median(t):.4f} ms ({100 * (np.median(t) / base_t - 1):+6.1f} %) "
          f"spread {min(rt):.4f}..{max(rt):.4f}", flush=True)

# precision: the binary16 store against the float store of the same cloud, at degree 3, over a few orbit frames
dmax, dsum, cnt = 0.0, 0.0, 0
for name in ("float4", "half4"):
    _lib.check(ctxs[name].L.gsr_set_sh_degree(ctxs[name].h, -1), "gsr_set_sh_degree")
for i in (0, F // 3, 2 * F // 3):
    a = ctxs["half4"].render(*frames[i])
    b = ctxs["float4"].render(*frames[i])
    d = np.abs(a.astype(np.float64) - b.astype(np.float64))
    dmax, dsum, cnt = max(dmax, float(d.max())), dsum + float(d.sum()), cnt + d.size
print(f"precision: |dRGBA| of the half4 frame against the float4 frame of the unrounded cloud over 3 frames: max {dmax:.3g}, mean {dsum / cnt:.3g} "
      f"(RGBA in [0, 1]; 1/255 = {1 / 255:.3g})", flush=True)
for c in ctxs.values():
    c.close()
