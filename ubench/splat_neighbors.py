"""Cost of splat neighbourhood selection (gsr_select_neighborhood) at c3 size (6 M splats): a shell of radius 5 and thickness 0.1 with
floaters and clumps, as in tests/test_gpu_splat_neighbors.py.  Radii that give a mean of about 8, 32 and 128 neighbours in the shell,
and one near the candidate limit.  Each case times one call per round: CUDA events around it on the context's stream, and the host wall
time of the whole call (it synchronises for the budget and for the stats).  Cases alternate round by round; medians over the rounds.
Then one profiled round (torch.profiler, CUDA activities) splits each call into its stages by kernel name: grid build (keys, the sort,
the gather and the impure marks), budget, query (SPARSE / GROW), union-find (union and compress) and the mask words.  The byte model
of DESIGN.md section 5.22 is printed beside each stage.  The card's name and power limit are read in the same run.
    python ubench/splat_neighbors.py [rounds]"""
import ctypes as C
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from godotgaussiansplatting_b200 import _lib  # noqa: E402
from tests.gsr_direct import Ctx  # noqa: E402

ROUNDS = int(sys.argv[1]) if len(sys.argv) > 1 else 5
N = 6_000_000
try:
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                         timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    gpu = "unknown"
print(f"GPU: {gpu}; {N} splats; {ROUNDS} rounds", flush=True)

rng = np.random.default_rng(1)
body = N - 3000 - 400 * 30
d = rng.normal(size=(body, 3))
d /= np.linalg.norm(d, axis=1, keepdims=True)
pts = [d * rng.uniform(4.95, 5.05, (body, 1)), rng.uniform(-15, 15, (3000, 3))]
pts += [rng.uniform(-15, 15, 3) + rng.normal(size=(30, 3)) * 0.01 for _ in range(400)]
xyz = np.concatenate(pts).astype(np.float32)[rng.permutation(N)]

L = _lib.lib()
c = Ctx(N, 64, 64)
nbytes = int(L.gsr_splat_store_bytes(c.h))
store = np.zeros(nbytes // 4, np.float32).reshape(15, -1, 4)
store[0, :N, :3] = xyz
_lib.check(L.gsr_restore_splat_store(c.h, C.c_void_p(store.ctypes.data)), "restore")
_lib.check(L.gsr_set_splat_count(c.h, N), "count")
c.sync()
words = (N + 31) // 32
sel = np.zeros(words, np.uint32)
sel[::1000] = 1
hid = np.zeros(words, np.uint32)
U32P = C.POINTER(C.c_uint32)


def call(mode, radius, count):
    _lib.check(L.gsr_set_splat_masks(c.h, hid.ctypes.data_as(U32P), sel.ctypes.data_as(U32P), words), "masks")
    c.sync()
    q = _lib.GsrNeighborhood(mode, radius, count, -1)
    st = _lib.GsrNeighborhoodStats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    e0.record()
    rc = L.gsr_select_neighborhood(c.h, C.byref(q), 0, C.byref(st))
    e1.record()
    e1.synchronize()
    wall = time.perf_counter() - t0
    return rc, e0.elapsed_time(e1), wall * 1e3, st


S, G, CC, SM = range(4)
cases = []
for r, tag in ((0.0215, "~8"), (0.0341, "~32"), (0.0541, "~128")):
    cases += [(f"SPARSE r={r} ({tag} nbrs)", S, r, 4), (f"GROW r={r}", G, r, 1), (f"CONNECTED r={r}", CC, r, 1),
              (f"SMALL_CLUSTERS r={r}", SM, r, 200)]
cases.append(("SPARSE r=0.08 (near the limit)", S, 0.08, 4))
cases.append(("GROW r=100 (over the limit: refused)", G, 100.0, 1))
for name, mode, r, k in cases:   # warm every case
    call(mode, r, k)
res = {name: ([], []) for name, *_ in cases}
stats = {}
for _ in range(ROUNDS):
    for name, mode, r, k in cases:
        rc, ev, wall, st = call(mode, r, k)
        res[name][0].append(ev)
        res[name][1].append(wall)
        stats[name] = (rc, st.participants, st.inside, st.candidates, st.clusters, st.largest_cluster)
print(f"{'case':42s} {'events ms':>10s} {'wall ms':>9s}  rc participants inside candidates clusters largest")
for name, *_ in cases:
    ev, wall = res[name]
    print(f"{name:42s} {np.median(ev):10.3f} {np.median(wall):9.3f}  {stats[name]}")

# one profiled round: the stages by kernel name
STAGES = [("grid build", ("neighbor_keys", "sort_hist", "onesweep", "neighbor_grid", "neighbor_impure")), ("budget", ("neighbor_budget",)),
          ("query", ("neighbor_query",)), ("union-find", ("neighbor_union", "neighbor_compress")), ("mask words", ("neighbor_combine",))]
from torch.profiler import ProfilerActivity, profile  # noqa: E402
for name, mode, r, k in cases[:-1]:
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call(mode, r, k)
    t = {s: 0.0 for s, _ in STAGES}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        for s, keys in STAGES:
            if any(key in e.name for key in keys):
                t[s] += e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
    n, cand = stats[name][1], stats[name][3]
    model = {"grid build": 8 * 4 * n + 32 * n, "budget": 27 * 12 * n, "query": 16 * cand, "union-find": 16 * cand, "mask words": 12 * N / 32}
    print(f"{name:42s} " + "  ".join(f"{s} {t[s]:.3f} ms ({model[s] / max(t[s], 1e-9) / 1e6:.0f} GB/s model)" for s, _ in STAGES if t[s] > 0))
c.close()
