"""Cost of selection transform edits (gsr_transform_selection) and store snapshots at c3 (6 M splats), for a degree-3 float store and a
degree-3 binary16 store: 1 %, 10 % and 100 % of the splats selected, the edit in place and from a device snapshot, and the snapshot
copy and restore.  Kernel time from CUDA events around `launches` back-to-back calls on the context's stream after a warm-up, the
cases alternated round by round, medians over the rounds.  Achieved bandwidth against the byte model of DESIGN.md section 5.18:
4 ceil(N / 32) mask bytes plus 2 x 16 (3 + P) bytes per selected splat; a snapshot copy or restore moves 2 x the store.  The card's
name and power limit are read in the same run.
    python ubench/selection_transform.py [launches per case and round] [rounds] [workload]"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from godotgaussiansplatting_b200 import _lib  # noqa: E402
from godotgaussiansplatting_b200.rasterizer import pack_mask  # noqa: E402
from tests.gsr_direct import Ctx  # noqa: E402

LAUNCHES = int(sys.argv[1]) if len(sys.argv) > 1 else 50
ROUNDS = int(sys.argv[2]) if len(sys.argv) > 2 else 5
wl = dict(bench.WORKLOADS[sys.argv[3] if len(sys.argv) > 3 else "c3"])
n = wl["n"]

try:
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                         timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    gpu = "unknown"
print(f"GPU: {gpu}; workload {wl['desc']}; {LAUNCHES} launches per case per round, {ROUNDS} rounds", flush=True)

U32P = C.POINTER(C.c_uint32)
FP = C.POINTER(C.c_float)
a = np.deg2rad(0.5)
EDIT = np.array([np.cos(a), np.sin(a), 0, -np.sin(a), np.cos(a), 0, 0, 0, 1, 0.001, 0, 0], dtype=np.float32)   # a small rotation
rng = np.random.default_rng(1)
FRACTIONS = (0.01, 0.10, 1.00)
SELECTIONS = {f: pack_mask(rng.random(n) < f, n) for f in FRACTIONS}
stream = torch.cuda.Stream()


def measure(ctx, call):
    for _ in range(5):
        call()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(LAUNCHES):
        call()
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) / LAUNCHES


results = {}
for half in (False, True):
    ctx = Ctx(n, 64, 64, _lib.GSR_FLAG_SH_HALF if half else 0)
    _lib.check(ctx.L.gsr_set_stream(ctx.h, C.c_void_p(stream.cuda_stream)), "gsr_set_stream")
    for lo, blk in bench.raw_chunks(wl):
        ctx.upload_ply_raw(blk, first=lo)
    nbytes = int(ctx.L.gsr_splat_store_bytes(ctx.h))
    planes = nbytes // (16 * ((n + 255) // 256 * 256))
    snap = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    _lib.check(ctx.L.gsr_copy_splat_store(ctx.h, C.c_void_p(snap.data_ptr())), "copy")
    empty = np.zeros_like(SELECTIONS[1.0])
    store = "half" if half else "float"
    cases = []
    for f in FRACTIONS:
        for src in ("in place", "snapshot"):
            cases.append((f"{store} {int(f * 100)}% {src}", f, src))
    cases += [(f"{store} copy", None, "copy"), (f"{store} restore", None, "restore")]

    def run(case):
        _, f, src = case
        if f is not None:
            sel = SELECTIONS[f]
            _lib.check(ctx.L.gsr_set_splat_masks(ctx.h, empty.ctypes.data_as(U32P), sel.ctypes.data_as(U32P), sel.size), "masks")
            ptr = None if src == "in place" else C.c_void_p(snap.data_ptr())
            return measure(ctx, lambda: _lib.check(ctx.L.gsr_transform_selection(ctx.h, EDIT.ctypes.data_as(FP), ptr), "transform"))
        fn = ctx.L.gsr_copy_splat_store if src == "copy" else ctx.L.gsr_restore_splat_store
        return measure(ctx, lambda: _lib.check(fn(ctx.h, C.c_void_p(snap.data_ptr())), src))

    times = {c[0]: [] for c in cases}
    for r in range(ROUNDS):
        order = cases if r % 2 == 0 else cases[::-1]
        for case in order:
            times[case[0]].append(run(case))
    words = (n + 31) // 32
    for name, f, src in cases:
        ms = float(np.median(times[name]))
        if f is None:
            moved = 2 * nbytes
        else:
            sel = int(np.unpackbits(SELECTIONS[f].view(np.uint8)).sum())
            moved = 4 * words + sel * 2 * 16 * planes
        results[name] = (ms, moved)
        print(f"{name:28s} {ms * 1e3:9.1f} us   {moved / 1e9:7.3f} GB (model)   {moved / (ms * 1e-3) / 1e9:7.0f} GB/s", flush=True)
    ctx.close()
