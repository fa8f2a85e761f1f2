"""Cost of splat delete and duplicate (gsr_delete_hidden, gsr_duplicate_selection) at c3 (6 M splats), for a degree-3 float store and a
degree-3 binary16 store: deletes of a 30 % random, a 30 % contiguous and a 1 % tail-only hidden mask, duplicates of 1 % and 10 % random
selections.  Each round restores the store, masks and count, then times one edit: CUDA events around the edit's kernels on the context's
stream (the event pair brackets the call; its one host synchronisation waits for the same kernels), and the host wall time of the whole
call.  Cases alternate round by round; medians over the rounds.  Achieved bandwidth against the byte model of DESIGN.md section 5.20:
4 ceil(n / 32) mask bytes, plus 2 x 16 (3 + P) bytes per moved splat (kept splats whose index does not change excluded), plus
16 (3 + P) bytes per vacated slot.  The card's name and power limit are read in the same run.
    python ubench/splat_delete.py [rounds] [workload]"""
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
from godotgaussiansplatting_b200.rasterizer import pack_mask  # noqa: E402
from tests.gsr_direct import Ctx  # noqa: E402

ROUNDS = int(sys.argv[1]) if len(sys.argv) > 1 else 7
wl = dict(bench.WORKLOADS[sys.argv[2] if len(sys.argv) > 2 else "c3"])
n = wl["n"]
m = n + n // 8

try:
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                         timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    gpu = "unknown"
print(f"GPU: {gpu}; workload {wl['desc']}; {ROUNDS} rounds", flush=True)

U32P = C.POINTER(C.c_uint32)
rng = np.random.default_rng(1)
zero = np.zeros(m, dtype=bool)
block = zero.copy()
block[n // 3:n // 3 + (3 * n) // 10] = True
tail = zero.copy()
tail[n - n // 100:n] = rng.random(n // 100) < 0.5   # a few floaters near the end: 0.5 % of the cloud, in its last 1 %
CASES = {
    "delete 30% random": ("delete", rng.random(m) < 0.3, zero),
    "delete 30% block": ("delete", block, zero),
    "delete 1% tail": ("delete", tail, zero),
    "duplicate 1%": ("duplicate", zero, rng.random(m) < 0.01),
    "duplicate 10%": ("duplicate", zero, rng.random(m) < 0.10),
}
for name, (op, hid, sel) in CASES.items():
    hid[n:], sel[n:] = False, False
    CASES[name] = (op, hid, sel & ~hid, pack_mask(hid, m), pack_mask(sel & ~hid, m))
stream = torch.cuda.Stream()


def model_bytes(op, hid, sel, planes):
    words = 4 * ((n + 31) // 32)
    if op == "delete":
        h = hid[:n]
        first = int(np.argmax(h)) if h.any() else n
        moved = int((~h[first:]).sum())
        return words + moved * 2 * 16 * planes + int(h.sum()) * 16 * planes
    return words + int(sel[:n].sum()) * 2 * 16 * planes


for half in (False, True):
    ctx = Ctx(m, 64, 64, _lib.GSR_FLAG_SH_HALF if half else 0)
    _lib.check(ctx.L.gsr_set_stream(ctx.h, C.c_void_p(stream.cuda_stream)), "gsr_set_stream")
    for lo, blk in bench.raw_chunks(wl):
        ctx.upload_ply_raw(blk, first=lo)
    nbytes = int(ctx.L.gsr_splat_store_bytes(ctx.h))
    planes = nbytes // (16 * ((m + 255) // 256 * 256))
    snap = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    _lib.check(ctx.L.gsr_copy_splat_store(ctx.h, C.c_void_p(snap.data_ptr())), "copy")
    store = "half" if half else "float"
    out = C.c_uint64(0)

    def run(name):
        op, hid, sel, hw, sw = CASES[name]
        _lib.check(ctx.L.gsr_restore_splat_store(ctx.h, C.c_void_p(snap.data_ptr())), "restore")
        _lib.check(ctx.L.gsr_set_splat_masks(ctx.h, hw.ctypes.data_as(U32P), sw.ctypes.data_as(U32P), hw.size), "masks")
        _lib.check(ctx.L.gsr_set_splat_count(ctx.h, n), "count")
        stream.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record(stream)
        fn = ctx.L.gsr_delete_hidden if op == "delete" else ctx.L.gsr_duplicate_selection
        _lib.check(fn(ctx.h, C.byref(out)), op)
        e1.record(stream)
        e1.synchronize()
        wall = time.perf_counter() - t0
        return e0.elapsed_time(e1), wall * 1e3

    names = list(CASES)
    for nm in names:   # warm-up
        run(nm)
    times = {nm: [] for nm in names}
    for r in range(ROUNDS):
        for nm in (names if r % 2 == 0 else names[::-1]):
            times[nm].append(run(nm))
    for nm in names:
        op, hid, sel, _, _ = CASES[nm]
        ev = float(np.median([t[0] for t in times[nm]]))
        wall = float(np.median([t[1] for t in times[nm]]))
        b = model_bytes(op, hid, sel, planes)
        print(f"{store} {nm:20s} {ev * 1e3:9.1f} us (events)  {wall * 1e3:9.1f} us (call)  {b / 1e9:7.3f} GB (model)  "
              f"{b / (ev * 1e-3) / 1e9:7.0f} GB/s", flush=True)
    ctx.close()
