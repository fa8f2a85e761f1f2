"""Cost of selection colour edits (gsr_recolor_selection) at c3 (6 M splats), for a degree-3 float store and a degree-3 binary16 store:
1 %, 10 % and 100 % of the splats selected, the edit in place and from a device snapshot.  Kernel time from CUDA events around
`launches` back-to-back calls on the context's stream after a warm-up, the cases alternated round by round, medians over the rounds.
Achieved bandwidth against the byte model of DESIGN.md section 5.19: 4 ceil(N / 32) mask bytes plus, per selected splat,
2 x 16 (1 + P) bytes in place (plane 2 and the SH planes) or 2 x 16 (3 + P) bytes from a snapshot (every plane).  The card's name and
power limit are read in the same run.
    python ubench/selection_color.py [launches per case and round] [rounds] [workload]"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from godotgaussiansplatting_b200 import _lib  # noqa: E402
from godotgaussiansplatting_b200.rasterizer import color_edit, pack_mask  # noqa: E402
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
EDIT = color_edit(gain=(1.02, 1.0, 0.98), saturation=1.01, view_dependence=0.99, opacity=0.99)   # a small grade: values stay in range
rng = np.random.default_rng(1)
FRACTIONS = (0.01, 0.10, 1.00)
SELECTIONS = {f: pack_mask(rng.random(n) < f, n) for f in FRACTIONS}
stream = torch.cuda.Stream()


def measure(call):
    for _ in range(5):
        call()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(LAUNCHES):
        call()
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) / LAUNCHES


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
    cases = [(f"{store} {int(f * 100)}% {src}", f, src) for f in FRACTIONS for src in ("in place", "snapshot")]

    def run(case):
        _, f, src = case
        sel = SELECTIONS[f]
        _lib.check(ctx.L.gsr_set_splat_masks(ctx.h, empty.ctypes.data_as(U32P), sel.ctypes.data_as(U32P), sel.size), "masks")
        ptr = None if src == "in place" else C.c_void_p(snap.data_ptr())
        return measure(lambda: _lib.check(ctx.L.gsr_recolor_selection(ctx.h, C.byref(EDIT), ptr), "recolour"))

    times = {c[0]: [] for c in cases}
    for r in range(ROUNDS):
        for case in (cases if r % 2 == 0 else cases[::-1]):
            times[case[0]].append(run(case))
    words = (n + 31) // 32
    for name, f, src in cases:
        ms = float(np.median(times[name]))
        sel = int(np.unpackbits(SELECTIONS[f].view(np.uint8)).sum())
        per_splat = 2 * 16 * ((planes - 2) if src == "in place" else planes)   # in place: plane 2 and the P SH planes
        moved = 4 * words + sel * per_splat
        print(f"{name:28s} {ms * 1e3:9.1f} us   {moved / 1e9:7.3f} GB (model)   {moved / (ms * 1e-3) / 1e9:7.0f} GB/s", flush=True)
    ctx.close()
