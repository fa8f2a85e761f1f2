"""Cost of the compressed PLY (gsr_export_compressed_ply, gsr_upload_compressed_ply) at c3 (6 M splats), for a degree-3 float store and a
degree-3 binary16 store, with gsr_export_ply and gsr_upload_ply of the same cloud beside them.  Export: STORE and MORTON order into
device and page-locked memory, masks not in use.  Upload: the MORTON file from pageable, page-locked and device memory.  Per call: CUDA
events around the call on the context's stream and the host wall time of the whole call.  Cases alternate round by round; medians over
the rounds.  Bandwidth against the byte model of DESIGN.md section 5.24 (export: 504 B read per degree-3 float splat by the decomposition
pass -- 384 for binary16 -- plus the bounds and key passes' 16 + 8 B and the sort's 4 x 16 B per slot, then 61.3 B per splat written;
upload: 61.3 B read and 240 / 144 B written per splat).  The card's name and power limit are read in the same run.
    python ubench/compressed_ply.py [rounds] [workload]"""
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
from godotgaussiansplatting_b200.ply_file import PLY_LAYOUT_3DGS  # noqa: E402
from tests.gsr_direct import Ctx  # noqa: E402

ROUNDS = int(sys.argv[1]) if len(sys.argv) > 1 else 7
wl = dict(bench.WORKLOADS[sys.argv[2] if len(sys.argv) > 2 else "c3"])
n = wl["n"]

try:
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                         timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    gpu = "unknown"
print(f"GPU: {gpu}; workload {wl['desc']}; {ROUNDS} rounds", flush=True)

KEPT = _lib.GSR_EXPORT_KEPT
STORE, MORTON = _lib.GSR_COMPRESS_STORE_ORDER, _lib.GSR_COMPRESS_MORTON
chunks = (n + 255) // 256
FILE_BYTES = chunks * 72 + n * (16 + 45)
stream = torch.cuda.Stream()


def buffers(kind):
    if kind == "device":
        t = [torch.empty((chunks, 18), device="cuda"), torch.empty((n, 4), dtype=torch.int32, device="cuda"),
             torch.empty((n, 45), dtype=torch.uint8, device="cuda")]
        return t, [x.data_ptr() for x in t]
    if kind == "pinned":
        t = [torch.empty((chunks, 18)).pin_memory(), torch.empty((n, 4), dtype=torch.int32).pin_memory(),
             torch.empty((n, 45), dtype=torch.uint8).pin_memory()]
        return t, [x.data_ptr() for x in t]
    t = [np.empty((chunks, 18), np.float32), np.empty((n, 4), np.uint32), np.empty((n, 45), np.uint8)]
    return t, [x.ctypes.data for x in t]


BUF = {k: buffers(k) for k in ("device", "pinned", "pageable")}
PLY_DEV = torch.empty(n * 62, dtype=torch.float32, device="cuda")
PLY_HOST = None


def timed(fn):
    stream.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    e0.record(stream)
    fn()
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1), (time.perf_counter() - t0) * 1e3


for half in (False, True):
    flags = _lib.GSR_FLAG_SH_HALF if half else 0
    ctx, dst_ctx = Ctx(n, 64, 64, flags), Ctx(n, 64, 64, flags)
    for c in (ctx, dst_ctx):
        _lib.check(c.L.gsr_set_stream(c.h, C.c_void_p(stream.cuda_stream)), "gsr_set_stream")
    for lo, blk in bench.raw_chunks(wl):
        ctx.upload_ply_raw(blk, first=lo)
    out = C.c_uint64(0)
    # the MORTON file every upload reads, in each kind of memory
    desc = {}
    for kind, (_, p) in BUF.items():
        d = _lib.GsrCompressedPly(p[0], p[1], p[2], n, chunks, 3, 18)
        _lib.check(ctx.L.gsr_export_compressed_ply(ctx.h, KEPT, -1, MORTON, C.byref(d), C.byref(out)), "export")
        desc[kind] = d
    ply_rows = np.empty((n, 62), np.float32)
    _lib.check(ctx.L.gsr_export_ply(ctx.h, KEPT, -1, C.c_void_p(ply_rows.ctypes.data), n, C.byref(out)), "gsr_export_ply")
    lay = _lib.GsrPlyLayout(*[getattr(PLY_LAYOUT_3DGS, f) for f in ("nprops", "sh_degree", "x", "f_dc", "f_rest", "opacity", "scale", "rot")])

    def export(order, kind):
        _, p = BUF[kind]
        d = _lib.GsrCompressedPly(p[0], p[1], p[2], n, chunks, 3, 18)
        return lambda: _lib.check(ctx.L.gsr_export_compressed_ply(ctx.h, KEPT, -1, order, C.byref(d), C.byref(out)), "export")

    def upload(kind):
        return lambda: _lib.check(dst_ctx.L.gsr_upload_compressed_ply(dst_ctx.h, C.byref(desc[kind]), 0, 0.0), "upload")

    CASES = {
        "export STORE device": export(STORE, "device"),
        "export MORTON device": export(MORTON, "device"),
        "export STORE pinned": export(STORE, "pinned"),
        "export MORTON pinned": export(MORTON, "pinned"),
        "export_ply device": lambda: _lib.check(ctx.L.gsr_export_ply(ctx.h, KEPT, -1, C.c_void_p(PLY_DEV.data_ptr()), n, C.byref(out)), "ply"),
        "upload pageable": upload("pageable"),
        "upload pinned": upload("pinned"),
        "upload device": upload("device"),
        "upload_ply pageable": lambda: _lib.check(dst_ctx.L.gsr_upload_ply(dst_ctx.h, ply_rows.ctypes.data_as(C.POINTER(C.c_float)), C.byref(lay), 0, n,
                                                                           0.0), "upload_ply"),
    }
    names = list(CASES)
    for nm in names:   # warm-up (the first export allocates the scratch)
        timed(CASES[nm])
    times = {nm: [] for nm in names}
    for r in range(ROUNDS):
        for nm in (names if r % 2 == 0 else names[::-1]):
            times[nm].append(timed(CASES[nm]))
    store_read = 384 if half else 504
    store_bytes = 144 if half else 240
    for nm in names:
        ev = float(np.median([t[0] for t in times[nm]]))
        wall = float(np.median([t[1] for t in times[nm]]))
        if nm.startswith("export ") or nm.startswith("upload "):
            b = (n * (store_read + 16 + 8 + 64) + FILE_BYTES) if nm.startswith("export") else (FILE_BYTES + n * store_bytes)
            bw = f"{b / 1e9:6.3f} GB (model) {b / (ev * 1e-3) / 1e9:7.0f} GB/s"
        else:
            bw = ""
        print(f"{'half' if half else 'float'} {nm:24s} {ev:9.3f} ms (events) {wall:9.3f} ms (call)  {bw}", flush=True)
    ctx.close()
    dst_ctx.close()
print(f"file: {FILE_BYTES / n:.1f} B per splat ({FILE_BYTES / 1e9:.3f} GB) against {248} B for the float PLY", flush=True)
