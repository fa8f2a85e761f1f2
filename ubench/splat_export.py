"""Cost of splat export (gsr_export_ply) at c3 (6 M splats), for a degree-3 float store and a degree-3 binary16 store: KEPT with 0 % (the
masks not in use), 10 % and 50 % random and 50 % contiguous hidden, SELECTED at 1 %, at d = 3, and KEPT 10 % at d = 0, into device
memory; KEPT 10 % at d = 3 into page-locked and pageable host memory; and, for the float store, kept_table() -- the host export through
store_to_table -- on the same store and masks.  Per call: CUDA events around the call on the context's stream (its counting pass, the
count's read-back and the writing pass) and the host wall time of the whole call.  Cases alternate round by round; medians over the
rounds.  Achieved bandwidth against the byte model of DESIGN.md section 5.23: 4 ceil(n / 32) mask bytes and 16 B of plane 0 per splat in
scope, both read once per pass, then (2 + P_d) x 16 B read and 4 x row-width bytes written per exported splat.  The card's name and
power limit are read in the same run.
    python ubench/splat_export.py [rounds] [workload]"""
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
from godotgaussiansplatting_b200.rasterizer import pack_mask, store_to_table  # noqa: E402
from tests.gsr_direct import Ctx  # noqa: E402

ROUNDS = int(sys.argv[1]) if len(sys.argv) > 1 else 7
wl = dict(bench.WORKLOADS[sys.argv[2] if len(sys.argv) > 2 else "c3"])
n = wl["n"]
m = n

try:
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                         timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    gpu = "unknown"
print(f"GPU: {gpu}; workload {wl['desc']}; {ROUNDS} rounds", flush=True)

U32P = C.POINTER(C.c_uint32)
KEPT, SELECTED = _lib.GSR_EXPORT_KEPT, _lib.GSR_EXPORT_SELECTED
rng = np.random.default_rng(1)
zero = np.zeros(m, dtype=bool)
block = zero.copy()
block[n // 4:n // 4 + n // 2] = True
r10 = rng.random(m) < 0.10
MASKS = {"none": None, "10% random": (r10, zero), "50% random": (rng.random(m) < 0.5, zero), "50% block": (block, zero),
         "1% selected": (zero, rng.random(m) < 0.01)}
# name: (masks, scope, degree, destination)
CASES = {
    "KEPT 0% d3 device": ("none", KEPT, 3, "device"),
    "KEPT 10% d3 device": ("10% random", KEPT, 3, "device"),
    "KEPT 50% d3 device": ("50% random", KEPT, 3, "device"),
    "KEPT 50% block d3 device": ("50% block", KEPT, 3, "device"),
    "SELECTED 1% d3 device": ("1% selected", SELECTED, 3, "device"),
    "KEPT 10% d0 device": ("10% random", KEPT, 0, "device"),
    "KEPT 10% d3 pinned": ("10% random", KEPT, 3, "pinned"),
    "KEPT 10% d3 pageable": ("10% random", KEPT, 3, "pageable"),
}
packed = {k: None if v is None else (pack_mask(v[0], m), pack_mask(v[1], m)) for k, v in MASKS.items()}
stream = torch.cuda.Stream()
rows_max = n * 62
dst = {"device": torch.empty(rows_max, dtype=torch.float32, device="cuda"), "pinned": torch.empty(rows_max, dtype=torch.float32).pin_memory(),
       "pageable": np.empty(rows_max, dtype=np.float32)}
ptr = {"device": dst["device"].data_ptr(), "pinned": dst["pinned"].data_ptr(), "pageable": dst["pageable"].ctypes.data}


def exported(masks, scope):
    if MASKS[masks] is None:
        return n if scope == KEPT else 0
    hid, sel = MASKS[masks]
    return int((sel[:n] if scope == SELECTED else ~hid[:n]).sum())


def model_bytes(masks, scope, degree, half):
    e = exported(masks, scope)
    K = (degree + 1) ** 2
    P = (3 * K + 7) // 8 if half else (3 * K + 3) // 4
    words = 0 if MASKS[masks] is None else 2 * 4 * ((n + 31) // 32)   # one mask word array per pass
    return words + 2 * 16 * e + e * ((2 + P) * 16 + 4 * (17 + 3 * (K - 1)))   # plane 0 of the splats in scope (none is vacant here)


for half in (False, True):
    ctx = Ctx(m, 64, 64, _lib.GSR_FLAG_SH_HALF if half else 0)
    _lib.check(ctx.L.gsr_set_stream(ctx.h, C.c_void_p(stream.cuda_stream)), "gsr_set_stream")
    for lo, blk in bench.raw_chunks(wl):
        ctx.upload_ply_raw(blk, first=lo)
    store = "half" if half else "float"
    out = C.c_uint64(0)
    current = [object()]

    def set_masks(name):
        if current[0] == name:
            return
        if packed[name] is None:
            _lib.check(ctx.L.gsr_clear_splat_masks(ctx.h), "clear")
        else:
            hw, sw = packed[name]
            _lib.check(ctx.L.gsr_set_splat_masks(ctx.h, hw.ctypes.data_as(U32P), sw.ctypes.data_as(U32P), hw.size), "masks")
        current[0] = name

    def run(name):
        masks, scope, degree, where = CASES[name]
        set_masks(masks)
        stream.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record(stream)
        _lib.check(ctx.L.gsr_export_ply(ctx.h, scope, degree, C.c_void_p(ptr[where]), n, C.byref(out)), "gsr_export_ply")
        e1.record(stream)
        e1.synchronize()
        wall = time.perf_counter() - t0
        assert out.value == exported(masks, scope), (name, out.value)
        return e0.elapsed_time(e1), wall * 1e3

    names = list(CASES)
    for nm in names:   # warm-up
        run(nm)
    times = {nm: [] for nm in names}
    for r in range(ROUNDS):
        for nm in (names if r % 2 == 0 else names[::-1]):
            times[nm].append(run(nm))
    for nm in names:
        masks, scope, degree, where = CASES[nm]
        ev = float(np.median([t[0] for t in times[nm]]))
        wall = float(np.median([t[1] for t in times[nm]]))
        b = model_bytes(masks, scope, degree, half)
        print(f"{store} {nm:26s} {ev:9.3f} ms (events)  {wall:9.3f} ms (call)  {b / 1e9:7.3f} GB (model)  "
              f"{b / (ev * 1e-3) / 1e9:7.0f} GB/s", flush=True)
    if not half:   # kept_table(): copy the store to pageable memory, read the masks, store_to_table
        set_masks("10% random")
        nbytes = int(ctx.L.gsr_splat_store_bytes(ctx.h))
        t0 = time.perf_counter()
        host = np.empty(nbytes // 4, dtype=np.float32)
        _lib.check(ctx.L.gsr_copy_splat_store(ctx.h, C.c_void_p(host.ctypes.data)), "copy")
        words = (m + 31) // 32
        hw, sw = np.zeros(words, np.uint32), np.zeros(words, np.uint32)
        _lib.check(ctx.L.gsr_get_splat_masks(ctx.h, hw.ctypes.data_as(U32P), sw.ctypes.data_as(U32P), words), "masks")
        t1 = time.perf_counter()
        table = store_to_table(host.reshape(-1, (m + 255) // 256 * 256, 4), n, 4, False, MASKS["10% random"][0][:n])
        t2 = time.perf_counter()
        assert table.shape[0] == exported("10% random", KEPT)
        print(f"float kept_table() KEPT 10% d3: {(t2 - t0) * 1e3:9.1f} ms (copy + masks {(t1 - t0) * 1e3:.1f} ms, store_to_table "
              f"{(t2 - t1) * 1e3:.1f} ms), one run", flush=True)
        del host, table
    ctx.close()
