"""Cost of splat property selection (gsr_select_where) and property histograms (gsr_splat_histogram) at c3 (6 M splats), for a degree-3
float store and a degree-3 binary16 store.  select_where: opacity alone, size + isotropy, colour distance, and a set of 8 filters.
Histograms of opacity at 64, 256 and 1024 bins on the trained (spread) opacities and on saturated ones (every opacity set to 1 with
gsr_recolor_selection, so every splat lands in one bin), and of size on log-spaced edges; one histogram of a cloud of one splat gives
the call's fixed cost (the upload of the counters and edges, the launch, one CTA's flush, the read-back).  Each case times one call:
CUDA events around it on the context's stream, and the host wall time of the whole call (a histogram synchronises once; select_where
is followed by an event synchronise).  Cases alternate round by round; medians over the rounds.  Achieved bandwidth against the byte
model of DESIGN.md section 5.21: 16 B of plane 0 plus 16 B per further plane the set reads, for every tested splat (an upper bound
for a multi-filter set, whose later planes only survivors read), plus the mask words (select_where: 12 B per 32 splats; histogram:
4 B per 32).  The card's name and power limit are read in the same run.
    python ubench/splat_properties.py [rounds] [workload]"""
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
from godotgaussiansplatting_b200.rasterizer import splat_filter  # noqa: E402
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

P = _lib
INF = float("inf")
WHERE = {
    "where opacity": [(P.GSR_PROP_OPACITY, 0.0, 0.1)],
    "where size+isotropy": [(P.GSR_PROP_SIZE, 1e-3, INF), (P.GSR_PROP_ISOTROPY, -INF, 0.2)],
    "where colour": [(P.GSR_PROP_COLOR_DISTANCE, 0.0, 0.05, (0.1, 0.6, 0.2))],
    "where 8 filters": [(P.GSR_PROP_OPACITY, 0.05, 1.0), (P.GSR_PROP_SIZE, 0.0, 10.0), (P.GSR_PROP_VOLUME, -INF, 1.0),
                        (P.GSR_PROP_ISOTROPY, 0.01, 1.0), (P.GSR_PROP_COLOR_DISTANCE, 0.0, 2.0, (0.5, 0.5, 0.5)),
                        (P.GSR_PROP_OPACITY, 0.1, 1.0), (P.GSR_PROP_SIZE, 1e-6, 5.0), (P.GSR_PROP_COLOR_DISTANCE, 0.0, 1.5, (0.2, 0.2, 0.2))],
}
HIST = {f"hist opacity {b} {kind}": (P.GSR_PROP_OPACITY, np.linspace(0.0, 1.0, b + 1).astype(np.float32), kind == "saturated")
        for kind in ("spread", "saturated") for b in (64, 256, 1024)}
HIST["hist size 256 log"] = (P.GSR_PROP_SIZE, np.geomspace(1e-6, 10.0, 257).astype(np.float32), False)
HIST["hist opacity 256 one splat"] = (P.GSR_PROP_OPACITY, np.linspace(0.0, 1.0, 257).astype(np.float32), False)   # the call's fixed cost


def planes_of(props):
    bits = 0
    for p in props:
        bits |= 2 if p == P.GSR_PROP_OPACITY else 4 if p == P.GSR_PROP_COLOR_DISTANCE else 3
    return bin(bits).count("1")


def model_bytes(name):
    if name in WHERE:
        return n * 16 * (1 + planes_of([f[0] for f in WHERE[name]])) + 12 * ((m + 31) // 32)
    k = 1 if "one splat" in name else n
    return k * 16 * (1 + planes_of([HIST[name][0]])) + 4 * ((k + 31) // 32)


stream = torch.cuda.Stream()
for half in (False, True):
    ctx = Ctx(m, 64, 64, _lib.GSR_FLAG_SH_HALF if half else 0)
    _lib.check(ctx.L.gsr_set_stream(ctx.h, C.c_void_p(stream.cuda_stream)), "gsr_set_stream")
    for lo, blk in bench.raw_chunks(wl):
        ctx.upload_ply_raw(blk, first=lo)
    nbytes = int(ctx.L.gsr_splat_store_bytes(ctx.h))
    spread = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    saturated = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    _lib.check(ctx.L.gsr_copy_splat_store(ctx.h, C.c_void_p(spread.data_ptr())), "copy")
    _lib.check(ctx.L.gsr_select_all(ctx.h, P.GSR_SELECT_SET), "select all")
    sat = _lib.GsrColorEdit()
    sat.matrix[:] = [1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0]
    sat.band_scale[:] = [1, 1, 1]
    sat.opacity_scale, sat.opacity_offset = 0.0, 1.0
    _lib.check(ctx.L.gsr_recolor_selection(ctx.h, C.byref(sat), None), "saturate")
    _lib.check(ctx.L.gsr_copy_splat_store(ctx.h, C.c_void_p(saturated.data_ptr())), "copy")
    _lib.check(ctx.L.gsr_clear_splat_masks(ctx.h), "clear")
    stream.synchronize()
    store = "half" if half else "float"
    filters = {k: (_lib.GsrSplatFilter * len(v))(*[splat_filter(*f) for f in v]) for k, v in WHERE.items()}
    counts = np.zeros(1024 + 3, dtype=np.uint64)
    mm = np.zeros(2, dtype=np.float32)
    state = {"sat": None}

    def run(name):
        if name in HIST:
            want = HIST[name][2]
            if state["sat"] != want:
                _lib.check(ctx.L.gsr_restore_splat_store(ctx.h, C.c_void_p((saturated if want else spread).data_ptr())), "restore")
                state["sat"] = want
        _lib.check(ctx.L.gsr_set_splat_count(ctx.h, 1 if "one splat" in name else n), "count")
        stream.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record(stream)
        if name in WHERE:
            _lib.check(ctx.L.gsr_select_where(ctx.h, filters[name], len(WHERE[name]), -1, P.GSR_SELECT_SET), name)
        else:
            prop, e, _ = HIST[name]
            f = splat_filter(prop)
            _lib.check(ctx.L.gsr_splat_histogram(ctx.h, C.byref(f), -1, P.GSR_HISTOGRAM_KEPT, e.ctypes.data_as(C.POINTER(C.c_float)),
                                                 e.size - 1, counts.ctypes.data_as(C.POINTER(C.c_uint64)),
                                                 mm.ctypes.data_as(C.POINTER(C.c_float))), name)
        e1.record(stream)
        e1.synchronize()
        wall = time.perf_counter() - t0
        return e0.elapsed_time(e1), wall * 1e3

    names = list(WHERE) + list(HIST)
    for nm in names:   # warm-up
        run(nm)
    times = {nm: [] for nm in names}
    for r in range(ROUNDS):
        for nm in (names if r % 2 == 0 else names[::-1]):
            times[nm].append(run(nm))
    for nm in names:
        ev = float(np.median([t[0] for t in times[nm]]))
        wall = float(np.median([t[1] for t in times[nm]]))
        b = model_bytes(nm)
        print(f"{store} {nm:28s} {ev * 1e3:9.1f} us (events)  {wall * 1e3:9.1f} us (call)  {b / 1e9:7.3f} GB (model)  "
              f"{b / (ev * 1e-3) / 1e9:7.0f} GB/s", flush=True)
    ctx.close()
