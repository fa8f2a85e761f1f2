"""Reference implementation of splat neighbourhood selection (include/gsr.h "Splat neighbourhood selection") for the tests.

TEST INFRASTRUCTURE.  Three parts:
  1. the rule in numpy float32 by brute force (every pair, in row blocks) for clouds up to about 20 k splats: participants, neighbours
     d2 = ((dx dx) + (dy dy)) + (dz dz) <= r2, clusters by a plain host union-find over those edges, and `candidates` from the float64
     cell rule;
  2. a serial C++ reference with a plain grid and a disjoint-set forest (tests/neighbor_reference/neighbor_emu.cpp, ref_*) for the large
     clouds, itself checked against part 1;
  3. the CPU kernel emulator of csrc/neighbors.cu (the same file, emu_*), launched like gsr_select_neighborhood.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from godotgaussiansplatting_b200.rasterizer import pack_mask, unpack_mask
from tests import cutout_reference as cr
from tests import selection_reference as sref

F32 = np.float32
HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "neighbor_reference")
SPARSE, GROW, CONNECTED, SMALL = range(4)
MODES = [SPARSE, GROW, CONNECTED, SMALL]
LIMIT = 1 << 34
_emu = None


# ---- the rule ---------------------------------------------------------------------------------------------------------------
def participants(plane0, hidden, first, count):
    """bool over the slots of plane0 (max_splats, 4): in [first, first + count), not hidden, x y z finite."""
    m = plane0.shape[0]
    idx = np.arange(m)
    h = np.zeros(m, bool)
    h[:len(hidden)] = hidden
    return (idx >= first) & (idx < first + count) & ~h & np.isfinite(plane0[:, :3]).all(axis=1)


def cells(xyz, radius):
    """floor(v / h) per axis in float64, clamped to [-2^62, 2^62]; h = radius (1 + 2^-20)."""
    h = float(F32(radius)) * (1.0 + 2.0 ** -20)
    with np.errstate(all="ignore"):
        q = np.floor(xyz.astype(np.float64) / h)
    return np.clip(q, -2.0 ** 62, 2.0 ** 62).astype(np.int64)


def candidates(xyz, part, radius):
    """The sum over participants of the participants of the 27 cells around its own."""
    c = cells(xyz[part], radius)
    occ = {}
    for t in map(tuple, c):
        occ[t] = occ.get(t, 0) + 1
    total = 0
    offs = [(dx, dy, dz) for dz in (-1, 0, 1) for dy in (-1, 0, 1) for dx in (-1, 0, 1)]
    for (x, y, z), k in occ.items():
        total += k * sum(occ.get((x + dx, y + dy, z + dz), 0) for dx, dy, dz in offs)
    return total


def edges(xyz, part, radius, block=512):
    """(i, j) slot pairs, i < j, of neighbouring participants, by brute force in float32."""
    idx = np.flatnonzero(part)
    p = np.ascontiguousarray(xyz[idx], dtype=F32)
    r2 = F32(radius) * F32(radius)
    I, J = [], []
    with np.errstate(all="ignore"):
        for b0 in range(0, len(idx), block):
            a = p[b0:b0 + block]
            d = [p[None, :, k] - a[:, None, k] for k in range(3)]   # x_j - x_i
            d2 = ((d[0] * d[0]) + (d[1] * d[1])) + (d[2] * d[2])
            ii, jj = np.nonzero(d2 <= r2)
            ii = ii + b0
            keep = ii < jj
            I.append(idx[ii[keep]])
            J.append(idx[jj[keep]])
    return (np.concatenate(I) if I else np.zeros(0, np.int64)), (np.concatenate(J) if J else np.zeros(0, np.int64))


def clusters_of(m, part, I, J):
    """The root (least slot) of every participant's cluster, by a plain union-find; -1 elsewhere."""
    par = np.arange(m)

    def find(x):
        while par[x] != x:
            par[x] = par[par[x]]
            x = par[x]
        return x

    for i, j in zip(I.tolist(), J.tolist()):
        a, b = find(i), find(j)
        if a != b:
            par[max(a, b)] = min(a, b)
    root = np.full(m, -1)
    for i in np.flatnonzero(part).tolist():
        root[i] = find(i)
    return root


def inside_rule(plane0, hidden, selected, first, count, radius, mode, threshold):
    """(inside bool over the slots, stats [participants, inside, candidates, clusters, largest])."""
    m = plane0.shape[0]
    part = participants(plane0, hidden, first, count)
    xyz = plane0[:, :3]
    sel = np.zeros(m, bool)
    sel[:len(selected)] = selected
    sel &= part
    I, J = edges(xyz, part, radius)
    clusters = largest = 0
    if mode == SPARSE:
        deg = np.bincount(I, minlength=m) + np.bincount(J, minlength=m)
        inside = part & (deg < threshold)
    elif mode == GROW:
        near = np.zeros(m, bool)
        near[I[sel[J]]] = True
        near[J[sel[I]]] = True
        inside = part & (sel | near)
    else:
        root = clusters_of(m, part, I, J)
        size = np.bincount(root[part], minlength=m)
        roots = np.flatnonzero(part & (root == np.arange(m)))
        clusters, largest = len(roots), int(size.max()) if len(roots) else 0
        if mode == CONNECTED:
            seeded = np.zeros(m, bool)
            seeded[root[sel]] = True
            inside = part & seeded[np.where(part, root, 0)]
        else:
            inside = part & (size[np.where(part, root, 0)] < threshold)
    stats = [int(part.sum()), int(inside.sum()), candidates(xyz, part, radius), clusters, largest]
    return inside, stats


def select_rule(plane0, hidden, selected, first, count, radius, mode, threshold, op):
    """(the selected mask after gsr_select_neighborhood, stats)."""
    inside, stats = inside_rule(plane0, hidden, selected, first, count, radius, mode, threshold)
    m = len(hidden)
    return sref.combine(op, np.asarray(selected, bool), inside[:m], np.asarray(hidden, bool)), stats


# ---- the serial C++ reference and the emulator ---------------------------------------------------------------------------------
def lib():
    global _emu
    if _emu is None:
        out_dir = HERE if os.access(HERE, os.W_OK) else tempfile.mkdtemp(prefix="gsr_neighbor_emu_")
        out = os.path.join(out_dir, "libneighbor_emu.so")
        deps = [os.path.join(HERE, "neighbor_emu.cpp"), os.path.abspath(__file__)] + cr._EMU_DEPS[1:] + [os.path.join(cr.CSRC, "neighbors.cu")]
        if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(d) for d in deps):
            tmp = f"{out}.{os.getpid()}.tmp"
            subprocess.run([os.environ.get("ORC_CXX", "/usr/bin/g++")] + cr._EMU_FLAGS + ["-I", cr.CUDA_INC, deps[0], "-o", tmp], check=True)
            os.replace(tmp, out)
        L = C.CDLL(out)
        vp, ull, u = C.c_void_p, C.c_ulonglong, C.c_uint
        L.emu_select_neighborhood.argtypes = [vp, ull, vp, vp, u, ull, ull, C.c_float, C.c_int, u, C.c_int, u, ull, u, vp]
        L.ref_select_neighborhood.argtypes = [vp, ull, vp, vp, C.c_float, C.c_int, u, vp, vp]
        _emu = L
    return _emu


def ref_select(plane0, hidden, selected, first, count, radius, mode, threshold, op):
    """select_rule by the serial C++ grid reference."""
    m = plane0.shape[0]
    part = participants(plane0, hidden, first, count)
    sel = np.zeros(m, bool)
    sel[:len(selected)] = selected
    xyz = np.ascontiguousarray(plane0[:, :3], dtype=F32)
    p8, s8 = part.astype(np.uint8), (sel & part).astype(np.uint8)
    inside = np.zeros(m, np.uint8)
    stats = np.zeros(5, np.uint64)
    assert lib().ref_select_neighborhood(xyz.ctypes.data, m, p8.ctypes.data, s8.ctypes.data, radius, mode, threshold, inside.ctypes.data,
                                         stats.ctypes.data) == 0
    h = len(hidden)
    return sref.combine(op, np.asarray(selected, bool), inside[:h].astype(bool), np.asarray(hidden, bool)), [int(x) for x in stats]


def ref_all_modes(plane0, hidden, selected, first, count, radius, threshold):
    """{mode: (inside bool over the slots, stats)} for every mode from one pass of the serial C++ reference."""
    m = plane0.shape[0]
    part = participants(plane0, hidden, first, count)
    sel = np.zeros(m, bool)
    sel[:len(selected)] = selected
    xyz = np.ascontiguousarray(plane0[:, :3], dtype=F32)
    p8, s8 = part.astype(np.uint8), (sel & part).astype(np.uint8)
    inside = np.zeros((4, m), np.uint8)
    stats = np.zeros((4, 5), np.uint64)
    assert lib().ref_select_neighborhood(xyz.ctypes.data, m, p8.ctypes.data, s8.ctypes.data, radius, -1, threshold, inside.ctypes.data,
                                         stats.ctypes.data) == 0
    return {md: (inside[md].astype(bool), [int(x) for x in stats[md]]) for md in MODES}


def emu_select(plane0, hidden, selected, first, count, radius, mode, threshold, op, bucket_bits=0, limit=LIMIT, ctas=4):
    """The emulated kernels on copies of the masks: (rc, selected after, stats); rc 1 = refused by the budget."""
    m = len(hidden)
    p0 = np.ascontiguousarray(plane0, dtype=F32)
    hw, sw = pack_mask(hidden, m), pack_mask(selected, m).copy()
    stats = np.zeros(5, np.uint64)
    rc = lib().emu_select_neighborhood(p0.ctypes.data, p0.shape[0], hw.ctypes.data, sw.ctypes.data, hw.size, first, count, radius, mode,
                                       threshold, op, bucket_bits, limit, ctas, stats.ctypes.data)
    assert rc in (0, 1), rc
    return rc, unpack_mask(sw, m), [int(x) for x in stats]
