"""Reference implementation of the compressed PLY (include/gsr.h "Compressed PLY") for the tests.

TEST INFRASTRUCTURE.  Three parts:
  1. the export rule restated in numpy float64 from float32 inputs: which splats are exported, the Morton keys and order, the
     sanitised values, the chunk statistics and the packed words and SH bytes.  The log-scales and quaternions are gsr_export_ply's, taken
     from the emulated export kernels of tests/export_reference.py (the same device function writes both);
  2. the decode rule restated in numpy float32, one IEEE operation at a time, and the store it implies: swizzle_splats (the host mirror
     of gsr_upload_ply's rule) of the decoded rows, with plane-2 z replaced by the alpha;
  3. the CPU kernel emulator of the export and decode kernels (tests/compressed_reference/compressed_emu.cpp).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from godotgaussiansplatting_b200.ply_file import PlyFile, degree_properties, swizzle_splats
from godotgaussiansplatting_b200.rasterizer import pack_mask
from tests import cutout_reference as cr
from tests import export_reference as er

F32, F64, U32 = np.float32, np.float64, np.uint32
HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "compressed_reference")
CHUNK = 256
NOT_EXPORTED = 0xFFFFFFFF
_emu = None


def sh_bytes(degree: int) -> int:
    return 3 * ((degree + 1) ** 2 - 1)


def chunk_count(rows: int) -> int:
    return (rows + CHUNK - 1) // CHUNK


def order_word(x) -> np.ndarray:
    """depth_order_word: float32 bits -> an unsigned word that orders as the float does (-0 below +0)."""
    u = np.asarray(x, dtype=F32).view(U32)
    return np.where(u >> 31 != 0, ~u, u | np.uint32(0x80000000)).astype(U32)


def order_float(w) -> np.ndarray:
    w = np.asarray(w, dtype=U32)
    return np.where(w >> 31 != 0, w ^ np.uint32(0x80000000), ~w).astype(U32).view(F32)


# ---- export rule ----------------------------------------------------------------------------------------------------------------
def exported(store, n: int, hidden, selected, selected_only: bool) -> np.ndarray:
    """The exported store indices, ascending: gsr_export_ply's rule with finite plane-0 x, y, z."""
    idx = er.exported(store, n, hidden, selected, selected_only)
    p0 = np.asarray(store, dtype=F32)[0, idx, :3]
    return idx[np.isfinite(p0).all(axis=1)]


def part1by2(v) -> np.ndarray:
    v = np.asarray(v, dtype=np.uint64) & 0x3FF
    v = (v | (v << 16)) & 0x030000FF
    v = (v | (v << 8)) & 0x0300F00F
    v = (v | (v << 4)) & 0x030C30C3
    v = (v | (v << 2)) & 0x09249249
    return v


def morton_keys(pos) -> np.ndarray:
    """(m, 3) float32 exported positions -> their 30-bit keys over the float32 bounds of the set."""
    p = np.asarray(pos, dtype=F32)
    lo, hi = p.min(axis=0), p.max(axis=0)
    cells = []
    for k in range(3):
        if hi[k] == lo[k]:
            cells.append(np.zeros(p.shape[0], dtype=np.uint64))
            continue
        c = np.floor((p[:, k].astype(F64) - F64(lo[k])) / (F64(hi[k]) - F64(lo[k])) * 1024.0)
        cells.append(np.minimum(c, 1023.0).astype(np.uint64))
    return ((part1by2(cells[2]) << 2) | (part1by2(cells[1]) << 1) | part1by2(cells[0])).astype(U32)


def norm(x, lo, hi) -> np.ndarray:
    x, lo, hi = (np.asarray(v, dtype=F32) for v in (x, lo, hi))
    r = hi.astype(F64) - lo.astype(F64)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = (x.astype(F64) - lo.astype(F64)) / r
    return np.where(x <= lo, 0.0, np.where(x >= hi, 1.0, np.where(r < 1e-5, 0.0, q)))


def unorm(v, bits: int) -> np.ndarray:
    t = float((1 << bits) - 1)
    return np.minimum(t, np.maximum(0.0, np.floor(np.asarray(v, dtype=F64) * t + 0.5))).astype(U32)


def sh_byte(v) -> np.ndarray:
    v = np.asarray(v, dtype=F32)
    with np.errstate(invalid="ignore", over="ignore"):
        t = np.trunc((v.astype(F64) / 8.0 + 0.5) * 256.0)
        b = np.minimum(255.0, np.maximum(0.0, t))
    return np.where(np.isnan(v), 128, np.nan_to_num(b)).astype(np.uint8)


def pack_rotation(q) -> np.ndarray:
    q = np.asarray(q, dtype=F32)
    i = np.argmax(np.abs(q), axis=1)                       # the first index wins a tie
    qi = q[np.arange(q.shape[0]), i]
    q = np.where((qi < 0)[:, None], -q, q)
    others = [np.where(i == 0, q[:, 1], q[:, 0]), np.where(i >= 2, q[:, 1], q[:, 2]), np.where(i == 3, q[:, 2], q[:, 3])]   # ascending
    f = [unorm(o.astype(F64) * np.sqrt(0.5) + 0.5, 10) for o in others]
    return (i.astype(U32) << 30) | (f[0] << 20) | (f[1] << 10) | f[2]


def scale_rot(store, bands: int, half: bool, n: int):
    """(n, 3) log-scales and (n, 4) quaternions of slots [0, n) as gsr_export_ply writes them (NaN rows for vacant slots)."""
    idx = er.exported(store, n, None, None, False)
    rows = er.emu_export(store, bands, half, None, None, n, False, 0)
    ls, q = np.full((n, 3), np.nan, dtype=F32), np.full((n, 4), np.nan, dtype=F32)
    ls[idx], q[idx] = rows[:, 10:13], rows[:, 13:17]
    return ls, q


def encode(store, n: int, bands: int, half: bool, hidden, selected, selected_only: bool, degree: int, morton: bool, sr=None):
    """The file the export writes: dict(idx = the rows' store indices in file order, keys = the key pass's keys of [0, n), chunks,
    packed, sh).  sr: scale_rot(store, bands, half, n) when the caller has it already."""
    s = np.asarray(store, dtype=F32)
    idx = exported(store, n, hidden, selected, selected_only)
    keys = np.full(n, NOT_EXPORTED, dtype=U32)
    if idx.size:
        keys[idx] = morton_keys(s[0, idx, :3]) if morton else 0
        idx = idx[np.argsort(keys[idx], kind="stable")]
    rows = idx.size
    ls_all, q_all = scale_rot(store, bands, half, n) if sr is None else sr
    vals = er.sh_values(store, n, bands, half)
    pos = s[0, idx, :3]
    ls = ls_all[idx]
    ls = np.where(np.isnan(ls), F32(-20), np.clip(ls, F32(-20), F32(20))).astype(F32)
    col = (vals[idx, 0:3].astype(F64) * 0.28209479177387814 + 0.5).astype(F32)
    col = np.where(np.isnan(col), F32(0.5), np.clip(col, F32(-64), F32(64))).astype(F32)
    alpha = s[2, idx, 2]
    alpha = np.where(np.isnan(alpha), F32(0), np.clip(alpha, F32(0), F32(1))).astype(F32)
    C_ = chunk_count(rows)
    chunks = np.zeros((C_, 18), dtype=F32)
    packed = np.zeros((rows, 4), dtype=U32)
    for c in range(C_):
        r = slice(c * CHUNK, min(rows, (c + 1) * CHUNK))
        for g, v in enumerate((pos, ls, col)):
            w = order_word(v[r])
            chunks[c, 6 * g:6 * g + 3] = order_float(w.min(axis=0))
            chunks[c, 6 * g + 3:6 * g + 6] = order_float(w.max(axis=0))
        ck = chunks[c]

        def p111011(v, lo, hi):
            return (unorm(norm(v[:, 0], lo[0], hi[0]), 11) << 21) | (unorm(norm(v[:, 1], lo[1], hi[1]), 10) << 11) | unorm(norm(v[:, 2], lo[2], hi[2]), 11)
        packed[r, 0] = p111011(pos[r], ck[0:3], ck[3:6])
        packed[r, 2] = p111011(ls[r], ck[6:9], ck[9:12])
        packed[r, 3] = ((unorm(norm(col[r, 0], ck[12], ck[15]), 8) << 24) | (unorm(norm(col[r, 1], ck[13], ck[16]), 8) << 16) |
                        (unorm(norm(col[r, 2], ck[14], ck[17]), 8) << 8) | unorm(alpha[r], 8))
    packed[:, 1] = pack_rotation(q_all[idx]) if rows else packed[:, 1]
    kd = (degree + 1) ** 2
    rest = vals[idx, 3:3 * kd].reshape(rows, kd - 1, 3).transpose(0, 2, 1).reshape(rows, 3 * (kd - 1))   # channel-major
    return dict(idx=idx, keys=keys, chunks=chunks, packed=packed, sh=sh_byte(rest))


# ---- decode rule ----------------------------------------------------------------------------------------------------------------
def decode(chunks, packed, sh, rows: int, chunk_floats: int, degree: int):
    """float32 rows of degree_properties(degree) (normals 0, opacity 0) and the alpha."""
    ch = np.asarray(chunks, dtype=F32).reshape(-1, chunk_floats)[np.arange(rows) // CHUNK]
    w = np.asarray(packed, dtype=U32).reshape(rows, 4)

    def u(v, b):
        return v.astype(F32) / F32((1 << b) - 1)

    def lerp(lo, hi, t):
        return lo + (hi - lo) * t

    def p111011(word, lo, hi):
        return np.stack([lerp(lo[:, 0], hi[:, 0], u(word >> 21, 11)), lerp(lo[:, 1], hi[:, 1], u((word >> 11) & 1023, 10)),
                         lerp(lo[:, 2], hi[:, 2], u(word & 2047, 11))], axis=1)
    pos = p111011(w[:, 0], ch[:, 0:3], ch[:, 3:6])
    ls = p111011(w[:, 2], ch[:, 6:9], ch[:, 9:12])
    c8 = np.stack([u((w[:, 3] >> 24) & 255, 8), u((w[:, 3] >> 16) & 255, 8), u((w[:, 3] >> 8) & 255, 8)], axis=1)
    col = lerp(ch[:, 12:15], ch[:, 15:18], c8) if chunk_floats == 18 else c8
    dc = (col - F32(0.5)) / F32(0.28209479177387814)
    alpha = u(w[:, 3] & 255, 8)
    i = (w[:, 1] >> 30).astype(np.int64)
    abc = [(u((w[:, 1] >> s) & 1023, 10) - F32(0.5)) * F32(1.41421356) for s in (20, 10, 0)]
    t = F32(1) - ((abc[0] * abc[0] + abc[1] * abc[1]) + abc[2] * abc[2])
    m = np.sqrt(np.where(t > 0, t, F32(0))).astype(F32)
    a, b, c = abc
    q = np.stack([np.where(i == 0, m, a), np.where(i == 0, a, np.where(i == 1, m, b)), np.where(i <= 1, b, np.where(i == 2, m, c)),
                  np.where(i == 3, m, c)], axis=1).astype(F32)
    sb = sh_bytes(degree)
    rest = ((np.asarray(sh, dtype=np.uint8).reshape(rows, sb).astype(F32) + F32(0.5)) * F32(0.03125) - F32(4.0)) if sb else np.zeros((rows, 0), F32)
    table = np.concatenate([pos, np.zeros((rows, 3), F32), dc, rest, np.zeros((rows, 1), F32), ls, q], axis=1).astype(F32)
    return table, alpha


def store_rule(table, alpha, degree: int, bands: int, half: bool, stride: int, first: int = 0, creation_time: float = 0.0, base=None):
    """The store after an upload of the decoded rows at `first` into `base` (a store of the same format, or zeros)."""
    rows = table.shape[0]
    lay = PlyFile.from_array(table, degree_properties(degree)).layout()
    s60 = swizzle_splats(table, creation_time, lay)
    s60[:, 10] = alpha
    part = er.store_from_structs(s60, bands, half, rows)
    out = np.zeros((part.shape[0], stride, 4), dtype=F32) if base is None else np.array(base, dtype=F32, copy=True)
    out[:, first:first + rows] = part
    return out


# ---- stores ---------------------------------------------------------------------------------------------------------------------
def random_store(rng, n: int, bands: int, half: bool, stride: int | None = None):
    """A store of n random splats (a realistic 3DGS table through swizzle_splats), slots past n zero."""
    t = np.zeros((n, 62), dtype=F32)
    t[:, 0:3] = rng.normal(size=(n, 3)) * 3.0
    t[:, 6:54] = rng.normal(size=(n, 48)) * 0.6
    t[:, 54] = rng.normal(size=n) * 2.0
    t[:, 55:58] = rng.uniform(-6, -1, size=(n, 3))
    t[:, 58:62] = rng.normal(size=(n, 4))
    s60 = swizzle_splats(t, 0.0)
    return er.store_from_structs(s60, bands, half, stride or n)


# ---- the CPU kernel emulator ----------------------------------------------------------------------------------------------------
def emu():
    global _emu
    if _emu is None:
        out_dir = HERE if os.access(HERE, os.W_OK) else tempfile.mkdtemp(prefix="gsr_compressed_emu_")
        out = os.path.join(out_dir, "libcompressed_emu.so")
        deps = [os.path.join(HERE, "compressed_emu.cpp")] + cr._EMU_DEPS[1:] + [os.path.join(cr.CSRC, "compressed_ply.cu")]
        if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(d) for d in deps):
            tmp = f"{out}.{os.getpid()}.tmp"
            subprocess.run([os.environ.get("ORC_CXX", "/usr/bin/g++")] + cr._EMU_FLAGS + ["-I", cr.CUDA_INC, deps[0], "-o", tmp], check=True)
            os.replace(tmp, out)
        L = C.CDLL(out)
        vp, ull = C.c_void_p, C.c_ulonglong
        L.emu_compress.argtypes = [C.c_int, C.c_int, vp, ull, ull, vp, vp, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp, vp, ull]
        L.emu_compress.restype = C.c_longlong
        L.emu_decompress.argtypes = [C.c_int, C.c_int, vp, vp, vp, ull, C.c_uint, C.c_int, C.c_float, vp, ull, ull]
        L.emu_decompress.restype = C.c_int
        _emu = L
    return _emu


def _ptr(a):
    return None if a is None else a.ctypes.data


def emu_compress(store, bands, half, hidden, selected, n, selected_only, degree, morton):
    """The emulated export: dict(count, keys (before the sort), vals (sorted), chunks, packed, sh)."""
    s = np.ascontiguousarray(store, dtype=F32)
    hw = None if hidden is None else pack_mask(hidden, len(hidden))
    sw = None if hidden is None else pack_mask(selected, len(selected))
    L = emu()
    count = L.emu_compress(bands, int(half), s.ctypes.data, s.shape[1], n, _ptr(hw), _ptr(sw), int(selected_only), int(morton), degree,
                           None, None, None, None, None, 0)
    assert count >= 0
    keys, vals = np.zeros(max(n, 1), dtype=U32), np.zeros(max(n, 1), dtype=U32)
    chunks = np.full((chunk_count(count), 18), np.nan, dtype=F32)
    packed = np.zeros((count, 4), dtype=U32)
    sh = np.zeros((count, sh_bytes(degree)), dtype=np.uint8)
    if count:
        got = L.emu_compress(bands, int(half), s.ctypes.data, s.shape[1], n, _ptr(hw), _ptr(sw), int(selected_only), int(morton), degree,
                             keys.ctypes.data, vals.ctypes.data, chunks.ctypes.data, packed.ctypes.data, sh.ctypes.data, count)
        assert got == count, got
    return dict(count=int(count), keys=keys[:n], vals=vals[:count], chunks=chunks, packed=packed, sh=sh)


def emu_decompress(chunks, packed, sh, rows, chunk_floats, degree, bands, half, store, first=0, creation_time=0.0):
    """The emulated upload into a copy of `store`; returns the new store."""
    out = np.array(store, dtype=F32, copy=True, order="C")
    ch = np.ascontiguousarray(chunks, dtype=F32)
    pk = np.ascontiguousarray(packed, dtype=U32)
    sb = np.ascontiguousarray(sh, dtype=np.uint8) if sh is not None else None
    rc = emu().emu_decompress(bands, int(half), ch.ctypes.data, pk.ctypes.data, _ptr(sb), rows, chunk_floats, degree, creation_time,
                              out.ctypes.data, out.shape[1], first)
    assert rc == 0
    return out
