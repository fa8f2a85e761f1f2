"""Compressed PLY (include/gsr.h "Compressed PLY") on the CPU: the export and decode kernels of compressed_ply.cu and ingest.cu, run by
the kernel emulator, against the numpy restatement of the rule (tests/compressed_reference.py) bit for bit; the round-trip bounds that
follow from the quantisation steps; and CompressedPlyFile's save and parse."""
from __future__ import annotations

import numpy as np
import pytest

from godotgaussiansplatting_b200.compressed_ply import CompressedPlyFile, is_compressed_ply
from tests import compressed_reference as cref
from tests import export_reference as er
from tests.transform_reference import sh_planes

F32, U32 = np.float32, np.uint32


def check_file(got, ref):
    assert got["count"] == ref["idx"].size
    np.testing.assert_array_equal(got["keys"], ref["keys"])
    np.testing.assert_array_equal(got["vals"], ref["idx"])
    np.testing.assert_array_equal(got["chunks"].view(U32), ref["chunks"].view(U32))
    np.testing.assert_array_equal(got["packed"], ref["packed"])
    np.testing.assert_array_equal(got["sh"], ref["sh"])


def masks(rng, n):
    hidden = rng.random(n) < 0.2
    selected = (rng.random(n) < 0.5) & ~hidden
    return hidden, selected


@pytest.mark.parametrize("bands", [1, 2, 3, 4])
@pytest.mark.parametrize("half", [False, True])
def test_emulated_export_matches_the_rule(bands, half):
    rng = np.random.default_rng(100 * bands + half)
    n = 700   # three chunks, the last partial
    store = cref.random_store(rng, n, bands, half, 768)
    store[0, 13, :3] = np.nan                               # vacant
    store[0, 14, 1] = np.inf                                # infinite position: not exported
    hidden, selected = masks(rng, 768)
    for scope, hid, sel, sel_only in (("masks off", None, None, False), ("kept", hidden, selected, False), ("selected", hidden, selected, True)):
        for degree in range(bands):
            for morton in (False, True):
                ref = cref.encode(store, n, bands, half, hid, sel, sel_only, degree, morton)
                got = cref.emu_compress(store, bands, half, hid, sel, n, sel_only, degree, morton)
                check_file(got, ref)
    assert 14 not in cref.exported(store, n, None, None, False) and 15 in cref.exported(store, n, None, None, False)


@pytest.mark.parametrize("n", [1, 255, 256, 257])
def test_row_counts_around_a_chunk(n):
    rng = np.random.default_rng(n)
    store = cref.random_store(rng, n, 2, False)
    for morton in (False, True):
        ref = cref.encode(store, n, 2, False, None, None, False, 1, morton)
        got = cref.emu_compress(store, 2, False, None, None, n, False, 1, morton)
        check_file(got, ref)
        assert got["chunks"].shape == (cref.chunk_count(n), 18)


def edge_store():
    """One chunk of identical splats, then a chunk of special values."""
    rng = np.random.default_rng(7)
    n = 512
    store = cref.random_store(rng, n, 4, False)
    store[:, 1:256] = store[:, 0:1]                        # chunk 0: identical splats (degenerate ranges)
    s = 256
    for name, S in er.special_covariances(rng):            # NaN / inf covariances, needles, 180 degree rotations, tied components
        er.put_special(store, s, S)
        s += 1
    # tied largest quaternion components: a 90 degree turn about x gives w = x
    R = er.rotation((1, 0, 0), np.pi / 2)
    er.set_covariance(store, s, R @ np.diag([1e-3, 2e-3, 3e-3]) @ R.T); s += 1
    store[2, s, 2] = 0.0; s += 1                           # alpha 0, 1, out of range and NaN
    store[2, s, 2] = 1.0; s += 1
    store[2, s, 2] = 1.5; s += 1
    store[2, s, 2] = np.nan; s += 1
    store[3, s, 0:3] = [np.nan, np.inf, -np.inf]; s += 1   # colour NaN and +-inf
    store[3, s, 0:3] = [1e3, -1e3, 0.0]; s += 1
    vals = [4.0, -4.0, 3.99, -3.99, 4.5, -9.0, np.nan, np.inf, -np.inf, 4.0 - 1 / 64]
    store[4, s, :] = vals[:4]; store[5, s, :] = vals[4:8]; store[6, s, :2] = vals[8:]; s += 1   # SH beyond +-4, NaN
    # values exactly at the chunk's bounds: the largest and smallest x of chunk 1
    store[0, s, 0] = 50.0; store[0, s + 1, 0] = -50.0
    return store, n


@pytest.mark.parametrize("morton", [False, True])
def test_edge_cases(morton):
    store, n = edge_store()
    ref = cref.encode(store, n, 4, False, None, None, False, 3, morton)
    got = cref.emu_compress(store, 4, False, None, None, n, False, 3, morton)
    check_file(got, ref)
    if not morton:   # chunk 0 of identical splats: every range is degenerate, every normalised value 0
        assert (got["chunks"][0, 0:3] == got["chunks"][0, 3:6]).all()
        assert (got["packed"][:256, 0] == 0).all() and (got["packed"][:256, 2] == 0).all()
        assert len(set(got["packed"][:256, 1].tolist())) == 1


def test_pack_rotation_ties_and_signs():
    q = np.array([[0.5, 0.5, 0.5, 0.5], [-0.5, 0.5, 0.5, 0.5], [0, 1, 0, 0], [0, 0, 0, -1], [0.7071068, 0, -0.7071068, 0]], dtype=F32)
    w = cref.pack_rotation(q)
    assert (w >> 30).tolist() == [0, 0, 1, 3, 0]            # the first of the tied largest components
    mid = cref.unorm(0.5, 10)
    assert int(w[2]) & 0x3FFFFFFF == (mid << 20) | (mid << 10) | mid
    assert int(w[3]) & 0x3FFFFFFF == (mid << 20) | (mid << 10) | mid   # negated: -1 at index 3 becomes +1


def round_trip(store, n, bands, half, degree, morton):
    """The emulated export, then the emulated upload into a fresh store of the same format."""
    f = cref.emu_compress(store, bands, half, None, None, n, False, degree, morton)
    out = np.zeros_like(store)
    out = cref.emu_decompress(f["chunks"], f["packed"], f["sh"] if degree else None, f["count"], 18, degree, bands, half, out)
    return f, out


def test_round_trip_bounds():
    """Each quantity comes back within half a quantisation step of its chunk range (the unorm rounds to nearest, the lerp adds a few
    float32 roundings):  position within (hi - lo) / (2 * 2047) on x, z and (hi - lo) / (2 * 1023) on y; alpha within 1 / 510; colour
    within (hi - lo) / 510; SH within 1 / 64 inside +-(4 - 1/64); the rotation within the 10-bit step of each component."""
    rng = np.random.default_rng(11)
    n, bands = 1000, 4
    store = cref.random_store(rng, n, bands, False)
    f, out = round_trip(store, n, bands, False, 3, True)
    idx = f["vals"]
    ch = f["chunks"][np.arange(n) // 256]
    src, dst = store[:, idx], out[:, :n]
    rng_xyz = ch[:, 3:6].astype(np.float64) - ch[:, 0:3]
    bound = rng_xyz / np.array([2 * 2047, 2 * 1023, 2 * 2047]) * (1 + 1e-5) + 1e-6
    assert (np.abs(dst[0, :, :3].astype(np.float64) - src[0, :, :3]) <= bound).all()
    assert (np.abs(dst[2, :, 2].astype(np.float64) - src[2, :, 2]) <= 1 / 510 + 1e-7).all()
    sv, dv = er.sh_values(store[:, idx], n, bands, False), er.sh_values(dst, n, bands, False)
    col_s = sv[:, :3].astype(np.float64) * 0.28209479177387814 + 0.5
    col_d = dv[:, :3].astype(np.float64) * 0.28209479177387814 + 0.5
    assert (np.abs(col_d - col_s) <= (ch[:, 15:18] - ch[:, 12:15]) / 510 * (1 + 1e-4) + 1e-6).all()
    inside = np.abs(sv[:, 3:]) <= 4 - 1 / 64
    assert (np.abs(dv[:, 3:] - sv[:, 3:])[inside] <= 1 / 64 + 1e-6).all()
    # the rotation: each stored quaternion component is within sqrt(2) / (2 * 1023) before the largest is rebuilt; the rebuilt unit
    # quaternion then differs from the exported one by an angle of a few of those steps
    _, q_src = cref.scale_rot(store, bands, False, n)
    tab, _ = cref.decode(f["chunks"], f["packed"], f["sh"], n, 18, 3)
    q_dst = tab[:, -4:].astype(np.float64)
    dot = np.abs((q_src[idx].astype(np.float64) * q_dst).sum(axis=1)) / np.linalg.norm(q_dst, axis=1)
    angle = 2 * np.arccos(np.minimum(1.0, dot))
    assert angle.max() <= 4 * np.sqrt(2) / (2 * 1023) * 2, angle.max()


@pytest.mark.parametrize("chunk_floats", [18, 12])
def test_emulated_decode_matches_the_store_rule(chunk_floats):
    rng = np.random.default_rng(chunk_floats)
    n = 600
    src = cref.random_store(rng, n, 4, False)
    for degree in range(4):
        f = cref.emu_compress(src, 4, False, None, None, n, False, degree, True)
        ch = f["chunks"] if chunk_floats == 18 else np.ascontiguousarray(f["chunks"][:, :12])
        table, alpha = cref.decode(ch, f["packed"], f["sh"], n, chunk_floats, degree)
        for bands in (1, 2, 3, 4):
            for half in (False, True):
                base = rng.normal(size=(3 + sh_planes(bands, half), 700, 4)).astype(F32)
                got = cref.emu_decompress(ch, f["packed"], f["sh"] if degree else None, n, chunk_floats, degree, bands, half, base, first=64,
                                          creation_time=2.5)
                want = cref.store_rule(table, alpha, degree, bands, half, 700, first=64, creation_time=2.5, base=base)
                np.testing.assert_array_equal(got.view(U32), want.view(U32))


def test_save_then_parse(tmp_path):
    rng = np.random.default_rng(3)
    n = 300
    store = cref.random_store(rng, n, 3, False)
    f = cref.emu_compress(store, 3, False, None, None, n, False, 2, True)
    cp = CompressedPlyFile.from_arrays(f["chunks"], f["packed"], f["sh"], 2)
    path = str(tmp_path / "c.ply")
    cp.save(path)
    header = ["ply", "format binary_little_endian 1.0", "element chunk 2"]
    header += [f"property float {p}" for p in ("min_x", "min_y", "min_z", "max_x", "max_y", "max_z", "min_scale_x", "min_scale_y",
                                               "min_scale_z", "max_scale_x", "max_scale_y", "max_scale_z", "min_r", "min_g", "min_b",
                                               "max_r", "max_g", "max_b")]
    header += ["element vertex 300"] + [f"property uint packed_{p}" for p in ("position", "rotation", "scale", "color")]
    header += ["element sh 300"] + [f"property uchar f_rest_{i}" for i in range(24)] + ["end_header"]
    raw = open(path, "rb").read()
    head = ("\n".join(header) + "\n").encode()
    assert raw.startswith(head)
    assert len(raw) == len(head) + 2 * 18 * 4 + 300 * 16 + 300 * 24
    assert is_compressed_ply(path)
    back = CompressedPlyFile(path)
    assert back.size == n and back.sh_degree == 2 and back.chunk_floats == 18
    np.testing.assert_array_equal(back.chunks.view(U32), f["chunks"].view(U32))
    np.testing.assert_array_equal(back.packed, f["packed"])
    np.testing.assert_array_equal(back.sh, f["sh"])
    # comments anywhere in the header, and an older file's 12-float chunks, degree 0
    old = CompressedPlyFile.from_arrays(f["chunks"][:, :12], f["packed"], None, 0)
    old.save(path)
    text = old.header().decode().split("\n")
    text.insert(2, "comment written by an older tool")
    text.insert(5, "comment another")
    with open(path, "wb") as fh:
        fh.write("\n".join(text).encode())
        fh.write(np.ascontiguousarray(old.chunks, dtype="<f4").tobytes() + old.packed.astype("<u4").tobytes())
    back = CompressedPlyFile(path)
    assert back.chunk_floats == 12 and back.sh is None and back.sh_degree == 0
    np.testing.assert_array_equal(back.chunks.view(U32), f["chunks"][:, :12].view(U32))
    np.testing.assert_array_equal(back.packed, f["packed"])
