"""The C-ABI from C: include/gsr.h is a strict C99 / C++17 header, and examples/gsr_host.c -- a minimal C host that plays
GaussianSplattingRasterizer.rasterize() for one frame -- links against libgsr.so, fails loudly without a GPU, and (on an
H100) produces the oracle's frame."""
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

from godotgaussiansplatting_b200 import _lib
from tests.scenes import make_scene

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GCC = shutil.which("gcc", path="/usr/bin") or shutil.which("gcc")
GXX = shutil.which("g++", path="/usr/bin") or shutil.which("g++")
pytestmark = pytest.mark.skipif(GCC is None, reason="no C compiler")


def build_host(tmp_path) -> str:
    exe = str(tmp_path / "gsr_host")
    libdir = os.path.dirname(_lib.LIB_PATH)
    subprocess.run([GCC, "-std=c99", "-pedantic", "-Wall", "-Wextra", "-Werror", "-O2", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "examples", "gsr_host.c"), "-L", libdir, "-lgsr", f"-Wl,-rpath,{libdir}", "-o", exe],
                   check=True, capture_output=True, text=True)
    return exe


def write_request(path, splat60, vp, ub, w, h, heatmap=0.0, flags=0):
    splat60 = np.ascontiguousarray(splat60, dtype=np.float32)
    with open(path, "wb") as f:
        f.write(struct.pack("<4sIIIfI", b"GSRQ", splat60.shape[0], w, h, heatmap, flags))
        f.write(splat60.tobytes())
        f.write(np.ascontiguousarray(vp, dtype=np.float32).tobytes())
        f.write(bytes(ub))


def test_header_is_strict_c99_and_cxx17():
    hdr = os.path.join(ROOT, "include", "gsr.h")
    subprocess.run([GCC, "-std=c99", "-pedantic", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-x", "c", hdr], check=True)
    if GXX:
        subprocess.run([GXX, "-std=c++17", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-x", "c++", hdr], check=True)


def test_struct_sizes_seen_by_a_c_compiler(tmp_path):
    src = tmp_path / "sizes.c"
    src.write_text('#include <stdio.h>\n#include "gsr.h"\nint main(void){printf("%zu %zu %zu %d\\n", sizeof(gsr_config), '
                   'sizeof(gsr_stats), sizeof(gsr_frame_record), GSR_HISTORY_FRAMES);return 0;}\n')
    exe = str(tmp_path / "sizes")
    subprocess.run([GCC, "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe], check=True)
    out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split()
    import ctypes as C
    assert [int(x) for x in out] == [C.sizeof(_lib.GsrConfig), C.sizeof(_lib.GsrStats), C.sizeof(_lib.GsrFrameRecord), 512]


def test_c_host_links_and_fails_loudly_without_a_gpu(tmp_path):
    exe = build_host(tmp_path)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 2 and "usage" in r.stderr and "libgsr" in r.stderr
    if _lib.lib().gsr_device_count() > 0:
        pytest.skip("a GPU is present: the no-device path cannot be exercised")
    splat60, vp, ub = make_scene(100, 1, 64, 48)
    req = tmp_path / "frame.gsrq"
    write_request(req, splat60, vp, ub, 64, 48)
    r = subprocess.run([exe, str(req), str(tmp_path / "out.rgba")], capture_output=True, text=True)
    assert r.returncode == 3, (r.returncode, r.stderr)
    assert "gsr_create failed" in r.stderr and "no CPU fallback" in r.stderr
    assert not (tmp_path / "out.rgba").exists()


@pytest.mark.gpu
def test_c_host_renders_the_oracle_frame(tmp_path):
    from oracle import oracle as orc
    n, w, h = 5000, 320, 240
    splat60, vp, ub = make_scene(n, 21, w, h, scale_boost=1.0)
    ref = orc.frame(splat60, vp, orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8)))
    assert not ref.overflow
    exe = build_host(tmp_path)
    req, out = tmp_path / "frame.gsrq", tmp_path / "out.rgba"
    write_request(req, splat60, vp, ub, w, h)
    r = subprocess.run([exe, str(req), str(out)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert f"duplicates {ref.duplicates} " in r.stdout and f"visible {ref.visible} " in r.stdout
    img = np.fromfile(out, dtype=np.float32).reshape(h, w, 4)
    assert np.abs(img - ref.rgba).max() <= 1e-4
    np.testing.assert_array_equal(img.view(np.uint32), ref.rgba.view(np.uint32))
