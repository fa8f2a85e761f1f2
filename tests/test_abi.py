"""The C-ABI shared library loads and exports every symbol include/gsr.h declares (no compute without a GPU)."""
import ctypes as C
import os
import re

from godotgaussiansplatting_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    text = open(os.path.join(ROOT, "include", "gsr.h")).read()
    return sorted(set(re.findall(r"GSR_API\s+[\w\s\*]+?\b(gsr_\w+)\s*\(", text)))


def test_header_and_binding_list_the_same_symbols():
    assert header_symbols() == sorted(_lib.EXPORTS)


def test_library_exports_every_declared_symbol():
    L = C.CDLL(_lib.LIB_PATH)
    for name in header_symbols():
        assert hasattr(L, name), f"{name} missing from libgsr.so"


def test_struct_layouts_match_the_header():
    assert C.sizeof(_lib.GsrConfig) == 24
    assert C.sizeof(_lib.GsrStats) == 104
    assert C.sizeof(_lib.GsrFrameRecord) == 64
    assert _lib.GsrStats.stage_ms.offset == 72 and _lib.GsrStats.staged.offset == 96


def test_error_strings_and_version():
    L = _lib.lib()
    assert L.gsr_error_string(0) == b"ok"
    assert b"no CPU fallback" in L.gsr_error_string(_lib.GSR_ERR_CUDA)
    assert L.gsr_version().startswith(b"gsr ")


def test_no_cpu_fallback_without_a_device():
    """On a box without a GPU every entry point must fail loudly (GSR_ERR_CUDA), never compute on the CPU."""
    L = _lib.lib()
    if L.gsr_device_count() > 0:
        return  # GPU box: covered by the -m gpu tests
    ctx = C.c_void_p()
    cfg = _lib.GsrConfig(0, 0, 1000, 10, 0)
    rc = L.gsr_create(C.byref(cfg), C.byref(ctx))
    assert rc == _lib.GSR_ERR_CUDA and not ctx.value
    assert b"no CPU fallback" in L.gsr_last_error()
    srt = C.c_void_p()
    assert L.gsr_sorter_create(0, 1000, C.byref(srt)) == _lib.GSR_ERR_CUDA
    k = (C.c_uint32 * 4)(3, 1, 2, 0)
    assert L.gsr_sort_pairs_host(0, k, None, 4) == _lib.GSR_ERR_CUDA
    assert list(k) == [3, 1, 2, 0]  # untouched


def test_invalid_arguments_are_rejected():
    L = _lib.lib()
    assert L.gsr_create(None, None) == _lib.GSR_ERR_INVALID
    ctx = C.c_void_p()
    cfg = _lib.GsrConfig(0, 0, 0, 10, 0)
    assert L.gsr_create(C.byref(cfg), C.byref(ctx)) == _lib.GSR_ERR_INVALID
    assert L.gsr_resize(None, 10, 10) == _lib.GSR_ERR_INVALID
    assert L.gsr_sync(None) == _lib.GSR_ERR_INVALID


def test_product_code_never_touches_the_oracle():
    """The product path must not import, link or execute anything under oracle/ (parity would be void)."""
    pkg = os.path.join(ROOT, "godotgaussiansplatting_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dirpath, f), errors="replace").read()
                code = "\n".join(l for l in text.splitlines() if not l.strip().startswith(("#", "//", "*", "/*")))
                assert "from oracle" not in code and "import oracle" not in code and "gsr_oracle" not in code, f


def test_library_is_not_the_cpu_emulation_build():
    """tests/kernel_emu compiles two kernel files for the CPU behind -DGSR_CPU_EMU (a logic pre-flight, test infrastructure).
    libgsr itself must never be built that way, must not export the harness, and must carry sm_90a device code."""
    from godotgaussiansplatting_b200 import build as gsr_build
    src = open(gsr_build.__file__).read()
    assert "GSR_CPU_EMU" not in src
    L = C.CDLL(_lib.LIB_PATH)
    for name in ("emu_composite", "emu_tile_ranges", "emu_band_fixup"):
        assert not hasattr(L, name), name
    raw = open(_lib.LIB_PATH, "rb").read()
    assert b"sm_90a" in raw and b"composite_kernel" in raw
