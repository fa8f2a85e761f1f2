"""Builds godotgaussiansplatting_b200/csrc/*.cu into the in-tree shared library `libgsr.so` for sm_90a (H100).

nvcc cross-compiles without a GPU; the .so travels to the GPU box with the repo snapshot.
-fmad=false is part of the numerical contract ("gsr deterministic math", DESIGN.md section 4): every
FMA in the kernels is an explicit __fmaf_rn.
"""
from __future__ import annotations

import glob
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libgsr.so")

NVCC_FLAGS = [
    "-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
    "-fmad=false", "-prec-div=true", "-prec-sqrt=true", "-ftz=false",
    "-Xcompiler", "-fPIC,-fvisibility=hidden", "-shared", "-cudart", "shared",
]


def nvcc_path() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found; libgsr has no CPU fallback and cannot be built without the CUDA toolkit")


def sources() -> list[str]:
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def needs_build() -> bool:
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + [os.path.join(HERE, "..", "include", "gsr.h"), __file__]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False, extra: list[str] | None = None, out: str | None = None) -> str:
    if not force and not needs_build() and out is None:
        return OUT
    cmd = [nvcc_path()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + (extra or []) + ["-o", out or OUT] + sources()
    env = dict(os.environ)
    # the image exports CC/CXX wrappers that nvcc must not pick up as host compiler
    res = subprocess.run(cmd + ["-ccbin", "/usr/bin/g++"], env=env, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError("nvcc failed")
    if verbose:
        sys.stderr.write(res.stdout + res.stderr)
    return out or OUT


GODOT_DIR = os.path.join(HERE, "godot")
GODOT_OUT = os.path.join(GODOT_DIR, "libgsr_godot.so")


def build_godot_shim(force: bool = False) -> str:
    """The GDExtension entry (godot/gsr_gdextension.c) -> godot/libgsr_godot.so, linked against the in-tree libgsr.so."""
    src = os.path.join(GODOT_DIR, "gsr_gdextension.c")
    deps = [src, os.path.join(GODOT_DIR, "gdextension_min.h"), os.path.join(HERE, "..", "include", "gsr.h"), OUT]
    if force or not os.path.exists(GODOT_OUT) or any(os.path.getmtime(d) > os.path.getmtime(GODOT_OUT) for d in deps if os.path.exists(d)):
        cmd = ["/usr/bin/gcc", "-std=gnu11", "-O2", "-Wall", "-Wextra", "-fPIC", "-fvisibility=hidden", "-shared", src, "-o", GODOT_OUT,
               "-L", HERE, "-lgsr", "-Wl,-rpath,$ORIGIN:$ORIGIN/.."]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            sys.stderr.write(res.stdout + res.stderr)
            raise RuntimeError("building the GDExtension shim failed")
    return GODOT_OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
