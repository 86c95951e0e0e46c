"""Build helpers: compile the in-tree native libraries (nvcc for sm_90a, g++ for host helpers).

Everything is built in-tree under quatro_b200/lib/, so the package is importable from the source
tree.  Nothing here falls back to a CPU implementation: if nvcc is missing the build raises.
"""
from __future__ import annotations

import os
import shutil
import subprocess
from pathlib import Path

PKG = Path(__file__).resolve().parent
ROOT = PKG.parent
LIB_DIR = PKG / "lib"
CSRC = PKG / "csrc"
CUDA_LIB = LIB_DIR / "libquatro_b200.so"
SYNTH_LIB = LIB_DIR / "libqb200_synth.so"
HOST_CXX = "/usr/bin/g++"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    # no implicit FMA contraction: float results must match the CPU oracle bit for bit; kernels
    # that want an FMA ask for it explicitly with fmaf()/__fmaf_rn().
    "-fmad=false",
    "-Xcompiler", "-fPIC", "-shared",
    "--expt-relaxed-constexpr",
]


def _newer(target: Path, sources) -> bool:
    if not target.exists():
        return True
    t = target.stat().st_mtime
    return any(Path(s).stat().st_mtime > t for s in sources)


def nvcc_path() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found: the CUDA path cannot be built (there is no CPU fallback)")


def cuda_tool(name: str) -> str:
    """A program of the CUDA toolkit the build uses (cuobjdump, ...): next to its nvcc, else from PATH."""
    cand = Path(nvcc_path()).parent / name
    return str(cand) if cand.exists() else name


def build_cuda(force: bool = False, verbose: bool = False) -> Path:
    srcs = sorted(CSRC.glob("*.cu"))
    deps = srcs + sorted(CSRC.glob("*.cuh")) + [ROOT / "include" / "quatro_b200.h"]
    if not force and not _newer(CUDA_LIB, deps):
        return CUDA_LIB
    LIB_DIR.mkdir(exist_ok=True)
    cmd = [nvcc_path(), *NVCC_FLAGS, "-ccbin", HOST_CXX, "-I", str(ROOT / "include"), "-I", str(CSRC),
           "-o", str(CUDA_LIB), *map(str, srcs), "-lcudart", "-ldl"]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
    if verbose:
        print(r.stdout + r.stderr)
    return CUDA_LIB


def build_synth(force: bool = False) -> Path:
    src = PKG / "synth" / "synth.cpp"
    if not force and not _newer(SYNTH_LIB, [src]):
        return SYNTH_LIB
    LIB_DIR.mkdir(exist_ok=True)
    cmd = [HOST_CXX, "-O2", "-std=c++17", "-fPIC", "-shared", "-o", str(SYNTH_LIB), str(src)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("g++ failed:\n" + r.stdout + r.stderr)
    return SYNTH_LIB
