"""In-tree build of the native libraries (nvcc for sm_90a; g++ for the workload generator).

The built .so files stay in-tree (git-ignored) so that they travel to the GPU box with the snapshot.
"""
from __future__ import annotations

import os
import shutil
import subprocess
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
LIB = PKG / "libgpumqtt.so"
WL_LIB = PKG / "libgmworkload.so"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC,-O3", "-shared",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found")


def _newer(target: Path, sources) -> bool:
    if not target.exists():
        return True
    t = target.stat().st_mtime
    return any(Path(s).stat().st_mtime > t for s in sources)


def build_engine(force: bool = False, verbose: bool = False) -> Path:
    srcs = [CSRC / "engine.cu", CSRC / "host_trie.cpp", CSRC / "retain_tree.cpp", CSRC / "router_host.cpp", CSRC / "batcher.cpp"]
    deps = srcs + sorted(CSRC.glob("*.h")) + sorted(CSRC.glob("*.cuh")) + [PKG.parent / "include" / "gpumqtt.h"]
    if force or _newer(LIB, deps):
        cmd = [_nvcc(), *NVCC_FLAGS, "-o", str(LIB), *map(str, srcs)]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        subprocess.check_call(cmd)
    return LIB


def build_workload(force: bool = False) -> Path:
    src = CSRC / "workload.cpp"
    if force or _newer(WL_LIB, [src]):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", "-o", str(WL_LIB), str(src)])
    return WL_LIB


def build_all(force: bool = False) -> None:
    build_engine(force)
    build_workload(force)
