"""Build the sm_90a CUDA library in-tree (raft_b200/libraft_b200.so) with nvcc."""
from __future__ import annotations

import os
import shutil
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
SO_PATH = os.path.join(_HERE, "libraft_b200.so")

NVCC_FLAGS = [
    "-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
    "--expt-relaxed-constexpr", "-shared", "-Xcompiler", "-fPIC",
]


def _nvcc() -> str:
    cand = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(cand):
        raise RuntimeError("nvcc not found; raft_b200 has no prebuilt or CPU fallback")
    return cand


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh")))


def is_stale() -> bool:
    if not os.path.exists(SO_PATH):
        return True
    t = os.path.getmtime(SO_PATH)
    deps = sources() + [os.path.join(_HERE, "..", "include", "raft_b200.h")]
    return any(os.path.getmtime(s) > t for s in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not is_stale():
        return SO_PATH
    units = [s for s in sources() if s.endswith(".cu")]
    cmd = [_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", SO_PATH] + units + ["-ldl"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    if verbose:
        print(res.stderr)
    return SO_PATH


if __name__ == "__main__":
    print(build(force=True, verbose=True))
