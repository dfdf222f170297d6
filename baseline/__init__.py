"""GPU baselines timed beside the engine (bench.py `gpu_baselines`; SURVEY.md 8(d)): measurement infrastructure,
never imported by the product.  gpu_composition.cu restates what the reference's surviving primitives compose to
(row norms + cuBLASLt SGEMM with CUBLAS_COMPUTE_32F + one elementwise pass [+ row arg-min pass])."""
from __future__ import annotations

import ctypes
import os
import shutil
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(_HERE, "libgpu_composition.so")
SRC = os.path.join(_HERE, "gpu_composition.cu")
_lib = None


def build(force: bool = False) -> str:
    if not force and os.path.exists(SO_PATH) and os.path.getmtime(SO_PATH) >= os.path.getmtime(SRC):
        return SO_PATH
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    cmd = [nvcc, "-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-shared",
           "-Xcompiler", "-fPIC", "-o", SO_PATH, SRC, "-lcublasLt", "-Xlinker", "-rpath", "-Xlinker", "/usr/local/cuda/lib64"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    return SO_PATH


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(SO_PATH):
            build()
        L = ctypes.CDLL(SO_PATH)
        vp, i64, ci, sz = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_size_t
        L.bl_last_error.restype = ctypes.c_char_p
        L.bl_init.restype = ci
        L.bl_pairwise_l2.restype = ci
        L.bl_pairwise_l2.argtypes = [vp, vp, vp, vp, vp, vp, i64, i64, i64, ci, vp, sz]
        L.bl_l2_nn.restype = ci
        L.bl_l2_nn.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, i64, i64, i64, i64, vp, sz]
        _lib = L
    return _lib


def check(rc: int) -> None:
    if rc:
        raise RuntimeError("gpu baseline: " + lib().bl_last_error().decode())
