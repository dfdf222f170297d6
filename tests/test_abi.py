"""CPU tier: the C-ABI library loads, exports every symbol include/raft_b200.h declares, answers the
size queries, validates arguments, and fails loudly (no CPU fallback) without a GPU."""
import ctypes
import os
import re

import pytest

from raft_b200 import _build, _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "raft_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b2d_[a-z0-9_]+)\s*\(", src)))


def test_library_builds_and_exports_every_declared_symbol():
    path = _build.build()
    assert os.path.exists(path)
    L = ctypes.CDLL(path)
    syms = header_symbols()
    assert len(syms) >= 10
    for s in syms:
        assert hasattr(L, s), f"{s} declared in include/raft_b200.h but not exported"
    assert sorted(_lib.SYMBOLS) == syms


def test_library_is_sm90a_only_and_has_wgmma_tma():
    import shutil
    import subprocess
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([cuobjdump, "-lelf", _build.SO_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out and "sm_100" not in out
    sass = subprocess.run([cuobjdump, "-sass", _build.SO_PATH], capture_output=True, text=True).stdout
    for mnemonic in ("HGMMA", "UTMALDG", "SYNCS"):
        assert mnemonic in sass, mnemonic


def test_workspace_queries():
    L = _lib.lib()
    assert L.b2d_version() >= 100
    # unexpanded metrics need no scratch; expanded ones need the packed fp16 hi/lo copies
    assert L.b2d_pairwise_workspace_bytes(3, 0, 1000, 1000, 64) == 0
    ws = L.b2d_pairwise_workspace_bytes(0, 0, 1000, 1000, 64)
    assert ws >= 2 * 1000 * 64 * 4 and ws < 4 * 1000 * 64 * 4 + 65536
    assert L.b2d_pairwise_workspace_bytes(13, 0, 10, 10, 4) == 2 ** 64 - 1   # Haversine: not on this path
    assert L.b2d_pairwise_workspace_bytes(16, 0, 10, 10, 4) == 0             # Hamming: SIMT path, no scratch
    assert L.b2d_fused_l2_nn_workspace_bytes(100, 200, 96) > 300 * 96 * 4


def test_invalid_arguments_are_reported_not_crashed():
    L = _lib.lib()
    rc = L.b2d_pairwise_distance(None, 0, 0, None, 8, None, 8, None, 8, 4, 4, 8, 1, 2.0, None, 0)
    assert rc == _lib.B2D_ERR_INVALID_ARG and b"null" in L.b2d_last_error()
    rc = L.b2d_pairwise_distance(None, 0, 0, 256, 4, 256, 8, 256, 8, 4, 4, 8, 1, 2.0, None, 0)
    assert rc == _lib.B2D_ERR_INVALID_ARG          # ldx < k
    rc = L.b2d_pairwise_distance(None, 13, 0, 256, 8, 256, 8, 256, 8, 4, 4, 8, 1, 2.0, None, 0)
    assert rc == _lib.B2D_ERR_UNSUPPORTED
    rc = L.b2d_pairwise_distance(None, 0, 0, 256, 8, 256, 8, 256, 8, 4, 4, 8, 1, 2.0, None, 0)
    assert rc == _lib.B2D_ERR_WORKSPACE
    with pytest.raises(_lib.LogicError):
        _lib.check(rc)
    assert L.b2d_pairwise_distance(None, 0, 0, None, 8, None, 8, None, 8, 0, 4, 8, 1, 2.0, None, 0) == _lib.B2D_OK


def test_no_cpu_fallback():
    """Without a GPU a compute call must fail with B2D_ERR_CUDA, never silently compute."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    L = _lib.lib()
    rc = L.b2d_pairwise_distance(None, 3, 0, 256, 8, 256, 8, 256, 8, 4, 4, 8, 1, 2.0, None, 0)
    assert rc == _lib.B2D_ERR_CUDA
    with pytest.raises(_lib.CudaError):
        _lib.check(rc)
    from raft_b200.common import DeviceResources
    with pytest.raises(RuntimeError):
        DeviceResources()


def test_product_never_imports_the_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "raft_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in txt and "from oracle" not in txt and "liboracle" not in txt, f
