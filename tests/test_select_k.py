"""select_k without a GPU: the ABI's workspace query and argument checks, the key transform compiled for the host
against the numpy oracle, the oracle itself, and the C++ shim's compile (its run is marked gpu)."""
import os
import subprocess

import numpy as np
import pytest

import cpp_build
from oracle.select_k import select_k as ref_select_k
from oracle.select_k import select_key
from raft_b200 import _lib

SIZE_MAX = 2 ** 64 - 1


@pytest.fixture(scope="module")
def build_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("select_k_cpp"))


def test_workspace_query():
    L = _lib.lib()
    for rows, n, k in ((0, 5, 0), (1, 5, 0), (1, 5, 6), (-1, 5, 1), (1, 2 ** 31, 1), (2 ** 31, 10, 1)):
        assert L.b2d_select_k_workspace_bytes(rows, n, k) == SIZE_MAX, (rows, n, k)
    assert L.b2d_select_k_workspace_bytes(0, 5, 3) == 0
    assert L.b2d_select_k_workspace_bytes(100000, 1024, 32) == 0            # whole rows sorted on chip
    assert L.b2d_select_k_workspace_bytes(16384, 100000, 1024) == 0         # one CTA per row, sort on chip
    assert L.b2d_select_k_workspace_bytes(1, 2 ** 28, 1024) >= 1024 * 8 + 2048 * 4   # split row: list + histogram
    assert L.b2d_select_k_workspace_bytes(100, 100000, 50000) >= 2 * 100 * 50000 * 8   # segmented sort: list + alt


def test_argument_errors():
    L = _lib.lib()
    ok_ptr = 256
    args = lambda ld, rows, n, k: (None, ok_ptr, ld, None, rows, n, k, 1, ok_ptr, ok_ptr, None, 0)   # noqa: E731
    assert L.b2d_select_k(*args(10, 4, 10, 0)) == _lib.B2D_ERR_INVALID_ARG
    assert L.b2d_select_k(*args(10, 4, 10, 11)) == _lib.B2D_ERR_INVALID_ARG
    assert L.b2d_select_k(*args(8, 4, 10, 3)) == _lib.B2D_ERR_INVALID_ARG           # ld < len
    assert L.b2d_select_k(*args(2 ** 31, 4, 2 ** 31, 3)) == _lib.B2D_ERR_UNSUPPORTED
    assert L.b2d_select_k(*args(10, 0, 10, 3)) == _lib.B2D_OK                       # no rows: nothing to do
    assert L.b2d_select_k(None, None, 10, None, 4, 10, 3, 1, None, None, None, 0) == _lib.B2D_ERR_INVALID_ARG
    rc = L.b2d_select_k(None, ok_ptr, 200000, None, 2, 200000, 5, 1, ok_ptr, ok_ptr, None, 0)
    assert rc == _lib.B2D_ERR_WORKSPACE
    with pytest.raises(_lib.LogicError):
        _lib.check(L.b2d_select_k(*args(10, 4, 10, 0)))


SPECIAL = [0x00000000, 0x80000000, 0x00000001, 0x80000001, 0x007FFFFF, 0x807FFFFF, 0x00800000, 0x80800000,
           0x3F800000, 0xBF800000, 0x7F7FFFFF, 0xFF7FFFFF, 0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00000,
           0x7F800001, 0xFF800001, 0x7FFFFFFF, 0xFFFFFFFF]


def test_key_transform_matches_oracle(build_dir):
    exe = cpp_build.build("select_k_key_test.cu", os.path.join(build_dir, "select_k_key_test"), standalone=True)
    bits = np.concatenate([np.array(SPECIAL, dtype=np.uint32),
                           np.random.default_rng(5).integers(0, 2 ** 32, 20000, dtype=np.uint64).astype(np.uint32)])
    res = subprocess.run([exe], input="\n".join("%08x" % b for b in bits), capture_output=True, text=True, timeout=60)
    assert res.returncode == 0, res.stderr
    got = np.array([[int(t, 16) for t in line.split()] for line in res.stdout.split("\n") if line], dtype=np.uint32)
    v = bits.view(np.float32)
    assert (got[:, 0] == select_key(v, True)).all()
    assert (got[:, 1] == select_key(v, False)).all()


def test_oracle_order():
    v = np.array([[0.5, np.nan, -0.0, 0.0, -np.inf, np.inf, -np.nan, 1e-45, -1e-45, -2.0]], dtype=np.float32)
    vals, idx = ref_select_k(v, 10, select_min=True)
    assert idx[0].tolist() == [4, 9, 8, 2, 3, 7, 0, 5, 1, 6]
    assert np.signbit(vals[0, 3]) and not np.signbit(vals[0, 4])          # the input bits come back unchanged
    vals, idx = ref_select_k(v, 10, select_min=False)
    assert idx[0].tolist() == [1, 6, 5, 0, 7, 2, 3, 8, 9, 4]
    # against a plain stable sort on random data with ties, with a payload
    rng = np.random.default_rng(1)
    x = rng.integers(-5, 5, (7, 300)).astype(np.float32)
    pay = rng.integers(0, 10 ** 9, x.shape)
    for sel_min in (True, False):
        _, i = ref_select_k(x, 40, select_min=sel_min, in_idx=pay)
        order = np.argsort(x if sel_min else -x, axis=1, kind="stable")[:, :40]
        assert (i == np.take_along_axis(pay, order, 1)).all()


def compile_shim(build_dir, mock_raft):
    exe = os.path.join(build_dir, "select_k_shim_mockraft" if mock_raft else "select_k_shim")
    return cpp_build.build("select_k_shim_test.cu", exe, mock_raft)


@pytest.mark.parametrize("mock_raft", [False, True])
def test_shim_compiles(build_dir, mock_raft):
    assert os.path.exists(compile_shim(build_dir, mock_raft))


@pytest.mark.gpu
@pytest.mark.parametrize("mock_raft", [False, True])
def test_shim_runs_on_gpu(build_dir, mock_raft):
    exe = compile_shim(build_dir, mock_raft)
    res = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert res.returncode == 0 and "PASS" in res.stdout, res.stdout + res.stderr
