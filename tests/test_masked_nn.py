"""CPU tier: masked_l2_nn -- the fp64 reference against a brute force, the C ABI's argument checks and workspace query,
the tile classification and the kernel's skip schedule (host replay), and the C++ shim's compile."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch
from scipy.spatial.distance import cdist

import cpp_build
from masked_nn_ref import FLT_MAX, NO_CANDIDATE, column_groups, masked_l2_nn as ref_masked_l2_nn, tile_classes
from raft_b200 import _lib


def brute(x, y, adj, gidx):
    d = cdist(x.astype(np.float64), y.astype(np.float64), "sqeuclidean")
    grp = column_groups(gidx, y.shape[0])
    ok = (grp >= 0)[None, :] & adj[:, np.maximum(grp, 0)]
    d = np.where(ok, d, np.inf)
    idx = np.argmin(d, axis=1)
    val = d[np.arange(len(x)), idx]
    idx = np.where(np.isfinite(val), idx, NO_CANDIDATE)
    return idx, np.where(np.isfinite(val), val, FLT_MAX)


def test_reference_against_brute_force():
    rng = np.random.default_rng(0)
    x = rng.integers(-3, 4, size=(120, 5)).astype(np.float32)      # small integers: many exact ties
    y = rng.integers(-3, 4, size=(400, 5)).astype(np.float32)
    y[350] = y[10]                                                  # the same point in two groups
    gidx = np.array([0, 50, 50, 200, 260, 380], dtype=np.int32)     # empty groups; the last ends before n
    adj = rng.random((120, 6)) < 0.4
    adj[:7] = False                                                 # rows without any adjacent group
    adj[7:20] = False
    adj[7:20, 5] = True                                             # only group 5 (rows 260..379): 350 and not 10
    x[7:20] = y[10]
    ri, rv = ref_masked_l2_nn(x, y, adj, gidx, block=64)
    bi, bv = brute(x, y, adj, gidx)
    assert (ri == bi).all()
    np.testing.assert_allclose(rv, bv, rtol=1e-12, atol=1e-9)
    assert (ri[:7] == NO_CANDIDATE).all() and (rv[:7] == FLT_MAX).all()
    assert (ri[7:20] == 350).all()
    # the tie across an adjacent and a non-adjacent group resolves to the adjacent one; among adjacent ones the smaller
    adj2 = np.zeros_like(adj)
    adj2[:, [0, 1, 3, 4, 5]] = True
    ri2, _ = ref_masked_l2_nn(x, y, adj2, gidx)
    assert (ri2[7:20] == 10).all()
    ri3, rv3 = ref_masked_l2_nn(x, y, adj, gidx, sqrt=True)
    assert (ri3 == ri).all() and np.allclose(rv3[rv < FLT_MAX], np.sqrt(rv[rv < FLT_MAX]))


def test_reference_nan_distances_never_win():
    """A NaN distance is no candidate (the library's NaN rule): a NaN row of y in an adjacent group must not hide the
    finite minimum of its block, and a row whose only adjacent row of y is NaN has no candidate."""
    x = np.array([[0, 0]], dtype=np.float32)
    y = np.array([[np.nan, 0], [1, 0], [3, 0]], dtype=np.float32)
    ri, rv = ref_masked_l2_nn(x, y, np.ones((1, 1), bool), np.array([3], np.int32))
    assert ri.tolist() == [1] and rv.tolist() == [1.0]
    ri, rv = ref_masked_l2_nn(x, y, np.ones((1, 1), bool), np.array([3], np.int32), sqrt=True)
    assert ri.tolist() == [1] and rv.tolist() == [1.0]
    # groups {0} (the NaN row) and {1, 2}: adjacent to the NaN row alone -> the sentinel; to both -> index 1
    gidx = np.array([1, 3], np.int32)
    x2 = np.array([[0, 0], [0, 0], [np.nan, 0]], dtype=np.float32)
    adj = np.array([[1, 0], [1, 1], [1, 1]], bool)
    ri, rv = ref_masked_l2_nn(x2, y, adj, gidx, block=2)
    assert ri.tolist() == [NO_CANDIDATE, 1, NO_CANDIDATE] and rv.tolist() == [FLT_MAX, 1.0, FLT_MAX]


def test_workspace_query():
    L = _lib.lib()
    base = L.b2d_masked_l2_nn_workspace_bytes(1000, 2000, 64, 10)
    assert base > 0 and base % 1024 == 0
    assert L.b2d_masked_l2_nn_workspace_bytes(1000, 2000, 64, 500) > base          # the adjacency bits grow with G
    assert L.b2d_masked_l2_nn_workspace_bytes(1000, 4000, 64, 10) > base
    assert L.b2d_masked_l2_nn_workspace_bytes(0, 0, 1, 0) >= 0
    for bad in ((-1, 2, 3, 4), (1, -2, 3, 4), (1, 2, -3, 4), (1, 2, 3, -4)):
        assert L.b2d_masked_l2_nn_workspace_bytes(*bad) == 2 ** 64 - 1


def _call(L, m=64, n=100, k=8, G=3, adj=1, gidx=1, ld_adj=None, ws_bytes=None, out=1):
    ws = ctypes.create_string_buffer(1 << 20)
    addr = (ctypes.addressof(ws) + 255) // 256 * 256
    p = 0x10000                                    # never dereferenced: the call must fail before touching memory
    return L.b2d_masked_l2_nn(None, p if out else None, p, k, p, k, None, None, p if adj else None,
                              G if ld_adj is None else ld_adj, p if gidx else None, G, m, n, k, 0, 1, addr,
                              (1 << 20) - 256 if ws_bytes is None else ws_bytes)


def test_invalid_arguments():
    L = _lib.lib()
    assert _call(L, m=-1) == _lib.B2D_ERR_INVALID_ARG
    assert _call(L, n=-1) == _lib.B2D_ERR_INVALID_ARG
    assert _call(L, G=-1, ld_adj=0) == _lib.B2D_ERR_INVALID_ARG
    assert _call(L, adj=0) == _lib.B2D_ERR_INVALID_ARG
    assert _call(L, gidx=0) == _lib.B2D_ERR_INVALID_ARG
    assert _call(L, ld_adj=2) == _lib.B2D_ERR_INVALID_ARG
    assert _call(L, out=0) == _lib.B2D_ERR_INVALID_ARG
    assert _call(L, k=0) == _lib.B2D_ERR_INVALID_ARG
    assert _call(L, n=2 ** 31) == _lib.B2D_ERR_INVALID_ARG
    assert _call(L, m=2 ** 31) == _lib.B2D_ERR_INVALID_ARG
    assert _call(L, ws_bytes=16) == _lib.B2D_ERR_WORKSPACE
    assert _call(L, m=0) == _lib.B2D_OK                 # nothing to do


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the error path of a machine without a GPU")
def test_valid_arguments_without_gpu_report_cuda_error():
    L = _lib.lib()
    assert _call(L) == _lib.B2D_ERR_CUDA
    assert _call(L, G=0, adj=0, gidx=0, ld_adj=0) == _lib.B2D_ERR_CUDA


@pytest.fixture(scope="module")
def schedule_exe(tmp_path_factory):
    return cpp_build.build("masked_schedule_test.cu", str(tmp_path_factory.mktemp("cpp") / "masked_schedule_test"),
                           standalone=True)


def _classify(exe, adj, gidx, m, n):
    lines = [f"{m} {n} {len(gidx)}", " ".join(str(int(v)) for v in gidx)]
    lines += ["".join("1" if v else "0" for v in row) for row in adj] if len(gidx) else []
    res = subprocess.run([exe, "classify"], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=60)
    assert res.returncode == 0, res.stderr
    return np.array([[int(c) for c in ln] for ln in res.stdout.split()], dtype=np.int64).reshape((m + 63) // 64, -1)


def test_tile_classes_match_numpy(schedule_exe):
    rng = np.random.default_rng(5)
    cases = 0
    for m, n in ((64, 128), (65, 129), (200, 700), (129, 1000), (33, 250)):
        for layout in ("tiny", "straddle", "short", "empty"):
            if layout == "tiny":
                sizes = rng.integers(1, 8, size=n)
            elif layout == "straddle":
                sizes = rng.integers(60, 200, size=n // 60 + 2)
            elif layout == "short":
                sizes = np.array([n // 3, 0, n // 4])
            else:
                sizes = np.array([0, 0, n, 0])
            gidx = np.minimum(np.cumsum(sizes), n).astype(np.int32)
            G = len(gidx)
            for p in (0.0, 0.3, 0.9, 1.0):
                adj = rng.random((m, G)) < p
                if p == 0.3:                       # whole slabs all / none adjacent to some groups
                    adj[:64, : G // 2] = True
                    adj[64:, G // 2:] = False
                got = _classify(schedule_exe, adj, gidx, m, n)
                assert (got == tile_classes(adj, gidx, m, n)).all(), (m, n, layout, p)
                cases += 1
    assert cases == 80


def test_skip_schedule_replay(schedule_exe):
    res = subprocess.run([schedule_exe], capture_output=True, text=True, timeout=120)
    assert res.returncode == 0 and "PASS" in res.stdout, res.stdout + res.stderr


def test_masked_shim_compiles_and_links(tmp_path):
    assert os.path.exists(cpp_build.build("masked_nn_test.cu", str(tmp_path / "masked_nn_test")))
