"""radius_neighbors without a GPU: the fp64 CSR reference of the GPU tier (tests/radius_ref.py) pinned to sklearn, every
argument check of the two C calls with its status and message, the workspace query and its recorded contract
(tests/golden/radius_neighbors_workspace_contract.json), B2D_ERR_CUDA without a device, and the C++ shim's compile (its
run on the GPU is in tests/test_radius_neighbors_shim.py)."""
import os

import numpy as np
import pytest
import torch

import cpp_build
import oracle
from radius_ref import composition, dist64, ref_csr64
from raft_b200 import _lib
from test_workspace_contract import load, replay_bytes, replay_errors

SIZE_MAX = 2 ** 64 - 1
P = 1 << 12   # a non-null pointer that is never dereferenced (every call below fails before any work)
E, U, W = _lib.B2D_ERR_INVALID_ARG, _lib.B2D_ERR_UNSUPPORTED, _lib.B2D_ERR_WORKSPACE


def count(indptr=P, metric=0, x=P, ldx=8, y=P, ldy=8, m=10, n=100, k=8, r=1.0, ws=P * 256, wsb=1 << 40):
    return _lib.lib().b2d_radius_neighbors_count(None, indptr, metric, x, ldx, y, ldy, m, n, k, r, ws, wsb)


def fill(indptr=P, nnz=50, indices=P, distances=P, metric=0, x=P, ldx=8, y=P, ldy=8, m=10, n=100, k=8, r=1.0, ws=P * 256,
         wsb=1 << 40):
    return _lib.lib().b2d_radius_neighbors_fill(None, indptr, nnz, indices, distances, metric, x, ldx, y, ldy, m, n, k, r,
                                                ws, wsb)


def status(rc):
    return rc, _lib.lib().b2d_last_error().decode()


def test_workspace_query():
    L = _lib.lib()
    for args in ((-1, 5, 3, 0), (5, -1, 3, 0), (5, 5, -3, 0), (5, 5, 3, -1)):
        assert L.b2d_radius_neighbors_workspace_bytes(*args) == SIZE_MAX
    for m, n, k in ((1000, 2000, 32), (100000, 100000, 128), (7, 9, 320)):
        c = L.b2d_radius_neighbors_workspace_bytes(m, n, k, 0)
        # the tensor path's operands come first: at least what pairwise_distance needs
        assert c > L.b2d_pairwise_workspace_bytes(0, _lib.B2D_F32, m, n, k)
        # fill adds the second key buffer (8 bytes per pair) and the sort's scratch
        f = L.b2d_radius_neighbors_workspace_bytes(m, n, k, 2 ** 20)
        assert f >= c + 8 * 2 ** 20
        assert L.b2d_radius_neighbors_workspace_bytes(m, n, k, 2 ** 21) - f == 8 * 2 ** 20


def test_workspace_contract_bytes():
    rows = replay_bytes(load("radius_neighbors_workspace_contract.json"), "b2d_radius_neighbors_workspace_bytes")
    assert len(rows) == 9 * 2 * 8 * 5 + 5
    for *args, want in rows:
        assert (want == SIZE_MAX) == (min(args) < 0), args


def test_workspace_contract_errors():
    assert replay_errors(load("radius_neighbors_workspace_contract.json")) == 24


@pytest.mark.parametrize("call", [count, fill])
def test_argument_errors_shared(call):
    metrics = "radius_neighbors supports L2Expanded, L2SqrtExpanded, CosineExpanded and CorrelationExpanded, got metric "
    for bad in (-1, 3, 4, 5, 6, 7, 8, 9, 11, 13, 20):
        assert status(call(metric=bad)) == (U, metrics + str(bad))
    assert status(call(m=-1)) == (E, "negative extent")
    assert status(call(n=-1)) == (E, "negative extent")
    assert status(call(k=-1)) == (E, "negative extent")
    assert status(call(k=0)) == (E, "k must be positive")
    assert status(call(k=321, ldx=321, ldy=321)) == (U, "radius_neighbors supports k <= 320 (the whole distance at once)")
    assert status(call(indptr=None)) == (E, "null indptr")
    assert status(call(x=None)) == (E, "null x / y")
    assert status(call(y=None)) == (E, "null x / y")
    assert status(call(ldx=7)) == (E, "leading dimension smaller than k")
    assert status(call(ldy=7)) == (E, "leading dimension smaller than k")
    assert status(call(m=2 ** 31)) == (E, "m and n must be below 2^31")
    assert status(call(n=2 ** 31)) == (E, "m and n must be below 2^31")
    assert status(call(wsb=10))[0] == W
    assert status(call(ws=None))[0] == W
    assert status(call(ws=P * 256 + 16))[0] == E
    with pytest.raises(_lib.LogicError):
        _lib.check(call(k=321))


def test_argument_errors_fill():
    assert status(fill(nnz=-1)) == (E, "negative nnz")
    for nnz in (2 ** 31, 2 ** 40):
        assert status(fill(nnz=nnz)) == (U, "nnz = %d exceeds 2^31 - 1 pairs per call: split the queries into smaller "
                                            "batches" % nnz)
    assert status(fill(nnz=2 ** 31 - 1, wsb=10))[0] == W   # the largest nnz passes its own check
    assert status(fill(indices=None)) == (E, "null indices / distances")
    assert status(fill(distances=None)) == (E, "null indices / distances")
    # nnz = 0 needs no output buffers; the workspace is still checked
    assert status(fill(nnz=0, indices=None, distances=None, wsb=10))[0] == W


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the error without a device")
def test_cuda_error_without_device():
    assert count(m=0, x=None, y=None) == _lib.B2D_ERR_CUDA   # indptr[0] = 0 is the only work
    assert count() == _lib.B2D_ERR_CUDA
    assert fill() == _lib.B2D_ERR_CUDA
    # nothing to do at all: OK without touching the device
    assert fill(m=0, x=None, y=None) == _lib.B2D_OK
    assert fill(nnz=0, indices=None, distances=None) == _lib.B2D_OK
    assert fill(r=-1.0) == _lib.B2D_OK and fill(r=float("nan")) == _lib.B2D_OK


def _sklearn_csr(q, x, radius, metric):
    from sklearn.neighbors import NearestNeighbors
    nn = NearestNeighbors(radius=radius, metric=metric, algorithm="brute").fit(x.astype(np.float64))
    dist, ind = nn.radius_neighbors(q.astype(np.float64), sort_results=True)
    indptr = np.concatenate([[0], np.cumsum([len(r) for r in ind])]).astype(np.int64)
    return indptr, np.concatenate(ind).astype(np.int64), np.concatenate(dist)


@pytest.mark.parametrize("metric", ["euclidean", "cosine", "sqeuclidean"])
def test_reference_matches_sklearn(metric):
    q, _, c = oracle.make_blobs(60, 7, seed=5)
    x, _, _ = oracle.make_blobs(300, 7, seed=6, centers=c)
    d = dist64(q, x, metric)
    radius = float(np.quantile(d, 0.05))
    # no tied distances and nothing within 1e-9 of the radius: membership and order are unambiguous
    assert len(np.unique(d)) == d.size and np.abs(d - radius).min() > 1e-9
    indptr, indices, dists = ref_csr64(q, x, radius, metric)
    if metric == "sqeuclidean":   # sklearn's euclidean with the square root of the radius
        sk = _sklearn_csr(q, x, np.sqrt(radius), "euclidean")
        sk = (sk[0], sk[1], sk[2] ** 2)
    else:
        sk = _sklearn_csr(q, x, radius, metric)
    assert indptr[-1] > 500
    assert np.array_equal(indptr, sk[0]) and np.array_equal(indices, sk[1])
    assert np.allclose(dists, sk[2], rtol=1e-9, atol=1e-12)


def test_composition_orders_ties_by_index_and_negative_zero_first():
    d = np.array([[1.0, 0.5, 1.0, 0.0, -0.0, np.nan, 2.0]], np.float32)
    indptr, indices, dists = composition(d, 1.0)
    assert indptr.tolist() == [0, 5]
    assert indices.tolist() == [4, 3, 1, 0, 2]
    assert np.signbit(dists[0]) and not np.signbit(dists[1])
    for r in (-0.5, float("nan")):
        assert composition(d, r)[0].tolist() == [0, 0]
    assert composition(d, float("inf"))[0].tolist() == [0, 6]


def test_shim_compiles(tmp_path):
    for mock in (False, True):
        exe = str(tmp_path / ("radius_shim_mockraft" if mock else "radius_shim"))
        assert os.path.exists(cpp_build.build("radius_shim_test.cu", exe, mock))
