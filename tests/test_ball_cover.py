"""neighbors.ball_cover without a GPU: every argument check of the five C calls with its status and message, the size
queries and their recorded contract (tests/golden/ball_cover_workspace_contract.json), B2D_ERR_CUDA without a device,
the oracle of the GPU tier on small hand-made cases, and the C++ shim's compile (its run on the GPU is in
tests/test_ball_cover_shim.py)."""
import os

import numpy as np
import pytest
import torch

import ball_cover_ref as ref
import cpp_build
from raft_b200 import _lib
from test_workspace_contract import load, replay_bytes, replay_errors

SIZE_MAX = 2 ** 64 - 1
P = 1 << 12      # a non-null pointer that is never dereferenced (every call below fails before any work)
IX = 1 << 20     # a 256-byte aligned one for the index
E, U, W = _lib.B2D_ERR_INVALID_ARG, _lib.B2D_ERR_UNSUPPORTED, _lib.B2D_ERR_WORKSPACE


def L():
    return _lib.lib()


def build(index=IX, x=P, ldx=2, n=100, d=2, metric=5, nl=0, seed=1, ws=P * 256, wsb=1 << 40):
    return L().b2d_ball_cover_build(None, index, x, ldx, n, d, metric, nl, seed, ws, wsb)


def knn(oi=P, od=P, index=IX, n=100, d=2, metric=5, nl=0, q=P, ldq=2, m=10, k=5):
    return L().b2d_ball_cover_knn(None, oi, od, index, n, d, metric, nl, q, ldq, m, k)


def count(indptr=P, index=IX, n=100, d=2, metric=5, nl=0, q=P, ldq=2, m=10, eps=0.5, ws=P * 256, wsb=1 << 40):
    return L().b2d_ball_cover_eps_count(None, indptr, index, n, d, metric, nl, q, ldq, m, eps, ws, wsb)


def fill(indptr=P, nnz=50, indices=P, distances=P, index=IX, n=100, d=2, metric=5, nl=0, q=P, ldq=2, m=10, eps=0.5,
         ws=P * 256, wsb=1 << 40):
    return L().b2d_ball_cover_eps_fill(None, indptr, nnz, indices, distances, index, n, d, metric, nl, q, ldq, m, eps,
                                       ws, wsb)


def status(rc):
    return rc, L().b2d_last_error().decode()


def test_size_queries():
    for args in ((0, 2, 0), (-1, 2, 0), (2 ** 31, 2, 0), (10, 1, 0), (10, 4, 0), (10, 2, -1), (10, 2, 11)):
        assert L().b2d_ball_cover_index_bytes(*args) == SIZE_MAX
        assert L().b2d_ball_cover_build_workspace_bytes(*args) == SIZE_MAX
    for n, d in ((1, 2), (1000, 3), (10 ** 6, 2)):
        full = L().b2d_ball_cover_index_bytes(n, d, 0)
        # the points (d + 2 words per row: coordinates, row id, s to the landmark) and the balls (d + 2 words each)
        assert full >= 4 * n * (d + 2)
        assert L().b2d_ball_cover_index_bytes(n, d, n) >= full + 4 * (n - int(np.ceil(np.sqrt(n)))) * (d + 1)
        # the default is ceil(sqrt(n)) landmarks
        assert L().b2d_ball_cover_index_bytes(n, d, int(np.ceil(np.sqrt(n)))) == full
        # two key and two value buffers of the sorts, and their scratch
        assert L().b2d_ball_cover_build_workspace_bytes(n, d, 0) >= 24 * n
    assert L().b2d_ball_cover_eps_workspace_bytes(-1, 0) == SIZE_MAX
    assert L().b2d_ball_cover_eps_workspace_bytes(5, -1) == SIZE_MAX
    assert L().b2d_ball_cover_eps_workspace_bytes(1000, 2 ** 20) - L().b2d_ball_cover_eps_workspace_bytes(1000, 2 ** 19) \
        == 8 * 2 ** 19


def test_workspace_contract_bytes():
    c = load("ball_cover_workspace_contract.json")
    for fn in ("b2d_ball_cover_index_bytes", "b2d_ball_cover_build_workspace_bytes"):
        for n, d, nl, want in replay_bytes(c, fn):
            assert (want == SIZE_MAX) == (not (1 <= n < 2 ** 31 and d in (2, 3) and 0 <= nl <= n)), (fn, n, d, nl)
    for m, nnz, want in replay_bytes(c, "b2d_ball_cover_eps_workspace_bytes"):
        assert (want == SIZE_MAX) == (min(m, nnz) < 0)


def test_workspace_contract_errors():
    assert replay_errors(load("ball_cover_workspace_contract.json")) == 4 * 3 * 3


INDEX_ERRORS = [
    (dict(metric=0), (U, "ball_cover supports L2Unexpanded and L2SqrtUnexpanded, got metric 0")),
    (dict(metric=1), (U, "ball_cover supports L2Unexpanded and L2SqrtUnexpanded, got metric 1")),
    (dict(metric=13), (U, "ball_cover supports L2Unexpanded and L2SqrtUnexpanded, got metric 13")),
    (dict(d=1), (U, "ball_cover supports d = 2 and d = 3, got d = 1")),
    (dict(d=4), (U, "ball_cover supports d = 2 and d = 3, got d = 4")),
    (dict(n=0), (E, "n must be positive")),
    (dict(n=-1), (E, "n must be positive")),
    (dict(n=2 ** 31), (E, "n must be below 2^31")),
    (dict(nl=-1), (E, "n_landmarks must be in [0, n] (0: ceil(sqrt(n)))")),
    (dict(nl=101), (E, "n_landmarks must be in [0, n] (0: ceil(sqrt(n)))")),
    (dict(index=None), (E, "null index")),
    (dict(index=IX + 16), (E, "index must be 256-byte aligned")),
]


@pytest.mark.parametrize("call", [build, knn, count, fill])
def test_index_argument_errors(call):
    for kw, want in INDEX_ERRORS:
        assert status(call(**kw)) == want, (call.__name__, kw)
    with pytest.raises(_lib.LogicError):
        _lib.check(call(d=4))


def test_build_argument_errors():
    assert status(build(x=None)) == (E, "null x")
    assert status(build(ldx=1)) == (E, "ldx smaller than d")
    assert status(build(d=3, ldx=2)) == (E, "ldx smaller than d")
    assert status(build(wsb=10))[0] == W
    assert status(build(ws=None))[0] == W
    assert status(build(ws=P * 256 + 16)) == (E, "workspace must be 256-byte aligned")


@pytest.mark.parametrize("call", [knn, count, fill])
def test_query_argument_errors(call):
    assert status(call(m=-1)) == (E, "negative extent")
    assert status(call(m=2 ** 31)) == (E, "m must be below 2^31")
    assert status(call(q=None)) == (E, "null queries")
    assert status(call(ldq=1)) == (E, "ldq smaller than d")


def test_knn_argument_errors():
    assert status(knn(k=0)) == (E, "k must be in [1, n]")
    assert status(knn(k=101)) == (E, "k must be in [1, n]")
    assert status(knn(n=10, k=11)) == (E, "k must be in [1, n]")
    assert status(knn(k=65)) == (U, "k > 64 is not supported")
    assert status(knn(oi=None)) == (E, "null out_idx / out_dist")
    assert status(knn(od=None)) == (E, "null out_idx / out_dist")


def test_eps_argument_errors():
    for call in (count, fill):
        assert status(call(indptr=None)) == (E, "null indptr")
        assert status(call(wsb=10))[0] == W
    assert status(fill(nnz=-1)) == (E, "negative nnz")
    for nnz in (2 ** 31, 2 ** 40):
        assert status(fill(nnz=nnz)) == (U, "nnz = %d exceeds 2^31 - 1 pairs per call: split the queries into smaller "
                                            "batches" % nnz)
    assert status(fill(nnz=2 ** 31 - 1, wsb=10))[0] == W
    assert status(fill(indices=None)) == (E, "null indices / distances")
    assert status(fill(distances=None)) == (E, "null indices / distances")


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the error without a device")
def test_cuda_error_without_device():
    assert build() == _lib.B2D_ERR_CUDA
    assert knn() == _lib.B2D_ERR_CUDA
    assert count() == _lib.B2D_ERR_CUDA
    assert count(m=0, q=None) == _lib.B2D_ERR_CUDA      # indptr[0] = 0 is the only work
    assert count(eps=-1.0) == _lib.B2D_ERR_CUDA         # indptr = 0
    assert fill() == _lib.B2D_ERR_CUDA
    # nothing to do at all: OK without touching the device
    assert knn(m=0, q=None, oi=None, od=None) == _lib.B2D_OK
    assert fill(m=0, q=None) == _lib.B2D_OK
    assert fill(nnz=0, indices=None, distances=None) == _lib.B2D_OK
    assert fill(eps=float("nan")) == _lib.B2D_OK and fill(eps=-1.0) == _lib.B2D_OK


def test_oracle_on_hand_made_points():
    x = torch.tensor([[0.0, 0.0], [1.0, 0.0], [0.0, 1.0], [float("nan"), 0.0], [3.0, 4.0]])
    q = torch.tensor([[0.0, 0.0], [float("nan"), 1.0], [0.5, 0.5]])
    i, d = ref.knn(q, x, 5, "euclidean")
    assert i.tolist() == [[0, 1, 2, 4, -1], [-1] * 5, [0, 1, 2, 4, -1]]
    assert d[0].tolist() == [0.0, 1.0, 1.0, 5.0, float("inf")]
    indptr, idx, dist = ref.eps_csr(q, x, 1.0, "sqeuclidean")
    assert indptr.tolist() == [0, 3, 3, 6] and idx.tolist() == [0, 1, 2, 0, 1, 2]
    assert dist.tolist() == [0.0, 1.0, 1.0, 0.5, 0.5, 0.5]
    # the contract's rounding: the three products and two sums each rounded on their own
    a = torch.tensor([[1e4 + 0.01, 1e4, 1e4]])
    b = torch.tensor([[1e4, 1e4 + 0.02, 1e4 + 0.03]])
    t = (a - b).numpy()[0]
    s = np.float32(np.float32(np.float32(t[0] * t[0]) + np.float32(t[1] * t[1])) + np.float32(t[2] * t[2]))
    assert ref.dist(a, b, "sqeuclidean").numpy()[0, 0] == s


def test_shim_compiles(tmp_path):
    for mock in (False, True):
        exe = str(tmp_path / ("ball_cover_shim_mockraft" if mock else "ball_cover_shim"))
        assert os.path.exists(cpp_build.build("ball_cover_shim_test.cu", exe, mock))
