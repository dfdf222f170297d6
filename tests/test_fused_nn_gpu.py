"""GPU tier: fusedL2NN (K3) and its sharded / packed-key building blocks against the oracle."""
import numpy as np
import pytest
import torch

import oracle
from raft_b200 import _lib
from raft_b200.common import DeviceResources
from raft_b200.distance import (fused_distance_nn, fused_l2_nn, fused_l2_nn_argmin, fused_l2_nn_sharded,
                                shard_bounds)

pytestmark = pytest.mark.gpu


def blobs(m, n, k, seed=0):
    x, _, c = oracle.make_blobs(m, k, seed=77 + seed)
    y, _, _ = oracle.make_blobs(n, k, seed=99 + seed, centers=c)
    return x, y


def tie_aware_index_check(gi, ri, x, y, tol=1e-5):
    """Indices must be bit-exact except where two candidates are closer than fp32 can separate;
    those are checked against the oracle's distance instead (SURVEY.md hard part D)."""
    bad = np.nonzero(gi != ri)[0]
    assert len(bad) <= max(1, len(gi) // 2000), f"{len(bad)} index mismatches"
    for i in bad:
        d_got = ((x[i].astype(np.float64) - y[gi[i]].astype(np.float64)) ** 2).sum()
        d_ref = ((x[i].astype(np.float64) - y[ri[i]].astype(np.float64)) ** 2).sum()
        assert abs(d_got - d_ref) <= tol * max(d_ref, 1.0), (i, d_got, d_ref)
    return len(bad)


@pytest.mark.parametrize("shape", [(1024, 1024, 32), (5000, 3000, 96), (777, 10000, 128), (300, 500, 200), (5, 3, 2)])
@pytest.mark.parametrize("sqrt", [False, True])
def test_fused_l2_nn_vs_oracle(shape, sqrt):
    x, y = blobs(*shape)
    ri, rv = oracle.fused_l2_nn(x, y, sqrt=sqrt)
    gi, gv = fused_l2_nn(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), sqrt=sqrt)
    gi, gv = gi.cpu().numpy(), gv.cpu().numpy()
    tie_aware_index_check(gi, ri, x, y)
    ok, msg = oracle.match_approx(gv, rv, 1e-4)
    assert ok, msg


def test_golden_nn(golden):
    for case in ("small", "cfg1"):
        x, y = golden[f"{case}_x"], golden[f"{case}_y"]
        gi, gv = fused_l2_nn(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), sqrt=False)
        assert (gi.cpu().numpy() == golden[f"{case}_nn_idx"]).all()
        assert oracle.match_approx(gv.cpu().numpy(), golden[f"{case}_nn_val"], 1e-4)[0]


@pytest.mark.parametrize("metric", ["sqeuclidean", "euclidean", "cosine", "correlation"])
def test_fused_distance_nn_metrics(metric):
    """raft::distance::fusedDistanceNN (SURVEY.md 8(f1)): arg-min under L2 and the cosine family."""
    x, y = blobs(900, 2100, 64, seed=5)
    mt = {"sqeuclidean": oracle.DistanceType.L2Expanded, "euclidean": oracle.DistanceType.L2SqrtExpanded,
          "cosine": oracle.DistanceType.CosineExpanded, "correlation": oracle.DistanceType.CorrelationExpanded}[metric]
    d = oracle.pairwise_distance(x, y, mt)
    ri, rv = d.argmin(axis=1), d.min(axis=1)
    gi, gv = fused_distance_nn(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), metric=metric)
    gi, gv = gi.cpu().numpy(), gv.cpu().numpy()
    bad = np.nonzero(gi != ri)[0]
    assert len(bad) <= 2
    for i in bad:   # near-ties only
        assert abs(d[i, gi[i]] - rv[i]) <= 1e-5 * max(rv[i], 1e-3)
    ok, msg = oracle.match_approx(gv, rv, 1e-4)
    assert ok, msg


def test_ties_go_to_smaller_index():
    """raft::argmin_op law (cpp/include/raft/core/operators.hpp:187-194): duplicates of the nearest
    database row in different tiles / chunks / halves -> the smallest index wins."""
    rng = np.random.default_rng(3)
    y = rng.standard_normal((2000, 48)).astype(np.float32) * 4
    x = y[[700, 31, 1500]] + 0.01
    for dup in ((700, 900, 1999), (31, 40, 300), (1500, 1501, 1755)):
        y[list(dup[1:])] = y[dup[0]]
    gi, _ = fused_l2_nn(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), sqrt=False)
    assert gi.cpu().tolist() == [700, 31, 1500]
    # all-identical database: index 0 for every query
    y0 = np.ones((1000, 16), np.float32)
    gi, gv = fused_l2_nn(torch.zeros(300, 16, device="cuda"), torch.from_numpy(y0).cuda(), sqrt=False)
    assert (gi == 0).all() and torch.allclose(gv, torch.full_like(gv, 16.0))


def test_argmin_wrapper_and_out():
    x, y = blobs(400, 600, 24)
    ri, _ = oracle.fused_l2_nn(x, y)
    out = torch.empty(400, dtype=torch.int32, device="cuda")
    ret = fused_l2_nn_argmin(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), out=out)
    assert ret is out and (out.cpu().numpy() == ri).all()
    ret2 = fused_l2_nn_argmin(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda())
    assert (ret2.copy_to_host() == ri).all()


def test_precomputed_norms_match():
    x, y = blobs(300, 700, 64)
    xt, yt = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    xn, yn = (xt * xt).sum(1), (yt * yt).sum(1)
    a = fused_l2_nn(xt, yt, sqrt=False)
    b = fused_l2_nn(xt, yt, sqrt=False, xn=xn, yn=yn)
    assert (a[0] == b[0]).all() and torch.allclose(a[1], b[1], rtol=1e-5, atol=1e-4)


def test_sharded_equals_unsharded_bit_for_bit():
    """SURVEY.md 8(e): each pair is evaluated by exactly one shard with a tiling-independent k
    order, so G-shard results equal the 1-shard result exactly.  Shards are played sequentially
    on one GPU here by accumulating into the same key buffer (atomicMin == all-reduce MIN)."""
    x, y = blobs(1500, 4099, 96)
    xt, yt = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    i1, v1 = fused_l2_nn(xt, yt, sqrt=False)
    L = _lib.lib()
    h = DeviceResources()
    m, k = x.shape
    for world in (2, 8):
        keys = torch.empty(m, dtype=torch.int64, device="cuda")
        kvp = torch.empty((m, 2), dtype=torch.int32, device="cuda")
        ws = None
        for r in range(world):
            lo, hi = shard_bounds(y.shape[0], world, r)
            ys = yt[lo:hi].contiguous()
            ws = h.workspace(L.b2d_fused_l2_nn_workspace_bytes(m, hi - lo, k))
            _lib.check(L.b2d_fused_l2_nn_keys(h.stream_ptr, keys.data_ptr(), xt.data_ptr(), k, ys.data_ptr(), k, None,
                                              None, m, hi - lo, k, lo, 1 if r == 0 else 0, ws.data_ptr(), ws.numel()))
        _lib.check(L.b2d_fused_l2_nn_finalize(h.stream_ptr, kvp.data_ptr(), keys.data_ptr(), m, 0, ws.data_ptr(), ws.numel()))
        h.sync()
        assert (kvp[:, 0] == i1).all()
        assert torch.equal(kvp[:, 1].view(torch.float32), v1)


def test_sharded_api_single_process():
    x, y = blobs(600, 2048, 32)
    ri, rv = oracle.fused_l2_nn(x, y, sqrt=True)
    gi, gv = fused_l2_nn_sharded(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), 0, sqrt=True)
    assert (gi.cpu().numpy() == ri).all()
    assert oracle.match_approx(gv.cpu().numpy(), rv, 1e-4)[0]


def test_row_norm_against_reference_spec():
    """raft::linalg::rowNorm (cpp/include/raft/linalg/norm.cuh:50-58): params of
    cpp/tests/linalg/norm.cu:237-240 (rows {11,1234} x cols {7,33,128,500}, tol 1e-5)."""
    L = _lib.lib()
    rng = np.random.default_rng(0)
    for rows in (11, 1234):
        for cols in (7, 33, 128, 500):
            x = rng.uniform(-1, 1, (rows, cols)).astype(np.float32)
            xt = torch.from_numpy(x).cuda()
            out = torch.empty(rows, device="cuda")
            for ntype, ref in ((1, np.abs(x.astype(np.float64)).sum(1)), (2, oracle.row_norm_sq(x)),
                               (3, np.abs(x).max(1))):
                _lib.check(L.b2d_row_norm(None, out.data_ptr(), xt.data_ptr(), cols, rows, cols, ntype, 0))
                torch.cuda.synchronize()
                assert oracle.match_approx(out.cpu().numpy(), ref, 1e-5)[0]
            _lib.check(L.b2d_row_norm(None, out.data_ptr(), xt.data_ptr(), cols, rows, cols, 2, 1))
            torch.cuda.synchronize()
            assert oracle.match_approx(out.cpu().numpy(), np.sqrt(oracle.row_norm_sq(x)), 1e-5)[0]


# ---- screened search (64 < k <= 128, n >= 16384): exact sub-sampled pass + coarse screen + exact
# re-evaluation of the candidates (raft_b200/csrc/screen_tc.cuh)

@pytest.mark.parametrize("shape", [(2000, 40000, 96), (1500, 20000, 128), (513, 33001, 70), (129, 16384, 65),
                                   (96, 50000, 96), (1, 16384, 128), (128, 70000, 80)])
@pytest.mark.parametrize("kind", ["blobs", "gauss"])
def test_screened_nn_vs_oracle(shape, kind):
    m, n, k = shape
    if kind == "blobs":
        x, y = blobs(m, n, k, seed=5)
    else:
        rng = np.random.default_rng(11)
        x = (rng.standard_normal((m, k)) * 3).astype(np.float32)
        y = (rng.standard_normal((n, k)) * 3 + 0.5).astype(np.float32)
    ri, rv = oracle.fused_l2_nn(x, y, sqrt=False)
    gi, gv = fused_l2_nn(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), sqrt=False)
    gi, gv = gi.cpu().numpy(), gv.cpu().numpy()
    tie_aware_index_check(gi, ri, x, y)
    ok, msg = oracle.match_approx(gv, rv, 1e-4)
    assert ok, msg


def test_screened_nn_ties_duplicates_and_wild_norms():
    """Duplicates of the nearest row in sampled and unsampled y blocks -> smallest index; rows whose
    norms differ by orders of magnitude keep the screening bound valid."""
    rng = np.random.default_rng(21)
    n, k = 40000, 96
    y = rng.standard_normal((n, k)).astype(np.float32) * 2
    y[::7] *= 50.0          # large-norm rows in every block
    y[3::11] *= 0.01        # tiny-norm rows
    q = [100, 300, 8200, 8447, 25000, 39999]   # blocks 0 (sampled), 1, 32 (sampled), 32, 97, 156
    x = y[q] + 1e-3
    y[[20000, 39000]] = y[100]     # later duplicates of a row in a sampled block
    y[[9000, 31000]] = y[300]      # later duplicates of a row in an unsampled block
    gi, gv = fused_l2_nn(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), sqrt=False)
    assert gi.cpu().tolist() == q
    ri, rv = oracle.fused_l2_nn(x, y, sqrt=False)
    assert (ri == np.array(q)).all()


def test_screened_nn_overflow_falls_back_to_exact():
    """All database rows identical: every column is a candidate, the list overflows and the exact
    kernel re-runs on the device -- same answer as the small case (index 0, distance k)."""
    y = np.ones((20000, 96), np.float32)
    gi, gv = fused_l2_nn(torch.zeros(700, 96, device="cuda"), torch.from_numpy(y).cuda(), sqrt=False)
    assert (gi == 0).all() and torch.allclose(gv, torch.full_like(gv, 96.0))
    # near-duplicates: 20000 rows within 1e-4 of each other, the true minimum hidden at a late index
    rng = np.random.default_rng(2)
    y = (np.ones((20000, 96)) + rng.standard_normal((20000, 96)) * 1e-4).astype(np.float32)
    x = rng.standard_normal((300, 96)).astype(np.float32)
    ri, rv = oracle.fused_l2_nn(x, y, sqrt=False)
    gi, gv = fused_l2_nn(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), sqrt=False)
    gi, gv = gi.cpu().numpy(), gv.cpu().numpy()
    # 20000 near-ties per row: the index is only defined up to fp32 resolution, the distance is not
    d_got = ((x.astype(np.float64) - y[gi].astype(np.float64)) ** 2).sum(1)
    assert np.all(np.abs(d_got - rv) <= 1e-5 * np.maximum(rv, 1.0))
    assert oracle.match_approx(gv, rv, 1e-4)[0]


def test_screened_sharded_matches_single():
    """Shards large enough to be screened themselves; the second shard starts from the first one's keys."""
    x, y = blobs(1000, 70000, 96, seed=9)
    xt, yt = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    i1, v1 = fused_l2_nn(xt, yt, sqrt=False)
    L = _lib.lib()
    h = DeviceResources()
    m, k = x.shape
    keys = torch.empty(m, dtype=torch.int64, device="cuda")
    kvp = torch.empty((m, 2), dtype=torch.int32, device="cuda")
    for r in range(2):
        lo, hi = shard_bounds(y.shape[0], 2, r)
        ys = yt[lo:hi].contiguous()
        ws = h.workspace(L.b2d_fused_l2_nn_workspace_bytes(m, hi - lo, k))
        _lib.check(L.b2d_fused_l2_nn_keys(h.stream_ptr, keys.data_ptr(), xt.data_ptr(), k, ys.data_ptr(), k, None,
                                          None, m, hi - lo, k, lo, 1 if r == 0 else 0, ws.data_ptr(), ws.numel()))
    _lib.check(L.b2d_fused_l2_nn_finalize(h.stream_ptr, kvp.data_ptr(), keys.data_ptr(), m, 0, ws.data_ptr(), ws.numel()))
    h.sync()
    assert (kvp[:, 0] == i1).all()
    assert torch.equal(kvp[:, 1].view(torch.float32), v1)


def test_sharded_head_exchange_path_matches_single():
    """fused_l2_nn_sharded's two-stage form (head of the shard, exchange of bounds, rest of the shard)
    visits every row once and returns what the one-call form returns."""
    rng = np.random.default_rng(13)
    x = (rng.standard_normal((1200, 96)) * 3).astype(np.float32)
    y = (rng.standard_normal((80000, 96)) * 3).astype(np.float32)
    xt, yt = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    i1, v1 = fused_l2_nn(xt, yt, sqrt=True)
    ri, rv = oracle.fused_l2_nn(x, y, sqrt=True)
    tie_aware_index_check(i1.cpu().numpy(), ri, x, y)
    for head in (0, 32768, 50000, 80000):
        i2, v2 = fused_l2_nn_sharded(xt, yt, 0, sqrt=True, head_rows=head)
        # every finalist of the screened search is measured with the same direct fp32 arithmetic
        assert (i2 == i1).all() and torch.equal(v2, v1)


def test_screened_nn_chunk_boundary():
    """Database larger than one 2^20-row chunk: second chunk continues from the first one's keys, its
    short remainder (< 16384 rows) takes the exact kernel; global indices on both sides of the boundary."""
    rng = np.random.default_rng(31)
    m, n, k = 96, (1 << 20) + 5000, 96
    y = (rng.standard_normal((n, k)) * 2).astype(np.float32)
    x = (rng.standard_normal((m, k)) * 2).astype(np.float32)
    targets = [5, (1 << 20) - 1, 1 << 20, n - 1, 700000, (1 << 20) + 4999]
    for i, t in enumerate(targets):
        x[i] = y[t] + 1e-3
    ri, rv = oracle.fused_l2_nn(x, y, sqrt=False, block=65536)
    gi, gv = fused_l2_nn(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), sqrt=False)
    gi, gv = gi.cpu().numpy(), gv.cpu().numpy()
    assert gi[: len(targets)].tolist() == targets
    tie_aware_index_check(gi, ri, x, y)
    # the planted neighbours sit 1e-3 away from rows of norm ~20: the short remainder chunk is measured by
    # the expanded form, whose cancellation floor is a few ulp of |x|^2 + |y|^2 (as in test_fuzz_gpu)
    floor = 16 * 2.0 ** -24 * ((x.astype(np.float64) ** 2).sum(1) + (y[gi].astype(np.float64) ** 2).sum(1))
    assert np.all(np.abs(gv - rv) <= 1e-4 * rv + floor)


def test_screened_nn_ragged_last_run_of_tiles():
    """129 query tiles in runs of 32: the last run is a single tile, so single-tile and multi-tile work items
    alternate on the same SM (the two MMA issuers must stay in step on every barrier)."""
    rng = np.random.default_rng(77)
    m, n, k = 16500, 40000, 96
    x = (rng.standard_normal((m, k)) * 2).astype(np.float32)
    y = (rng.standard_normal((n, k)) * 2).astype(np.float32)
    ri, rv = oracle.fused_l2_nn(x, y, sqrt=False)
    gi, gv = fused_l2_nn(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), sqrt=False)
    gi, gv = gi.cpu().numpy(), gv.cpu().numpy()
    tie_aware_index_check(gi, ri, x, y)
    assert oracle.match_approx(gv, rv, 1e-4)[0]


@pytest.mark.parametrize("metric", ["cosine", "correlation"])
@pytest.mark.parametrize("shape", [(700, 30000, 96), (96, 20000, 128), (300, 17000, 70)])
@pytest.mark.parametrize("kind", ["blobs", "gauss"])
def test_screened_cosine_family_nn(metric, shape, kind):
    """The screened search also serves the cosine family: rows are unit vectors after prep, the screen's
    margin is 1.05 * 2^-10 and the candidates are re-measured as 1 - <x', y'> / (|x'||y'|) in fp64."""
    m, n, k = shape
    if kind == "blobs":
        x, y = blobs(m, n, k, seed=21)
    else:
        rng = np.random.default_rng(5)
        x = (rng.standard_normal((m, k)) + 0.3).astype(np.float32)
        y = (rng.standard_normal((n, k)) + 0.3).astype(np.float32)
    mt = oracle.DistanceType.CosineExpanded if metric == "cosine" else oracle.DistanceType.CorrelationExpanded
    d = oracle.pairwise_distance(x, y, mt)
    ri, rv = d.argmin(axis=1), d.min(axis=1)
    gi, gv = fused_distance_nn(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), metric=metric)
    gi, gv = gi.cpu().numpy(), gv.cpu().numpy()
    bad = np.nonzero(gi != ri)[0]
    assert len(bad) <= max(2, m // 500)
    for i in bad:   # near-ties only
        assert abs(d[i, gi[i]] - rv[i]) <= 2e-5 * max(rv[i], 1e-3)
    # 1 - cos of near-parallel vectors: absolute floor of a few fp32 ulp of 1
    assert np.all(np.abs(gv - rv) <= 1e-4 * np.abs(rv) + 4e-7)


@pytest.mark.parametrize("n", [3000, 70000])
def test_fused_l2_nn_with_outlier_rows(n):
    """Sentinel rows (1e9) in the queries and in the database: ordinary rows must still find their exact nearest
    neighbour (per-row exponents, prep.cuh); with n = 70000 the screened search sees rows of y with their own
    exponent and must hand over to the exact kernel."""
    rng = np.random.default_rng(5)
    x = rng.standard_normal((1500, 96)).astype(np.float32)
    y = rng.standard_normal((n, 96)).astype(np.float32)
    x[3] *= 1.0e9
    y[n // 2] *= 1.0e9
    y[7] *= 2.0e8
    ri, rv = oracle.fused_l2_nn(x, y, sqrt=False)
    gi, gv = fused_l2_nn(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), sqrt=False)
    gi, gv = gi.cpu().numpy(), gv.cpu().numpy()
    tie_aware_index_check(gi, ri, x, y)
    ok, msg = oracle.match_approx(gv, rv, 1e-4)
    assert ok, msg
