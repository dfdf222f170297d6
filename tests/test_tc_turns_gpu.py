"""GPU tier: the resident tensor-core kernel (k <= 128) with one x ring per consumer warpgroup and ordered MMA turns.

Each consumer warpgroup reads the 64-row slab of every x tile from a ring of its own, fed by a producer warp of its own,
and the two warpgroups take turns issuing their MMAs.  These tests run what the protocol adds: a last x tile whose
second slab lies wholly outside the matrix (m % 128 <= 64) or is cut short; one item per CTA and grids smaller than the
SM count; items that end on a one-half y block; masked tiles that are NONE for slab 1 only, many tiles in a row.  Pairwise
results are checked against the fp64 oracle, arg-min and kNN results against exact references; the masked arg-min with
the per-row bound of test_masked_nn_paths_gpu.py."""
import numpy as np
import pytest
import torch

import oracle
from oracle import DistanceType as DT
from raft_b200.distance import fused_l2_nn, masked_l2_nn, pairwise_distance
from raft_b200.neighbors import brute_force
from test_masked_nn_paths_gpu import check as masked_check

pytestmark = pytest.mark.gpu
EPS = 1e-4


def blobs(m, n, k, seed=0):
    x, _, c = oracle.make_blobs(m, k, seed=2468 + seed)
    y, _, _ = oracle.make_blobs(n, k, seed=8642 + seed, centers=c)
    return x, y


def check(got, ref, eps=EPS):
    ok, msg = oracle.match_approx(got, ref, eps)
    assert ok, msg


def nn_indices_ok(gi, ri, x, y):
    """Indices equal the oracle's except at rare fp32 near-ties (fp64 distances within 1e-5 relative)."""
    bad = np.nonzero(gi != ri)[0]
    assert len(bad) <= max(1, len(gi) // 2000), f"{len(bad)} index mismatches"
    for i in bad:
        d_got = ((x[i].astype(np.float64) - y[gi[i]].astype(np.float64)) ** 2).sum()
        d_ref = ((x[i].astype(np.float64) - y[ri[i]].astype(np.float64)) ** 2).sum()
        assert abs(d_got - d_ref) <= 1e-5 * max(d_ref, 1.0), (i, gi[i], ri[i], d_got, d_ref)


@pytest.mark.parametrize("mrem", [1, 64, 65, 127])     # slab 1 of the last x tile: outside / outside / 1 row / 63 rows
@pytest.mark.parametrize("k", [32, 128])                # nkb = 1, 4
@pytest.mark.parametrize("n", [300, 1024])              # last y block one half / whole
def test_pairwise_ragged_last_tile(mrem, k, n):
    m = 128 * 9 + mrem
    x, y = blobs(m, n, k, seed=mrem)
    got = pairwise_distance(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), metric=DT.L2Expanded).copy_to_host()
    check(got, oracle.pairwise_distance(x, y, DT.L2Expanded))


@pytest.mark.parametrize("m,n", [(1, 100), (64, 256), (100, 300), (200, 700)])   # 1 to 6 items: one item per CTA
@pytest.mark.parametrize("metric", [DT.L2SqrtExpanded, DT.CosineExpanded])
def test_pairwise_one_item_per_cta(m, n, metric):
    x, y = blobs(m, n, 96, seed=5)
    got = pairwise_distance(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), metric=metric).copy_to_host()
    check(got, oracle.pairwise_distance(x, y, metric))


@pytest.mark.parametrize("mrem", [1, 64, 65, 127])
@pytest.mark.parametrize("n", [2660, 300])               # many y blocks / two, each run ending on a one-half y block
def test_fused_l2_nn_ragged(mrem, n):
    m = 128 * 40 + mrem
    x, y = blobs(m, n, 128, seed=7 + mrem)
    ri, rv = oracle.fused_l2_nn(x, y, sqrt=False)
    gi, gv = fused_l2_nn(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), sqrt=False)
    gi, gv = gi.cpu().numpy(), gv.cpu().numpy()
    nn_indices_ok(gi, ri, x, y)
    check(gv, rv)


@pytest.mark.parametrize("mrem", [1, 64, 127])
def test_knn_ragged(mrem):
    m, n, kk = 128 * 12 + mrem, 256 * 6 + 100, 16
    x, y = blobs(m, n, 128, seed=11 + mrem)
    gd, gi = brute_force.knn(torch.from_numpy(y).cuda(), torch.from_numpy(x).cuda(), k=kk)
    gd, gi = gd.cpu().numpy(), gi.cpu().numpy()
    true_d = ((x[:, None, :].astype(np.float64) - y[gi].astype(np.float64)) ** 2).sum(-1)
    ri, rv = oracle.knn_l2(x, y, kk)
    check(gd, rv)
    check(gd, true_d)
    assert all(len(set(r.tolist())) == kk for r in gi)
    assert (gi != ri).mean() < 0.01


@pytest.mark.parametrize("k", [64, 128])
@pytest.mark.parametrize("mrem", [0, 64])
def test_masked_slab1_none_runs(k, mrem):
    """The odd 64-row slab (warpgroup 1) of x tile t is adjacent to group 0 only unless t % 5 == 4; the even slab to every
    group.  Outside group 0 warpgroup 1 has runs of four tiles with nothing to multiply while warpgroup 0 multiplies every
    tile, so the two warpgroups' rings and turns run far apart in what they compute."""
    m, n = 128 * 80 + mrem, 8192 + 100
    x, y = blobs(m, n, k, seed=13)
    G = n // 1024 + 1
    gidx = np.minimum(np.arange(1024, 1024 * (G + 1), 1024), n).astype(np.int32)
    adj = np.ones((m, G), bool)
    for t in range((m + 127) // 128):
        if t % 5 != 4:
            adj[128 * t + 64:128 * t + 128, 1:] = False
    gi, gv = masked_l2_nn(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), torch.from_numpy(adj).cuda(),
                          torch.from_numpy(gidx).cuda())
    masked_check(x, y, adj, gidx, gi.cpu().numpy(), gv.cpu().numpy())     # every row, no count allowance
