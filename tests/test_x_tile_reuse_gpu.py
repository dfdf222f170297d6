"""GPU tier: the resident tensor-core kernel loads each x tile once for both halves of a y block.

With k <= 128 a work item keeps its 256-row y block in shared memory and walks a run of 128-row x tiles; both 128-column
halves of the y block read the same staged x k-blocks, and only the last half releases them.  These tests run that ring
where it wraps mid-tile (nkb = 1, 3 against 4 or 5 stages), where the last y block has one half only, where items run
several x tiles, with one to three y blocks, and through every epilogue: stored distances (TMA and register stores),
the exact and the screened fusedL2NN, and the fused kNN with its sub-range passes."""
import numpy as np
import pytest
import torch

import oracle
from oracle import DistanceType as DT
from raft_b200.distance import fused_l2_nn, pairwise_distance
from raft_b200.neighbors import brute_force

pytestmark = pytest.mark.gpu
EPS = 1e-4


def blobs(m, n, k, seed=0):
    x, _, c = oracle.make_blobs(m, k, seed=1357 + seed)
    y, _, _ = oracle.make_blobs(n, k, seed=7531 + seed, centers=c)
    return x, y


def check(got, ref, eps=EPS):
    ok, msg = oracle.match_approx(got, ref, eps)
    assert ok, msg


def check_nn_indices(gi, ri, x, y):
    """The arg-min must be the oracle's index; where it is not, the two rows must be a near-tie that the fp32 expanded
    form cannot separate (fp64 distances within 1e-5 relative), and such rows must be rare."""
    bad = np.nonzero(gi != ri)[0]
    assert len(bad) <= max(1, len(gi) // 2000), f"{len(bad)} index mismatches"
    for i in bad:
        d_got = ((x[i].astype(np.float64) - y[gi[i]].astype(np.float64)) ** 2).sum()
        d_ref = ((x[i].astype(np.float64) - y[ri[i]].astype(np.float64)) ** 2).sum()
        assert abs(d_got - d_ref) <= 1e-5 * max(d_ref, 1.0), (i, gi[i], ri[i], d_got, d_ref)


# 41000 rows = 321 x tiles against 5 y blocks: 1605 tile pairs, more than 6 per SM, so every item runs 2 x tiles
@pytest.mark.parametrize("k", [32, 96, 128])       # nkb = 1, 3, 4 against 4 x stages
@pytest.mark.parametrize("n", [1124, 1280, 1125])  # last y block one half / whole / one half with register stores
def test_pairwise_many_tiles_per_item(k, n):
    m = 41000
    x, y = blobs(m, n, k)
    got = pairwise_distance(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), metric=DT.L2Expanded).copy_to_host()
    check(got, oracle.pairwise_distance(x, y, DT.L2Expanded))


@pytest.mark.parametrize("n", [200, 400, 700])     # 1, 2, 3 y blocks
@pytest.mark.parametrize("m", [100, 5000])         # one x tile (fewer items than SMs) / many
def test_pairwise_few_y_blocks(m, n):
    k = 96
    x, y = blobs(m, n, k, seed=1)
    got = pairwise_distance(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), metric=DT.L2SqrtExpanded).copy_to_host()
    check(got, oracle.pairwise_distance(x, y, DT.L2SqrtExpanded))


@pytest.mark.parametrize("k", [32, 96, 128])       # nkb = 1, 3, 4 against 5 x stages
@pytest.mark.parametrize("n", [2660, 2816])        # last y block one half / whole
def test_fused_l2_nn_exact(k, n):
    m = 30000
    x, y = blobs(m, n, k, seed=2)
    ri, rv = oracle.fused_l2_nn(x, y, sqrt=False)
    gi, gv = fused_l2_nn(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), sqrt=False)
    gi, gv = gi.cpu().numpy(), gv.cpu().numpy()
    check_nn_indices(gi, ri, x, y)
    check(gv, rv)


@pytest.mark.parametrize("k", [96, 128])           # screened: the sel_s = 32 subsets run through the resident kernel
def test_fused_l2_nn_screened(k):
    m, n = 3000, 256 * 80 + 100
    x, y = blobs(m, n, k, seed=3)
    ri, rv = oracle.fused_l2_nn(x, y, sqrt=False)
    gi, gv = fused_l2_nn(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), sqrt=False)
    gi, gv = gi.cpu().numpy(), gv.cpu().numpy()
    check_nn_indices(gi, ri, x, y)
    check(gv, rv)


@pytest.mark.parametrize("k", [32, 96, 128])
def test_knn_sub_range_passes(k):
    # 5220 database rows: passes of 128, 128, 256, ... rows, the last one a ragged sub-range
    m, n, kk = 3000, 256 * 20 + 100, 16
    x, y = blobs(m, n, k, seed=4)
    gd, gi = brute_force.knn(torch.from_numpy(y).cuda(), torch.from_numpy(x).cuda(), k=kk)
    gd, gi = gd.cpu().numpy(), gi.cpu().numpy()
    ri, rv = oracle.knn_l2(x, y, kk)
    true_d = ((x[:, None, :].astype(np.float64) - y[gi].astype(np.float64)) ** 2).sum(-1)
    check(gd, rv)
    check(gd, true_d)
    assert all(len(set(r.tolist())) == kk for r in gi)
    assert (gi != ri).mean() < 0.01
