"""GPU tier: the staged TMA-store epilogue of the tensor-core pairwise kernel.

An aligned result leaves the kernel through shared-memory staging boxes of 64 rows x 32 columns and TMA stores; TMA
clips a box at the matrix bounds.  These tests pin what that path must not touch (rows below the matrix, the padding
of a wider leading dimension) and run enough tiles per CTA that every staging box is reused many times."""
import numpy as np
import pytest
import torch

import oracle
from oracle import DistanceType as DT
from raft_b200.distance import pairwise_distance

pytestmark = pytest.mark.gpu
EPS = 1e-4
SENTINEL = -7.0


def blobs(m, n, k, seed=0):
    x, _, c = oracle.make_blobs(m, k, seed=2468 + seed)
    y, _, _ = oracle.make_blobs(n, k, seed=8642 + seed, centers=c)
    return x, y


def check(got, ref, eps=EPS):
    ok, msg = oracle.match_approx(got, ref, eps)
    assert ok, msg


@pytest.mark.parametrize("k", [64, 200])   # resident y block / streamed operands
def test_rows_below_the_matrix_untouched(k):
    m, n = 200, 256                          # 200 = 3 x 64 + 8: the last staging box is mostly outside the matrix
    x, y = blobs(m, n, k)
    buf = torch.full((m + 64, n), SENTINEL, device="cuda")
    pairwise_distance(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), out=buf[:m], metric=DT.L2Expanded)
    got = buf.cpu().numpy()
    check(got[:m], oracle.pairwise_distance(x, y, DT.L2Expanded))
    assert (got[m:] == SENTINEL).all()


@pytest.mark.parametrize("n,ld", [(148, 160), (300, 304)])
def test_padding_of_a_wider_leading_dimension_untouched(n, ld):
    m, k = 130, 96
    x, y = blobs(m, n, k, seed=1)
    buf = torch.full((m, ld), SENTINEL, device="cuda")
    pairwise_distance(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), out=buf[:, :n], metric=DT.L2SqrtExpanded)
    got = buf.cpu().numpy()
    check(got[:, :n], oracle.pairwise_distance(x, y, DT.L2SqrtExpanded))
    assert (got[:, n:] == SENTINEL).all()


@pytest.mark.parametrize("metric", [DT.L2Expanded, DT.CosineExpanded, DT.InnerProduct])
@pytest.mark.parametrize("k", [128, 256])
def test_many_tiles_per_cta(metric, k):
    # 40 x 12 items of 128 x 256 on at most 132 CTAs: every CTA fills and reuses its staging ring many times
    m, n = 5000, 3000
    x, y = blobs(m, n, k, seed=2)
    got = pairwise_distance(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), metric=metric).copy_to_host()
    ref = oracle.pairwise_distance(x, y, metric)
    if metric == DT.InnerProduct:   # inner products cancel to ~0 for some pairs: compare against |x||y|
        scale = np.linalg.norm(x, axis=1)[:, None] * np.linalg.norm(y, axis=1)[None, :]
        assert np.max(np.abs(got - ref) / scale) < EPS
    else:
        check(got, ref)


def test_self_distance_diagonal_is_zero():
    x, _ = blobs(700, 1, 128, seed=3)
    xd = torch.from_numpy(x).cuda()
    got = pairwise_distance(xd, xd, metric=DT.L2Expanded).copy_to_host()
    assert (np.diag(got) == 0).all()
    check(got, oracle.pairwise_distance(x, x, DT.L2Expanded))
