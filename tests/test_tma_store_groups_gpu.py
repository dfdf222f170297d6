"""GPU tier: the column-group edges of the staged TMA-store epilogue.

The result leaves the kernel in boxes of 32 rows x 64 columns through a 3-D view of dist (32 columns x column group x
row) that holds the n // 32 whole column groups only; when n % 32 != 0 the box holding the last, partial group also goes
out through a second view, n % 32 columns wide.  The partial group can be the first or the second group of its box
(n // 32 even or odd), and there may be no whole group at all (n < 32).  Each case checks the values against the fp64 oracle and that nothing is written
into the padding of a wider leading dimension or into the rows below the matrix."""
import pytest
import torch

import oracle
from oracle import DistanceType as DT
from raft_b200.distance import pairwise_distance
from test_pairwise_paths_gpu import plan_of

pytestmark = pytest.mark.gpu
EPS = 1e-4
SENTINEL = -7.0


@pytest.mark.parametrize("n", [4, 28, 36, 60, 164, 196, 220, 256])   # n // 32 = 0, 0, 1, 1, 5, 6, 6, 8
@pytest.mark.parametrize("k", [64, 200])                              # resident y block / streamed operands
def test_partial_column_group_with_padding(n, k):
    m, ld = 70, n + 12                                                # 70 = 2 x 32 + 6: a ragged last box of rows
    x, _, c = oracle.make_blobs(m, k, seed=1357 + n)
    y, _, _ = oracle.make_blobs(n, k, seed=7531 + n, centers=c)
    buf = torch.full((m + 40, ld), SENTINEL, device="cuda")
    xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    assert plan_of(DT.L2SqrtExpanded, xd, yd, buf[:m, :n])["stores"] == "tma"
    pairwise_distance(xd, yd, out=buf[:m, :n], metric=DT.L2SqrtExpanded)
    got = buf.cpu().numpy()
    ok, msg = oracle.match_approx(got[:m, :n], oracle.pairwise_distance(x, y, DT.L2SqrtExpanded), EPS)
    assert ok, msg
    assert (got[:m, n:] == SENTINEL).all()
    assert (got[m:] == SENTINEL).all()
