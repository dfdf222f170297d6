"""GPU tier: parity AT THE BASELINE.json SHAPES (VERDICT r1, next #1).

The CPU oracle cannot visit 10^10 pairs, so every shape is checked by fp64 re-evaluation on the device
(oracle/device_check.py: the same definitions as oracle.py) of >= 2*10^5 sampled pairs including the corners of
the kernels' 128 x 256 tiles and the matrix edges; fusedL2NN by the exact fp64 arg-min of 65536 sampled queries
against the FULL 8M-row database.  Tolerance: 1e-4 relative with raft::CompareApprox's absolute-below-eps rule
(cpp/tests/test_utils.h:31-45); arg-min: strict index equality reported and bounded (>= 99.99 %), the rest must be
fp32-inseparable near-ties (tie law cpp/include/raft/core/operators.hpp:187-194).
Data: make_blobs-like (5 centres U[-10,10]^k, sigma 1), the benchmark's generator (SURVEY.md 8(d)).
"""
import pytest
import torch

from oracle import DistanceType as DT
from oracle import device_check as dc
from raft_b200.common import DeviceResources
from raft_b200.distance import fused_l2_nn, pairwise_distance

pytestmark = pytest.mark.gpu
EPS = 1e-4


def blobs(rows, cols, seed, centers):
    g = torch.Generator(device="cuda").manual_seed(seed)
    lab = torch.randint(0, centers.shape[0], (rows,), device="cuda", generator=g)
    out = torch.randn(rows, cols, device="cuda", generator=g)
    out += centers[lab]
    return out


def centers(cols):
    g = torch.Generator(device="cuda").manual_seed(42)
    return torch.rand(5, cols, device="cuda", generator=g) * 20.0 - 10.0


def free_gb():
    torch.cuda.empty_cache()                      # what an earlier test left in the caching allocator is free
    return torch.cuda.mem_get_info()[0] / 2 ** 30


@pytest.mark.parametrize("metric", [DT.L1, DT.L2Unexpanded, DT.Linf])
def test_config3_unexpanded_50k_x_50k_x_256(metric):
    if free_gb() < 14:
        pytest.skip("needs ~11 GB of free device memory")
    c = centers(256)
    x, y = blobs(50_000, 256, 1234, c), blobs(50_000, 256, 4321, c)
    out = torch.full((50_000, 50_000), float("nan"), dtype=torch.float32, device="cuda")
    pairwise_distance(x, y, out=out, metric=metric)
    r = dc.check_pairwise_sampled(out, x, y, metric, count=200_000, eps=EPS)
    assert r["n_bad"] == 0, r
    assert torch.isfinite(out[::127, ::131]).all()


def test_config5_fp16_inputs_200k_x_200k_x_64_row_blocks():
    """fp16 in / fp32 accumulate: the 160 GB result is produced in four 50000-row blocks into one reused buffer;
    every block is exact w.r.t. the fp16-rounded inputs (1e-4 bar), and the tolerance study vs the ORIGINAL fp32
    inputs stays at the fp16 rounding level."""
    if free_gb() < 45:
        pytest.skip("needs ~42 GB of free device memory")
    m, k, blk = 200_000, 64, 50_000
    c = centers(k)
    x32, y32 = blobs(m, k, 1234, c), blobs(m, k, 4321, c)
    x, y = x32.half(), y32.half()
    out = torch.empty((blk, m), dtype=torch.float32, device="cuda")
    worst32 = 0.0
    for r0 in range(0, m, blk):
        out.fill_(float("nan"))
        pairwise_distance(x[r0:r0 + blk], y, out=out, metric=DT.L2Expanded)
        r = dc.check_pairwise_sampled(out, x, y, DT.L2Expanded, count=60_000, eps=EPS, row_offset=r0, seed=r0 + 1)
        assert r["n_bad"] == 0, (r0, r)
        r32 = dc.check_pairwise_sampled(out, x32, y32, DT.L2Expanded, count=60_000, eps=1.0, row_offset=r0, seed=r0 + 1)
        worst32 = max(worst32, r32["max_rel_err"])
    assert worst32 < 5e-2, worst32                # fp16 input rounding (2^-11 per element, amplified by cancellation)


def test_config4_fused_l2_nn_1m_x_8m_x_96_sampled_queries_vs_full_db():
    """The bench's fusedL2NN job on one GPU (8 chunks of 2^20 db rows, bounds carried across chunks): 65536 sampled
    queries are checked against the exact fp64 arg-min over all 8M rows."""
    if free_gb() < 30:
        pytest.skip("needs ~25 GB of free device memory")
    m, n, k, sample = 1_000_000, 8_000_000, 96, 65_536
    c = centers(k)
    q, db = blobs(m, k, 1234, c), blobs(n, k, 4321, c)
    h = DeviceResources()
    idx, val = fused_l2_nn(q, db, sqrt=False, handle=h)
    h.sync()
    g = torch.Generator(device="cuda").manual_seed(3)
    rows = torch.randperm(m, device="cuda", generator=g)[:sample]
    rows[:4] = torch.tensor([0, 127, 128, m - 1], device="cuda")
    ref_val, ref_idx = [], []
    for s0 in range(0, sample, 16384):            # 16384 x 65536 fp64 tiles: ~8.6 GB at a time
        v, a = dc.nn_exact_fp64(q[rows[s0:s0 + 16384]], db)
        ref_val.append(v); ref_idx.append(a)
    ref_val, ref_idx = torch.cat(ref_val), torch.cat(ref_idx)
    r = dc.check_nn(idx[rows], val[rows], ref_val, ref_idx, q[rows], lambda ix: db[ix], eps=EPS)
    assert r["val_n_bad"] == 0, r
    assert r["idx_strict_match"] >= 0.9999, r
    assert r["idx_tie_aware_match"] == 1.0, r
    assert int(idx.min()) >= 0 and int(idx.max()) < n


# (last in the file: the module-scoped 40 GB output buffer stays allocated until the module ends, and on an
# 80 GB card the other shapes would not fit next to it)
@pytest.fixture(scope="module")
def cfg2():
    """configs[1]: 100000 x 100000 x 128 fp32 inputs + ONE reused 40 GB output buffer."""
    if free_gb() < 60:
        pytest.skip("needs ~45 GB of free device memory")
    c = centers(128)
    x, y = blobs(100_000, 128, 1234, c), blobs(100_000, 128, 4321, c)
    out = torch.empty((100_000, 100_000), dtype=torch.float32, device="cuda")
    yield x, y, out
    del out
    torch.cuda.empty_cache()


@pytest.mark.parametrize("metric", [DT.L2Expanded, DT.CosineExpanded, DT.CorrelationExpanded, DT.L2SqrtExpanded])
def test_config2_expanded_100k_x_100k_x_128(cfg2, metric):
    x, y, out = cfg2
    out.fill_(float("nan"))                      # a tile that is never written cannot pass
    pairwise_distance(x, y, out=out, metric=metric)
    r = dc.check_pairwise_sampled(out, x, y, metric, count=200_000, eps=EPS)
    assert r["n_bad"] == 0, r
    assert r["checked"] >= 200_000
    # every 128 x 256 tile was written: one probe per tile row / column band, and a strided sweep
    assert torch.isfinite(out[::127, ::251]).all()
    assert torch.isfinite(out[-1]).all() and torch.isfinite(out[:, -1]).all()


def test_config2_self_distance_diagonal_is_zero(cfg2):
    x, _, out = cfg2
    pairwise_distance(x, x, out=out, metric=DT.L2Expanded)
    assert (out.diagonal() == 0).all()           # x == y aliasing: d(i, i) = 0 exactly (CHANGELOG.md:1057,1213)
    r = dc.check_pairwise_sampled(out, x, x, DT.L2Expanded, count=100_000, eps=EPS)
    assert r["n_bad"] == 0, r
