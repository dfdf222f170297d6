"""GPU tier: raft_b200.distance.pairwise_distance (through the C ABI) against the CPU oracle.

Shapes follow the reference's historical distance tests ({1024,1024,32}, {1024,32,1024},
{32,1024,1024}; SURVEY.md section 4) plus ragged sizes, x==y aliasing, padded leading dimensions,
Fortran order and caller-provided outputs.  Tolerance: 1e-4 relative with the absolute-below-eps
rule of raft::CompareApprox (cpp/tests/test_utils.h:31-45), as BASELINE.json's north_star states."""
import numpy as np
import pytest
import torch

import oracle
from oracle import DistanceType as DT
from raft_b200 import LogicError
from raft_b200.common import DeviceResources, device_ndarray, set_output_as
from raft_b200.distance import pairwise_distance

pytestmark = pytest.mark.gpu
EPS = 1e-4

EXPANDED = [DT.L2Expanded, DT.L2SqrtExpanded, DT.CosineExpanded, DT.CorrelationExpanded]
UNEXPANDED = [DT.L1, DT.L2Unexpanded, DT.L2SqrtUnexpanded, DT.Linf, DT.Canberra, DT.LpUnexpanded]


def blobs(m, n, k, seed=0):
    x, _, c = oracle.make_blobs(m, k, seed=1234 + seed)
    y, _, _ = oracle.make_blobs(n, k, seed=4321 + seed, centers=c)
    return x, y


def run(x, y, metric, p=2.0, **kw):
    out = pairwise_distance(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), metric=metric, p=p, **kw)
    return out.copy_to_host()


def check(got, ref, eps=EPS):
    ok, msg = oracle.match_approx(got, ref, eps)
    assert ok, msg


@pytest.mark.parametrize("metric", EXPANDED + UNEXPANDED)
@pytest.mark.parametrize("shape", [(1024, 1024, 32), (333, 257, 45), (129, 300, 128), (64, 50, 7)])
def test_metric_vs_oracle(metric, shape):
    x, y = blobs(*shape)
    check(run(x, y, metric, p=3.0), oracle.pairwise_distance(x, y, metric, 3.0))


def test_inner_product_vs_oracle():
    # inner products cancel to ~0 for some pairs: compare against the magnitude |x||y|
    x, y = blobs(500, 400, 100)
    got = run(x, y, DT.InnerProduct)
    ref = oracle.pairwise_distance(x, y, DT.InnerProduct)
    scale = np.sqrt(oracle.row_norm_sq(x))[:, None] * np.sqrt(oracle.row_norm_sq(y))[None, :]
    assert np.abs(got - ref).max() <= 1e-5 * scale.max()
    assert (np.abs(got - ref) <= 1e-5 * scale + 1e-6).all()


@pytest.mark.parametrize("metric", [DT.L2Expanded, DT.L2SqrtExpanded, DT.CosineExpanded, DT.L1])
@pytest.mark.parametrize("shape", [(1024, 32, 1024), (32, 1024, 1024), (300, 700, 1000), (513, 300, 300)])
def test_reference_test_shapes_large_k(metric, shape):
    # k > 256: the tensor path accumulates K in chunks of 128 with an fp32 add per chunk, which keeps
    # the 1e-4 bar (a single 1024-deep MMA chain measured 2.1e-4 on intra-cluster pairs; the
    # reference's own tests used 1e-3 for these shapes, SURVEY.md section 4)
    x, y = blobs(*shape)
    check(run(x, y, metric), oracle.pairwise_distance(x, y, metric))


@pytest.mark.parametrize("metric", [DT.L2Expanded, DT.L2SqrtExpanded, DT.CosineExpanded, DT.L1, DT.Linf])
def test_uniform_data(metric):
    rng = np.random.default_rng(5)
    x = rng.uniform(-1, 1, (700, 96)).astype(np.float32)
    y = rng.uniform(-1, 1, (450, 96)).astype(np.float32)
    check(run(x, y, metric), oracle.pairwise_distance(x, y, metric))


@pytest.mark.parametrize("name", ["prob_KLDivergence", "prob_JensenShannon", "prob_HellingerExpanded",
                                  "bool_HammingUnexpanded", "bool_RusselRaoExpanded", "bool_JaccardExpanded",
                                  "bool_DiceExpanded", "count_BrayCurtis"])
def test_distribution_and_boolean_metrics(golden, name):
    # SURVEY.md 8(f) item 4: the remaining dense metrics of the enum, against the golden fixtures
    pre, metric = name.split("_")
    x, y = golden[f"{pre}_x"], golden[f"{pre}_y"]
    got = run(x, y, DT[metric]).astype(np.float64)
    ref = golden[name]
    fin = np.isfinite(ref)
    assert (np.isinf(got) == np.isinf(ref)).all()
    ok, msg = oracle.match_approx(got[fin], ref[fin], EPS)
    assert ok, msg
    # and a larger ragged shape against the oracle
    rng = np.random.default_rng(4)
    if pre == "prob":
        a = rng.random((300, 70)); b = rng.random((260, 70))
        a /= a.sum(1, keepdims=True); b /= b.sum(1, keepdims=True)
    elif pre == "count":
        a = rng.random((300, 70)) * 9; b = rng.random((260, 70)) * 9
    else:
        a = (rng.random((300, 70)) > 0.5); b = (rng.random((260, 70)) > 0.5)
    a, b = a.astype(np.float32), b.astype(np.float32)
    check(run(a, b, DT[metric]), oracle.pairwise_distance(a, b, DT[metric]))


def test_canberra_zero_over_zero_is_zero():
    rng = np.random.default_rng(9)
    x = rng.standard_normal((150, 40)).astype(np.float32)
    y = rng.standard_normal((130, 40)).astype(np.float32)
    x[:, ::3] = 0.0
    y[:, ::3] = 0.0          # shared zero coordinates: 0/0 terms must contribute 0, not NaN
    x[7] = 0.0
    y[11] = 0.0              # a fully-zero pair
    got = run(x, y, DT.Canberra)
    assert np.isfinite(got).all() and got[7, 11] == 0.0
    check(got, oracle.pairwise_distance(x, y, DT.Canberra))


@pytest.mark.parametrize("k", [32, 64, 96, 128, 160, 288])
def test_every_k_regime_of_the_tensor_kernel(k):
    # k <= 96: double-buffered staging; k <= 128: resident y block; k > 128: streaming operands
    x, y = blobs(515, 1028, k, seed=k)
    for metric in (DT.L2Expanded, DT.CosineExpanded):
        check(run(x, y, metric), oracle.pairwise_distance(x, y, metric))


def test_wide_dynamic_range_rows():
    # one power-of-two scale per matrix: rows 2^12 below the matrix maximum keep full precision
    x, y = blobs(300, 260, 64)
    x[::2] *= 2.0 ** -12
    y[::3] *= 2.0 ** -12
    check(run(x, y, DT.L2Expanded), oracle.pairwise_distance(x, y, DT.L2Expanded))
    check(run(x, y, DT.CosineExpanded), oracle.pairwise_distance(x, y, DT.CosineExpanded))


def test_golden_fixtures(golden):
    for case in ("small", "cfg1"):
        x, y = golden[f"{case}_x"], golden[f"{case}_y"]
        for name in ("L2Expanded", "L2SqrtExpanded", "CosineExpanded", "L1", "L2Unexpanded", "Linf",
                     "Canberra", "CorrelationExpanded"):
            check(run(x, y, DT[name]), golden[f"{case}_{name}"])
        check(run(x, y, DT.LpUnexpanded, p=3.0), golden[f"{case}_LpUnexpanded_p3"])


def test_config1_scipy_metric_strings():
    """BASELINE.json configs[0]: 1024x1024x32 fp32 vs cdist (the oracle is pinned to cdist)."""
    x, y = blobs(1024, 1024, 32)
    for name, mt in (("euclidean", DT.L2SqrtExpanded), ("sqeuclidean", DT.L2Expanded), ("cityblock", DT.L1),
                     ("chebyshev", DT.Linf), ("canberra", DT.Canberra), ("cosine", DT.CosineExpanded),
                     ("correlation", DT.CorrelationExpanded)):
        check(run(x, y, name), oracle.pairwise_distance(x, y, mt))
    check(run(x, y, "minkowski", p=1.5), oracle.pairwise_distance(x, y, DT.LpUnexpanded, 1.5))


def test_aliased_inputs_zero_diagonal():
    x, _ = blobs(300, 1, 64)
    xt = torch.from_numpy(x).cuda()
    for metric in (DT.L2Expanded, DT.L2SqrtExpanded):
        got = pairwise_distance(xt, xt, metric=metric).copy_to_host()
        assert (np.diag(got) == 0).all()
        check(got, oracle.pairwise_distance(x, x, metric))
    got = pairwise_distance(xt, xt, metric=DT.L1).copy_to_host()
    assert (np.diag(got) == 0).all()


def test_symmetry_property():
    x, y = blobs(260, 390, 96)
    for metric in (DT.L2Expanded, DT.CosineExpanded, DT.L1):
        a = run(x, y, metric)
        b = run(y, x, metric)
        # A.B^T vs B.A^T go through different operand roles of the tensor core: equal up to the
        # accumulation-order noise, far inside the 1e-4 bar
        assert np.array_equal(a, b.T) or oracle.match_approx(a, b.T, 2e-5)[0]


def test_padded_leading_dimensions_and_out_param():
    x, y = blobs(200, 150, 40)
    xp = torch.zeros(200, 48, device="cuda"); xp[:, :40] = torch.from_numpy(x).cuda()
    yp = torch.zeros(150, 56, device="cuda"); yp[:, :40] = torch.from_numpy(y).cuda()
    outp = torch.full((200, 160), -7.0, device="cuda")
    for metric in (DT.L2Expanded, DT.L1):
        ret = pairwise_distance(xp[:, :40], yp[:, :40], out=outp[:, :150], metric=metric)
        assert ret is not None
        got = outp.cpu().numpy()
        check(got[:, :150], oracle.pairwise_distance(x, y, metric))
        assert (got[:, 150:] == -7.0).all()      # padding untouched


def test_unaligned_output_falls_back_to_manual_stores():
    x, y = blobs(130, 259, 32)
    buf = torch.zeros(130 * 259 + 1, device="cuda")
    out = buf[1:].view(130, 259)                  # 4-byte aligned only, odd row pitch
    pairwise_distance(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), out=out, metric=DT.L2Expanded)
    check(out.cpu().numpy(), oracle.pairwise_distance(x, y, DT.L2Expanded))


@pytest.mark.parametrize("metric", [DT.L2Expanded, DT.CosineExpanded, DT.L1, DT.Linf])
def test_fortran_order(metric):
    x, y = blobs(210, 170, 33)
    xf = torch.from_numpy(x).cuda().t().contiguous().t()    # column-major storage
    yf = torch.from_numpy(y).cuda().t().contiguous().t()
    out = pairwise_distance(xf, yf, metric=metric)
    got = out.copy_to_host()
    assert got.shape == (210, 170)
    check(got, oracle.pairwise_distance(x, y, metric))


def test_fortran_order_kl_divergence_is_not_transposed():
    # KLDivergence is the one asymmetric metric: the column-major entry computes D^T with the operands
    # exchanged, so the kernel must swap their roles back (ADVICE r1; the reference's op had an explicit
    # !is_row_major branch)
    rng = np.random.default_rng(11)
    a = rng.random((90, 37)); b = rng.random((70, 37))
    a /= a.sum(1, keepdims=True); b /= b.sum(1, keepdims=True)
    a, b = a.astype(np.float32), b.astype(np.float32)
    af = torch.from_numpy(a).cuda().t().contiguous().t()
    bf = torch.from_numpy(b).cuda().t().contiguous().t()
    got = pairwise_distance(af, bf, metric=DT.KLDivergence).copy_to_host()
    ref = oracle.pairwise_distance(a, b, DT.KLDivergence)
    check(got, ref)
    assert not oracle.match_approx(got, oracle.pairwise_distance(b, a, DT.KLDivergence).T, EPS)[0]


def test_fp16_inputs_tolerance_study():
    """BASELINE.json configs[4] (fp16 in / fp32 accumulate): exact w.r.t. the fp16-rounded inputs,
    ~1e-3 w.r.t. the original fp32 inputs."""
    x, y = blobs(512, 384, 64)
    xh, yh = x.astype(np.float16), y.astype(np.float16)
    got = pairwise_distance(torch.from_numpy(xh).cuda(), torch.from_numpy(yh).cuda(), metric=DT.L2Expanded).copy_to_host()
    check(got, oracle.pairwise_distance(xh, yh, DT.L2Expanded))
    ref32 = oracle.pairwise_distance(x, y, DT.L2Expanded)
    rel = np.abs(got - ref32) / np.maximum(ref32, 1e-6)
    assert np.quantile(rel, 0.999) < 2e-2


def test_fp16_exact_operands_skip_cross_terms_and_stay_exact():
    # operands that are exact in fp16 (here: small integers in fp32 storage) take the 1-product
    # path; the result must be the exact integer distance
    rng = np.random.default_rng(2)
    x = rng.integers(-8, 9, (300, 96)).astype(np.float32)
    y = rng.integers(-8, 9, (520, 96)).astype(np.float32)
    got = run(x, y, DT.L2Expanded)
    ref = oracle.pairwise_distance(x, y, DT.L2Expanded)
    assert np.array_equal(got.astype(np.float64), ref)
    got = run(x[:, :32].copy(), y[:, :32].copy(), DT.InnerProduct)
    assert np.array_equal(got.astype(np.float64), oracle.pairwise_distance(x[:, :32], y[:, :32], DT.InnerProduct))
    x = rng.integers(-8, 9, (130, 400)).astype(np.float32)   # streaming layout (k > 128), chunked (k > 320)
    y = rng.integers(-8, 9, (260, 400)).astype(np.float32)
    assert np.array_equal(run(x, y, DT.L2Expanded).astype(np.float64), oracle.pairwise_distance(x, y, DT.L2Expanded))
    assert np.array_equal(run(x[:, :200].copy(), y[:, :200].copy(), DT.L2Expanded).astype(np.float64),
                          oracle.pairwise_distance(x[:, :200], y[:, :200], DT.L2Expanded))


def test_output_conversion_and_handle():
    x, y = blobs(64, 48, 16)
    h = DeviceResources()
    set_output_as("torch")
    try:
        out = pairwise_distance(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), metric="l1", handle=h)
        h.sync()
        assert isinstance(out, torch.Tensor)
    finally:
        set_output_as("raft")
    out = pairwise_distance(device_ndarray(x), device_ndarray(y), metric="l1")
    assert isinstance(out, device_ndarray)
    check(out.copy_to_host(), oracle.pairwise_distance(x, y, DT.L1))


def test_error_behaviour():
    a = torch.zeros(4, 8, device="cuda"); b = torch.zeros(4, 9, device="cuda")
    with pytest.raises(ValueError):
        pairwise_distance(a, b)
    with pytest.raises(ValueError):
        pairwise_distance(a, a, metric="haversine")
    with pytest.raises(TypeError):
        pairwise_distance(a, a.double())
    with pytest.raises((ValueError, LogicError)):
        pairwise_distance(a, a, metric="minkowski", p=0.0)
    with pytest.raises(ValueError):
        pairwise_distance(a, a, out=torch.zeros(3, 4, device="cuda"))
    # empty problems are no-ops
    out = pairwise_distance(torch.zeros(0, 8, device="cuda"), a)
    assert out.shape == (0, 4)


def test_full_size_sampled_check():
    """Size-independent check at a BASELINE-scale shape: sample pairs of a 50000 x 40000 x 128
    result and compare them with the oracle (the full matrix is 8 GB; the oracle sees 2e5 pairs)."""
    m, n, k = 50000, 40000, 128
    g = torch.Generator(device="cuda").manual_seed(7)
    centers = (torch.rand(5, k, device="cuda", generator=g) * 20 - 10)
    x = centers[torch.randint(0, 5, (m,), device="cuda", generator=g)] + torch.randn(m, k, device="cuda", generator=g)
    y = centers[torch.randint(0, 5, (n,), device="cuda", generator=g)] + torch.randn(n, k, device="cuda", generator=g)
    out = pairwise_distance(x, y, metric=DT.L2Expanded).tensor
    ii = torch.randint(0, m, (200000,), device="cuda", generator=g)
    jj = torch.randint(0, n, (200000,), device="cuda", generator=g)
    # include tile corners / edges
    ii[:4] = torch.tensor([0, m - 1, 0, m - 1], device="cuda"); jj[:4] = torch.tensor([0, n - 1, n - 1, 0], device="cuda")
    got = out[ii, jj].cpu().numpy()
    xs, ys = x[ii].cpu().numpy().astype(np.float64), y[jj].cpu().numpy().astype(np.float64)
    ref = ((xs - ys) ** 2).sum(axis=1)
    check(got, ref)
    # every row block / column block was written (no stale tile): min over each 128x256 tile > 0
    assert torch.isfinite(out).all()
    assert (out.view(-1)[:: 104729] >= 0).all()


@pytest.mark.parametrize("metric", [DT.L2Expanded, DT.L2SqrtExpanded, DT.InnerProduct])
@pytest.mark.parametrize("where", ["x", "y", "both"])
def test_outlier_rows_do_not_degrade_ordinary_rows(metric, where):
    """ADVICE r1 (medium): one sentinel row ~1e9 in O(1) data used to push every ordinary row into the fp16
    subnormals (single power-of-two scale per matrix).  Rows far below the matrix maximum now take their own
    exponent (prep.cuh), so the ordinary pairs keep the 1e-4 bar; pairs that involve the sentinel are exact to
    fp32 rounding of their own (huge) magnitude."""
    rng = np.random.default_rng(21)
    x = rng.standard_normal((300, 72)).astype(np.float32)
    y = rng.standard_normal((520, 72)).astype(np.float32)
    if where in ("x", "both"):
        x[17] = 1.0e9 * rng.standard_normal(72).astype(np.float32)
    if where in ("y", "both"):
        y[333] = 3.0e8 * rng.standard_normal(72).astype(np.float32)
        y[5, 11] = -7.0e7                                    # a single huge element inside an ordinary row
    got = run(x, y, metric).astype(np.float64)
    ref = oracle.pairwise_distance(x, y, metric)
    if metric == DT.InnerProduct:
        scale = np.sqrt(oracle.row_norm_sq(x))[:, None] * np.sqrt(oracle.row_norm_sq(y))[None, :]
        assert (np.abs(got - ref) <= 2e-5 * scale + 1e-6).all()
    else:
        check(got, ref)


F64_METRICS = [DT.L2Expanded, DT.L2SqrtExpanded, DT.CosineExpanded, DT.CorrelationExpanded, DT.InnerProduct, DT.L1,
               DT.L2Unexpanded, DT.L2SqrtUnexpanded, DT.Linf, DT.Canberra, DT.LpUnexpanded]


@pytest.mark.parametrize("metric", F64_METRICS)
def test_fp64_inputs_every_metric(metric):
    """double in / double out (SURVEY.md 8(a2), 8(f4)): the SIMT fp64 path agrees with the fp64 oracle to ~1e-12."""
    x, y = blobs(150, 131, 37)
    x64, y64 = x.astype(np.float64) + 1e-9, y.astype(np.float64) - 1e-9      # values that fp32 cannot represent
    out = pairwise_distance(torch.from_numpy(x64).cuda(), torch.from_numpy(y64).cuda(), metric=metric, p=3.0)
    got = out.copy_to_host()
    assert got.dtype == np.float64
    ref = oracle.pairwise_distance(x64, y64, metric, 3.0)
    assert np.allclose(got, ref, rtol=1e-11, atol=1e-9), float(np.abs(got - ref).max())


@pytest.mark.parametrize("name", ["prob_KLDivergence", "prob_JensenShannon", "prob_HellingerExpanded", "bool_HammingUnexpanded",
                                  "bool_RusselRaoExpanded", "bool_JaccardExpanded", "bool_DiceExpanded", "count_BrayCurtis"])
def test_fp64_distribution_and_boolean_metrics(golden, name):
    pre, metric = name.split("_")
    x, y = golden[f"{pre}_x"].astype(np.float64), golden[f"{pre}_y"].astype(np.float64)
    got = pairwise_distance(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), metric=DT[metric]).copy_to_host()
    ref = golden[name]
    fin = np.isfinite(ref)
    assert (np.isinf(got) == np.isinf(ref)).all()
    assert np.allclose(got[fin], ref[fin], rtol=1e-9, atol=1e-12)


def test_fp64_fortran_order_and_kl_roles():
    rng = np.random.default_rng(3)
    a = rng.random((70, 21)); b = rng.random((50, 21))
    a /= a.sum(1, keepdims=True); b /= b.sum(1, keepdims=True)
    af = torch.from_numpy(a).cuda().t().contiguous().t()
    bf = torch.from_numpy(b).cuda().t().contiguous().t()
    for metric in (DT.KLDivergence, DT.L2Expanded, DT.CosineExpanded):
        got = pairwise_distance(af, bf, metric=metric).copy_to_host()
        assert np.allclose(got, oracle.pairwise_distance(a, b, metric), rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("metric", [DT.L2Expanded, DT.L2SqrtExpanded, DT.CosineExpanded, DT.L1])
def test_nan_rows_propagate_and_stay_local(metric):
    """A NaN in an input row poisons exactly that row's / column's distances (the finalisation clamp must not turn
    NaN into 0: fmaxf(NaN, 0) = 0), every other pair keeps the 1e-4 bar."""
    x, y = blobs(300, 260, 96)
    x[7, 13] = np.nan
    y[201, 95] = np.nan
    got = run(x, y, metric)
    assert np.isnan(got[7]).all() and np.isnan(got[:, 201]).all()
    keep_r, keep_c = np.arange(300) != 7, np.arange(260) != 201
    sub = got[keep_r][:, keep_c]
    assert np.isfinite(sub).all()
    check(sub, oracle.pairwise_distance(x[keep_r], y[keep_c], metric))
