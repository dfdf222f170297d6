"""kernel_density on the GPU against the fp64 model of tests/kde_ref.py.

Two references:
  * the reduction alone: the model evaluated on the engine's own pairwise_distance(queries, dataset, "sqeuclidean"),
    which is bit for bit the d^2 the EPI_KDE epilogue sees.  The bound, derived from the fp32 evaluation in kde_row32:
    the log-sum-exp kernels form u = log2 w - s d^2 with two roundings (|du| <= 2^-23 |u|), sum 2^(u - M) with ex2.approx
    (2^-22 relative) over a 5-level tree and a 2-level quad combine, then fold in fp64, so |d out| <= 2^-22 ln 2 |lse| +
    2^-20 < 1e-6 (1 + |lse|), lse = out - log_norm + log W.  The compact kernels evaluate each K to within 4e-7 absolute
    (the cos / sqrt approximations near the support edge), so a row whose model sum is S adds 4e-7 sum_j w_j / S over its
    support.
  * the raw inputs: the model between d^2 (1 - 1e-4) - a and d^2 (1 + 1e-4) + a, a = 2^-20 (|q|^2 + |x|^2) (the distance
    bar of the expanded form): every kernel decreases in d^2, so the exact answer for the engine's d^2 lies between the
    two.  Compact kernels use data with no pair inside that band around h2.
"""
import math

import numpy as np
import pytest
import torch

import kde_ref as R
import oracle
from raft_b200 import _lib
from raft_b200.distance import DistanceType, pairwise_distance
from raft_b200.neighbors import kernel_density

pytestmark = pytest.mark.gpu


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def engine_d2(q, x):
    return pairwise_distance(cuda(q), cuda(x), metric=DistanceType.L2Expanded).copy_to_host()


def kd(x, q, kernel, h, w=None, **kw):
    xd = x if torch.is_tensor(x) else cuda(x)
    qd = q if torch.is_tensor(q) else cuda(q)
    return kernel_density(xd, qd, bandwidth=h, kernel=kernel, sample_weight=None if w is None else cuda(w), **kw) \
        .cpu().numpy()


def gap_h(d2, quantile=0.05, rel=1e-3):
    """a bandwidth whose h^2 lies in a gap of the d^2 values, at least rel away from every one (relative), near the
    quantile"""
    v = np.unique(np.asarray(d2, np.float64).ravel())
    v = v[np.isfinite(v) & (v > 0)]
    start = int(quantile * len(v))
    for i in range(start, len(v) - 1):
        lo, hi = v[i], v[i + 1]
        if hi > lo * (1 + 4 * rel) + 1e-6:
            return math.sqrt(math.sqrt(lo * hi))
    raise AssertionError("no gap")


def check_reduction(x, q, kernel, h, w=None, got=None, d2=None):
    """the engine against the model on the engine's own d^2, to the bound of the module docstring"""
    d2 = engine_d2(q, x) if d2 is None else d2
    got = kd(x, q, kernel, h, w) if got is None else got
    dim = x.shape[1]
    want = R.score_from_d2(d2, kernel, h, w) + R.log_norm(kernel, h, dim)
    wsum = x.shape[0] if w is None else float(np.asarray(w, np.float64).sum())
    lse = want - R.log_norm(kernel, h, dim) + math.log(wsum)
    tol = 1e-6 * (1 + np.abs(lse))
    if kernel in R.COMPACT:
        ww = np.ones(x.shape[0]) if w is None else np.asarray(w, np.float64)
        supp = (np.asarray(d2, np.float64) < R.h2_of(h)) * ww
        with np.errstate(divide="ignore", invalid="ignore"):
            tol = tol + 4e-7 * supp.sum(1) / np.exp(lse)
    fin = np.isfinite(want)
    assert np.array_equal(fin, np.isfinite(got)), np.nonzero(fin != np.isfinite(got))
    assert np.array_equal(np.isnan(want), np.isnan(got))
    assert np.array_equal(want[~fin & ~np.isnan(want)], got[~fin & ~np.isnan(want)])
    err = np.abs(got - want)[fin]
    assert (err <= tol[fin]).all(), (kernel, float(err.max()), float((err / tol[fin]).max()))
    return got


def envelope(x, q, kernel, h, w=None):
    """(lo, hi) of the model over the distance bar of the expanded form"""
    d2 = R.d2_64(q, x)
    a = 2.0 ** -20 * ((np.asarray(q, np.float64) ** 2).sum(1)[:, None] + (np.asarray(x, np.float64) ** 2).sum(1)[None])
    ln = R.log_norm(kernel, h, x.shape[1])
    lo = R.score_from_d2(d2 * (1 + 1e-4) + a, kernel, h, w) + ln
    hi = R.score_from_d2(np.maximum(d2 * (1 - 1e-4) - a, 0), kernel, h, w) + ln
    if kernel in R.COMPACT:   # no pair changes sides inside the bar
        band = np.abs(d2 - R.h2_of(h)) <= 1e-4 * d2 + a
        assert not band.any()
    return lo, hi


def check_raw(x, q, kernel, h, w=None, got=None):
    got = kd(x, q, kernel, h, w) if got is None else got
    lo, hi = envelope(x, q, kernel, h, w)
    slack = 1e-6 * (1 + np.abs(hi))
    fin = np.isfinite(hi)
    assert np.array_equal(np.isfinite(got), fin)
    assert ((got[fin] >= lo[fin] - slack[fin]) & (got[fin] <= hi[fin] + slack[fin])).all(), kernel
    return got


def blobs(m, n, d, seed):
    q, _, c = oracle.make_blobs(m, d, seed=seed)
    x, _, _ = oracle.make_blobs(n, d, seed=seed + 1, centers=c)
    return x, q


# ------------------------------------------------------------------------------------------------- 1. the reduction
@pytest.mark.parametrize("kernel", R.KERNELS)
@pytest.mark.parametrize("weighted", [False, True])
def test_reduction_matches_model_on_engine_d2(kernel, weighted):
    x, q = blobs(700, 1500, 24, 11)
    w = np.random.default_rng(3).uniform(0, 3, 1500).astype(np.float32) if weighted else None
    d2 = engine_d2(q, x)
    h = gap_h(d2, 0.02) if kernel in R.COMPACT else 2.0
    check_reduction(x, q, kernel, h, w, d2=d2)


def test_tophat_counts_are_exact():
    x, q = blobs(900, 2000, 16, 21)
    d2 = engine_d2(q, x)
    for quant in (0.001, 0.01, 0.2):
        h = gap_h(d2, quant)
        out = kd(x, q, "tophat", h)
        cnt = (d2 < R.h2_of(h)).sum(1)
        live = cnt > 0
        got = np.rint(np.exp(out[live] - R.log_norm("tophat", h, 16)) * 2000)
        assert np.array_equal(got, cnt[live]) and np.isneginf(out[~live]).all()


# ------------------------------------------------------------------------------------------------- 2. raw fp64 model
@pytest.mark.parametrize("kernel", R.KERNELS)
def test_against_fp64_model(kernel):
    x, q = blobs(300, 800, 12, 31)
    h = gap_h(R.d2_64(q, x), 0.05, rel=3e-4) if kernel in R.COMPACT else 1.5
    check_raw(x, q, kernel, h)


# ------------------------------------------------------------------------------------------------------- 3. shapes
@pytest.mark.parametrize("m,n", [(1, 300), (127, 255), (129, 257), (300, 1), (383, 100), (256, 513)])
def test_ragged_shapes(m, n):
    x, q = blobs(m, n, 20, 41)
    for kernel in ("gaussian", "epanechnikov", "exponential"):
        d2 = engine_d2(q, x)
        h = 2.0 if kernel != "epanechnikov" else gap_h(d2, 0.3)
        check_reduction(x, q, kernel, h, d2=d2)


@pytest.mark.parametrize("d", [1, 31, 33, 128, 129, 320])
def test_feature_counts_both_kernel_variants(d):
    x, q = blobs(260, 700, d, 50 + d)
    d2 = engine_d2(q, x)
    for kernel in R.KERNELS:
        h = gap_h(d2, 0.1) if kernel in R.COMPACT else math.sqrt(float(np.median(d2)))
        check_reduction(x, q, kernel, h, d2=d2)


def test_pitched_dataset():
    x, q = blobs(200, 600, 40, 61)
    pad = torch.zeros(600, 48, device="cuda")
    pad[:, :40] = cuda(x)
    view = pad[:, :40]
    assert view.stride() == (48, 1)
    for kernel in ("gaussian", "cosine"):
        h = 3.0 if kernel == "gaussian" else gap_h(engine_d2(q, x), 0.2)
        got = kd(view, q, kernel, h)
        assert np.array_equal(got.view(np.int64), kd(x, q, kernel, h).view(np.int64))


# ------------------------------------------------------------------------------------------------- 4. determinism
def test_bit_identical_across_batches_runs_and_graph_replay():
    x, q = blobs(1000, 3000, 32, 71)
    w = np.random.default_rng(5).uniform(0, 1, 3000).astype(np.float32)
    for kernel in ("gaussian", "tophat", "cosine"):
        h = 4.0
        base = kd(x, q, kernel, h, w, batch_cols=256)
        for b in (768, 0, 1000, 256):
            assert np.array_equal(kd(x, q, kernel, h, w, batch_cols=b).view(np.int64), base.view(np.int64)), (kernel, b)
    s = torch.cuda.Stream()
    from raft_b200.common import DeviceResources
    handle = DeviceResources(stream=s)
    xd, qd = cuda(x), cuda(q)
    with torch.cuda.stream(s):
        first = kernel_density(xd, qd, bandwidth=4.0, batch_cols=512, handle=handle).clone()
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        out = kernel_density(xd, qd, bandwidth=4.0, batch_cols=512, handle=handle)
    for _ in range(2):
        out.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out.view(torch.int64), first.view(torch.int64))
    assert np.array_equal(first.cpu().numpy().view(np.int64), kd(x, q, "gaussian", 4.0).view(np.int64))


# --------------------------------------------------------------------------------------------------- 5. self pairs
def test_self_pairs():
    _, x = blobs(700, 1, 16, 81)   # (the 700 query rows)
    xd = cuda(x)
    same = pairwise_distance(xd, xd, metric=DistanceType.L2Expanded).copy_to_host()
    copy = pairwise_distance(xd.clone(), xd, metric=DistanceType.L2Expanded).copy_to_host()
    assert (np.diag(same) == 0).all()
    resid = np.diag(copy)
    assert (resid > 0).any()
    h = math.sqrt(0.5 * resid[resid > 0].min())   # below every non-zero self residue and every other pair
    assert (same + np.eye(700) * 1e9 > 4 * h * h).all()
    got_same = kd(xd, xd, "tophat", h)
    assert np.isfinite(got_same).all()   # each row counts itself, d^2_ii = 0
    assert np.allclose(np.exp(got_same - R.log_norm("tophat", h, 16)) * 700, 1.0, rtol=1e-12)
    got_copy = kd(xd, xd.clone(), "tophat", h)
    assert np.array_equal(np.isfinite(got_copy), resid == 0)
    for kernel in ("gaussian", "linear"):
        check_reduction(x, x, kernel, 3.0, got=kd(xd, xd, kernel, 3.0), d2=same)
        check_reduction(x, x, kernel, 3.0, got=kd(xd, xd.clone(), kernel, 3.0), d2=copy)


# -------------------------------------------------------------------------------------------------- 6. range edges
@pytest.mark.parametrize("kernel", ["gaussian", "exponential"])
def test_far_queries_are_finite(kernel):
    x, q = blobs(50, 400, 8, 91)
    off = np.zeros(8, np.float32)
    off[0] = 141.4 if kernel == "gaussian" else 1e4   # d^2 / 2h^2 ~ 1e4, d / h ~ 1e4
    qf = (q + off).astype(np.float32)
    got = kd(x, qf, kernel, 1.0)
    assert np.isfinite(got).all() and (got < -5e3).all()
    check_raw(x, qf, kernel, 1.0, got=got)
    check_reduction(x, qf, kernel, 1.0, got=got)


def test_empty_support_is_minus_inf():
    x, q = blobs(40, 300, 8, 92)
    qf = (q + 1000).astype(np.float32)
    for kernel in R.COMPACT:
        assert np.isneginf(kd(x, qf, kernel, 1.0)).all()


# ------------------------------------------------------------------------------------------------ 7. NaN and weights
def test_nan_rows():
    x, q = blobs(300, 900, 16, 101)
    qn, xn = q.copy(), x.copy()
    qn[7, 3] = np.nan
    xn[123, 0] = np.nan
    for kernel in R.KERNELS:
        h = 2.0 if kernel not in R.COMPACT else 6.0
        clean = kd(x, q, kernel, h)
        got = kd(x, qn, kernel, h)
        assert np.isnan(got[7]) and not np.isnan(np.delete(got, 7)).any()
        np.testing.assert_allclose(np.delete(got, 7), np.delete(clean, 7), rtol=1e-6, atol=1e-6)
        assert np.isnan(kd(xn, q, kernel, h)).all()


def test_zero_weights_remove_rows():
    x, q = blobs(400, 1200, 24, 111)
    w = np.ones(1200, np.float32)
    w[::3] = 0
    keep = w > 0
    for kernel in R.KERNELS:
        d2 = engine_d2(q, x)
        h = gap_h(d2, 0.05) if kernel in R.COMPACT else 2.5
        a = kd(x, q, kernel, h, w)
        b = kd(x[keep], q, kernel, h)
        fin = np.isfinite(b)
        assert np.array_equal(np.isfinite(a), fin)
        np.testing.assert_allclose(a[fin], b[fin], rtol=2e-6, atol=2e-6)


def test_weighted_matches_sklearn():
    from sklearn.neighbors import KernelDensity
    x, q = blobs(120, 700, 5, 121)
    w = np.random.default_rng(9).uniform(0, 2, 700).astype(np.float32)
    for kernel in R.KERNELS:
        h = gap_h(R.d2_64(q, x), 0.05, rel=3e-4) if kernel in R.COMPACT else 1.7
        got = check_raw(x, q, kernel, h, w)
        sk = KernelDensity(kernel=kernel, bandwidth=h, atol=0, rtol=0).fit(x.astype(np.float64), sample_weight=w) \
            .score_samples(q.astype(np.float64))
        fin = np.isfinite(got)
        lo, hi = envelope(x, q, kernel, h, w)
        np.testing.assert_allclose(got[fin], sk[fin], rtol=0, atol=float(np.max(hi[fin] - lo[fin])) + 1e-5)


@pytest.mark.parametrize("bad", ["negative", "nan", "inf", "zero"])
def test_bad_weights(bad):
    x, q = blobs(64, 300, 8, 131)
    w = np.ones(300, np.float32)
    if bad == "zero":
        w[:] = 0
    else:
        w[17] = {"negative": -1.0, "nan": np.nan, "inf": np.inf}[bad]
    xd, qd, wd = cuda(x), cuda(q), cuda(w)
    out = torch.full((64,), 7.0, dtype=torch.float64, device="cuda")
    L = _lib.lib()
    nb = L.b2d_kde_workspace_bytes(64, 300, 8, 0)
    ws = torch.empty(nb, dtype=torch.uint8, device="cuda")
    for kernel in range(6):
        _lib.check(L.b2d_kde_score_samples(torch.cuda.current_stream().cuda_stream, kernel, 1.0, xd.data_ptr(), 8,
                                           wd.data_ptr(), qd.data_ptr(), 8, 64, 300, 8, 0, out.data_ptr(), ws.data_ptr(),
                                           nb))
        assert torch.isnan(out).all()
    with pytest.raises(ValueError):
        kernel_density(xd, qd, sample_weight=wd)


def test_bandwidth_rules_and_empty_queries():
    x, q = blobs(100, 500, 6, 141)
    from raft_b200.neighbors.kernel_density import bandwidth_of
    for rule in ("scott", "silverman"):
        h = bandwidth_of(rule, 500, 6)
        assert np.array_equal(kd(x, q, "gaussian", rule).view(np.int64), kd(x, q, "gaussian", h).view(np.int64))
    assert kd(x, q[:0], "gaussian", 1.0).shape == (0,)


# -------------------------------------------------------------------------------------------------- 8. one large case
def test_large_sampled_rows_against_fp64_on_device():
    g = torch.Generator(device="cuda").manual_seed(7)
    m, n, d, h = 20000, 1 << 20, 96, 3.0
    c = torch.randn(64, d, device="cuda", generator=g) * 4
    x = (c[torch.randint(0, 64, (n,), device="cuda", generator=g)] + torch.randn(n, d, device="cuda", generator=g))
    q = (c[torch.randint(0, 64, (m,), device="cuda", generator=g)] + torch.randn(m, d, device="cuda", generator=g))
    out = kernel_density(x, q, bandwidth=h)
    assert torch.isfinite(out).all()
    rows = torch.arange(0, m, 397, device="cuda")
    qs, x64 = q[rows].double(), x.double()
    d2 = ((qs * qs).sum(1)[:, None] + (x64 * x64).sum(1)[None] - 2 * qs @ x64.T).clamp_min(0)
    a = 2.0 ** -20 * ((qs * qs).sum(1)[:, None] + (x64 * x64).sum(1)[None])
    ln = R.log_norm("gaussian", h, d) - math.log(n)
    lo = torch.logsumexp(-(d2 * (1 + 1e-4) + a) / (2 * h * h), 1) + ln
    hi = torch.logsumexp(-(d2 * (1 - 1e-4) - a).clamp_min(0) / (2 * h * h), 1) + ln
    got = out[rows]
    slack = 1e-6 * (1 + hi.abs())
    assert ((got >= lo - slack) & (got <= hi + slack)).all()
