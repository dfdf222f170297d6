"""kernel_density without a GPU: the fp64 model of the GPU tier (tests/kde_ref.py) pinned to sklearn, every kernel's
normalisation against quadrature (and sklearn's wrong cosine normalisation at even d, recorded), every argument check of
the C call with its status and message, the workspace query and its recorded contract
(tests/golden/kde_workspace_contract.json), B2D_ERR_CUDA without a device, the bandwidth rules, and the C++ shim's
compile (its run on the GPU is in tests/test_kde_shim.py)."""
import math
import os

import numpy as np
import pytest
import torch
from scipy import integrate

import cpp_build
import kde_ref as R
from raft_b200 import _lib
from raft_b200.neighbors.kernel_density import bandwidth_of
from test_workspace_contract import load, replay_bytes, replay_errors

SIZE_MAX = 2 ** 64 - 1
P = 1 << 12   # a non-null pointer that is never dereferenced (every call below fails before any work)
E, U, W = _lib.B2D_ERR_INVALID_ARG, _lib.B2D_ERR_UNSUPPORTED, _lib.B2D_ERR_WORKSPACE
CONTRACT = "kde_workspace_contract.json"


def kde(kernel=0, h=1.0, y=P, ldy=8, w=None, x=P, ldx=8, m=10, n=100, d=8, batch=0, out=P, ws=P * 256, wsb=1 << 40):
    return _lib.lib().b2d_kde_score_samples(None, kernel, h, y, ldy, w, x, ldx, m, n, d, batch, out, ws, wsb)


def status(rc):
    return rc, _lib.lib().b2d_last_error().decode()


# ---------------------------------------------------------------------------------------------------------------- model
def _data(d, seed):
    rng = np.random.default_rng(seed)
    x = rng.normal(size=(200, d)).astype(np.float32)
    q = rng.normal(size=(30, d)).astype(np.float32)
    w = rng.uniform(0, 2, 200).astype(np.float32)
    w[::17] = 0
    return x, q, w


@pytest.mark.parametrize("d", [1, 2, 3, 5, 16])
@pytest.mark.parametrize("kernel", R.KERNELS)
@pytest.mark.parametrize("weighted", [False, True])
def test_model_matches_sklearn(d, kernel, weighted):
    from sklearn.neighbors import KernelDensity
    if kernel == "cosine" and d % 2 == 0:
        pytest.skip("sklearn's cosine normalisation is wrong at even d (test_sklearn_cosine_norm_defect)")
    x, q, w = _data(d, 100 + d)
    w = w if weighted else None
    h = 0.9 * math.sqrt(d)
    d2 = R.d2_64(q, x)
    # nothing within 1e-6 of the support edge: sklearn's dist < h and the model's d^2 < fp32(h^2) agree
    assert np.abs(d2 - h * h).min() > 1e-6 * h * h
    got = R.score64(x, q, kernel, h, w)
    sk = KernelDensity(kernel=kernel, bandwidth=h, atol=0, rtol=0).fit(x.astype(np.float64), sample_weight=w) \
        .score_samples(q.astype(np.float64))
    live = np.isfinite(got)
    np.testing.assert_allclose(got[live], sk[live], rtol=1e-10, atol=0)
    # an empty support is -inf (sklearn's tree returns a finite floor for some of those rows)
    support = ((d2 < R.h2_of(h)) & ((w if weighted else np.ones(200)) > 0)).any(axis=1)
    assert (live == support).all() if kernel in R.COMPACT else live.all()
    assert live.sum() >= 20


def _log_norm_quad(kernel, d):
    """-log of the integral of K(|x|; 1) over R^d by quadrature of S_(d-1) r^(d-1) K(r), scaled at its maximum"""
    logk = {"gaussian": lambda r: -0.5 * r * r, "exponential": lambda r: -r,
            "tophat": lambda r: 0.0, "epanechnikov": lambda r: math.log1p(-r * r), "linear": lambda r: math.log1p(-r),
            "cosine": lambda r: math.log(math.cos(0.5 * math.pi * r))}[kernel]
    top = 1.0 if kernel in R.COMPACT else 60.0 + 4.0 * d
    grid = np.linspace(1e-9, top * (1 - 1e-12), 20001)
    f = [(d - 1) * math.log(r) + logk(r) for r in grid]
    c, mode = max(f), grid[int(np.argmax(f))]
    g = lambda r: math.exp((d - 1) * math.log(r) + logk(r) - c) if 0 < r < top else 0.0   # noqa: E731
    val = sum(integrate.quad(g, a, b, epsabs=0, epsrel=1.2e-14, limit=500)[0]
              for a, b in ((0, mode), (mode, top)))
    return -(R.log_sphere(d) + c + math.log(val))


@pytest.mark.parametrize("kernel", R.KERNELS)
def test_log_norm_matches_quadrature(kernel):
    worst = 0.0
    for d in range(1, 321):
        want, got = _log_norm_quad(kernel, d), R.log_norm(kernel, 1.0, d)
        worst = max(worst, abs(got - want) / max(1.0, abs(want)))
    assert worst < 1e-12, worst
    # the bandwidth enters as -d log h
    assert R.log_norm(kernel, 2.5, 7) == pytest.approx(R.log_norm(kernel, 1.0, 7) - 7 * math.log(2.5), rel=1e-14)


def test_sklearn_cosine_norm_defect():
    from sklearn.neighbors._ball_tree import kernel_norm
    exact = {d: R.log_norm("cosine", 1.0, d) for d in (1, 2, 4, 6, 8, 32, 128, 320)}
    for d in (1, 3, 5, 7, 9, 11):
        assert kernel_norm(1.0, d, "cosine", return_log=True) == pytest.approx(R.log_norm("cosine", 1.0, d), rel=1e-9)
    assert kernel_norm(1.0, 2, "cosine", return_log=True) == pytest.approx(-1.386, abs=1e-3)
    assert exact[2] == pytest.approx(-0.374, abs=1e-3)
    assert kernel_norm(1.0, 6, "cosine", return_log=True) == pytest.approx(-5.52, abs=1e-2)
    assert exact[6] == pytest.approx(-0.114, abs=1e-3)
    for d in (4, 8, 32, 128, 320):
        assert math.isnan(kernel_norm(1.0, d, "cosine", return_log=True))
        assert math.isfinite(exact[d])


def test_model_from_d2_rules():
    d2 = np.array([[0.0, 0.25, 4.0, 1.0], [0.0, np.nan, 1.0, 1.0], [9.0, 16.0, 25.0, 36.0]], np.float32)
    w = np.array([1.0, 2.0, 0.0, 1.0])
    for kernel in R.KERNELS:
        s = R.log_sum_from_d2(d2, kernel, 1.0, w)
        assert np.isnan(s[1])
        if kernel in R.COMPACT:   # strict support: d^2 = 1 = h^2 is outside, the zero weight drops d^2 = 4
            assert s[2] == -np.inf
            k = {"tophat": [1, 1], "epanechnikov": [1, 0.75], "linear": [1, 0.5],
                 "cosine": [1, math.cos(math.pi / 4)]}[kernel]
            assert s[0] == pytest.approx(math.log(k[0] + 2 * k[1]), rel=1e-15)
        else:
            assert np.isfinite(s).sum() == 2
    far = R.log_sum_from_d2(np.array([[2e4, 3e4]]), "gaussian", 1.0)
    assert far[0] == pytest.approx(-1e4 + math.log1p(math.exp(-5e3)), rel=1e-15)


def test_bandwidth_rules():
    assert bandwidth_of("scott", 1000, 3) == 1000 ** (-1 / 7)
    assert bandwidth_of("silverman", 1000, 3) == (1000 * 5 / 4) ** (-1 / 7)
    assert bandwidth_of(0.25, 10, 2) == 0.25
    with pytest.raises(ValueError):
        bandwidth_of("auto", 10, 2)


# ------------------------------------------------------------------------------------------------------------- C ABI
def test_workspace_query():
    L = _lib.lib()
    for args in ((-1, 5, 3, 0), (5, -1, 3, 0), (5, 5, -3, 0), (5, 5, 3, -1)):
        assert L.b2d_kde_workspace_bytes(*args) == SIZE_MAX
    for m, n, k in ((1000, 2000, 32), (100000, 100000, 128), (7, 900, 320)):
        ws = L.b2d_kde_workspace_bytes(m, n, k, 0)
        # the tensor path's operands come first: at least what pairwise_distance needs
        assert ws > L.b2d_pairwise_workspace_bytes(0, _lib.B2D_F32, m, n, k)
        # the partials of one slab: 8 bytes per row and 128-column half, the slab rounded up to 256 columns
        a, b = L.b2d_kde_workspace_bytes(m, n, k, 256), L.b2d_kde_workspace_bytes(m, n, k, 512)
        assert abs((b - a) - 16 * m) < 1024   # (each region is rounded up to 1024 bytes)
        assert L.b2d_kde_workspace_bytes(m, n, k, 1) == a == L.b2d_kde_workspace_bytes(m, n, k, 255)
    # the default keeps the partials near 1 GiB and never beyond the whole dataset
    big = L.b2d_kde_workspace_bytes(1 << 20, 1 << 20, 32, 0) - L.b2d_kde_workspace_bytes(1 << 20, 1 << 20, 32, 256)
    assert 2 ** 30 - 2 ** 25 <= big + 16 * (1 << 20) <= 2 ** 30 + 2 ** 25
    assert L.b2d_kde_workspace_bytes(10, 300, 8, 0) == L.b2d_kde_workspace_bytes(10, 300, 8, 10 ** 9)


def test_workspace_contract_bytes():
    rows = replay_bytes(load(CONTRACT), "b2d_kde_workspace_bytes")
    assert len(rows) == 8 * 6 * 8 * 5 + 4
    for *args, want in rows:
        assert (want == SIZE_MAX) == (min(args) < 0), args


def test_workspace_contract_errors():
    assert replay_errors(load(CONTRACT)) == 21


def test_argument_errors():
    for bad in (-1, 6, 100):
        assert status(kde(kernel=bad)) == (E, "unknown kernel %d" % bad)
    for kw in ({"m": -1}, {"n": -1}, {"d": -1}):
        assert status(kde(**kw)) == (E, "negative extent")
    assert status(kde(batch=-1)) == (E, "negative batch_cols")
    assert status(kde(m=2 ** 31)) == (E, "m and n must be below 2^31")
    assert status(kde(n=2 ** 31)) == (E, "m and n must be below 2^31")
    assert status(kde(n=0)) == (E, "n and d must be positive")
    assert status(kde(d=0)) == (E, "n and d must be positive")
    assert status(kde(d=321, ldx=321, ldy=321)) == (U, "kernel_density supports d <= 320 (the whole distance at once)")
    for h in (0.0, -1.0, float("inf"), float("nan")):
        assert status(kde(h=h)) == (E, "bandwidth must be finite and > 0")
    for h in (1e-25, 1e-20):   # 0.5 / fp32(h h) overflows (or h h is 0 in fp32)
        assert status(kde(h=h)) == (E, "0.5 / bandwidth^2 is not finite in fp32")
    assert status(kde(y=None)) == (E, "null dataset / queries / out")
    assert status(kde(x=None)) == (E, "null dataset / queries / out")
    assert status(kde(out=None)) == (E, "null dataset / queries / out")
    assert status(kde(ldx=7)) == (E, "leading dimension smaller than d")
    assert status(kde(ldy=7)) == (E, "leading dimension smaller than d")
    assert status(kde(wsb=10))[0] == W
    assert status(kde(ws=None))[0] == W
    assert status(kde(ws=P * 256 + 16))[0] == E
    # m == 0 does nothing, once the arguments that do not depend on m are valid
    assert kde(m=0, x=None, y=None, out=None, ws=None, wsb=0) == _lib.B2D_OK
    assert status(kde(m=0, n=0)) == (E, "n and d must be positive")
    with pytest.raises(_lib.LogicError):
        _lib.check(kde(kernel=7))


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the error without a device")
def test_cuda_error_without_device():
    assert kde() == _lib.B2D_ERR_CUDA
    assert kde(w=P, kernel=5, batch=256) == _lib.B2D_ERR_CUDA


def test_shim_compiles(tmp_path):
    for mock in (False, True):
        exe = str(tmp_path / ("kde_shim_mockraft" if mock else "kde_shim"))
        assert os.path.exists(cpp_build.build("kde_shim_test.cu", exe, mock))
