"""GPU tier: gram_matrix (the kernel Gram matrices, fused into the distance kernel's epilogue).  Every kernel value is
checked against the engine's own pre-transform value (pairwise_distance InnerProduct, or L2Expanded for rbf, on the same
inputs) with the transform bound of tests/gram_ref.py, the linear kernel bit for bit, and against the fp64 reference with
the pairwise bounds carried through |f'|; over the resident, streaming and K-chunked paths, both store paths, padded and
Fortran-order outputs, aliased inputs, NaN and outlier rows, CUDA-graph capture and the full 100000^2 x 128 shape."""
import numpy as np
import pytest
import torch

import gram_ref
import oracle
from raft_b200 import LogicError, _lib
from raft_b200.common import DeviceResources, device_ndarray, set_output_as
from raft_b200.distance import gram_matrix, pairwise_distance

pytestmark = pytest.mark.gpu
DEV = "cuda"
KERNELS = gram_ref.KERNELS
PARAMS = {"linear": (0, 1.0, 0.0), "polynomial": (3, 0.02, 0.5), "rbf": (0, 0.01, 0.0), "tanh": (0, 0.001, -0.25)}
TDT = {"f32": torch.float32, "f16": torch.float16, "f64": torch.float64}
SHAPES = [(129, 300), (192, 511), (193, 257), (255, 1000)]   # m % 128 in {1, 64, 65, 127}; n ragged, n % 4 == 0 and != 0
KS = [1, 7, 32, 128, 129, 320, 321, 1000]


def data(m, n, k, dtype="f32", seed=0):
    x, _, c = oracle.make_blobs(m, k, seed=101 + seed)
    y, _, _ = oracle.make_blobs(n, k, seed=907 + seed, centers=c)
    x, y = torch.from_numpy(x).to(DEV), torch.from_numpy(y).to(DEV)
    return x.to(TDT[dtype]), y.to(TDT[dtype])


def params_for(kernel, x, y):
    """gamma scaled to the data, so that the transform is exercised over its whole range and not saturated"""
    degree, gamma, coef0 = PARAMS[kernel]
    k = x.shape[1]
    return degree, (gamma * 32.0 / k if kernel != "linear" else gamma), coef0


def base(x, y, kernel, out=None):
    """the engine's own pre-transform value"""
    return pairwise_distance(x, y, out=out, metric=gram_ref.base_metric(kernel))


def host(a):
    if isinstance(a, np.ndarray):
        return a
    if isinstance(a, device_ndarray):
        return a.copy_to_host()
    return a.cpu().numpy()


def assert_all(ok, what):
    assert ok.all(), "%s: %d of %d outside the bound, first at %s" % (what, (~ok).sum(), ok.size, np.argwhere(~ok)[0])


def check(got, x, y, kernel, degree, gamma, coef0, dtype="f32", u=None):
    """the transform bound against the engine's pre-transform value u, and the fp64 reference"""
    got = host(got)
    xh, yh = x.double().cpu().numpy(), y.double().cpu().numpy()
    if dtype == "f64":
        assert got.dtype == np.float64
        u = gram_ref.base_value(xh, yh, kernel)
        scale = np.sqrt((xh ** 2).sum(1))[:, None] * np.sqrt((yh ** 2).sum(1))[None, :]
        du = 1e-12 * (scale if kernel != "rbf" else np.abs(u)) + 1e-300
        ref = gram_ref.gram_matrix(xh, yh, kernel, degree, gamma, coef0)
        t = gram_ref.affine(kernel, u, gamma, coef0)
        fp = gram_ref.fprime(kernel, t, degree) if kernel != "linear" else np.ones_like(u)
        bound = fp * abs(gamma if kernel != "linear" else 1.0) * du * 1.01 + 1e-14 * np.abs(ref) + 1e-300
        with np.errstate(invalid="ignore"):
            ok = (np.abs(got - ref) <= bound) | (np.isnan(got) & np.isnan(ref))
        assert_all(ok, "fp64 %s vs oracle" % kernel)
        return
    assert got.dtype == np.float32
    if u is None:
        u = base(x, y, kernel)
    assert_all(gram_ref.transform_check(got, host(u), kernel, degree, gamma, coef0), "%s transform" % kernel)
    assert_all(gram_ref.oracle_check(got, xh, yh, kernel, degree, gamma, coef0), "%s vs oracle" % kernel)


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("dtype", ["f32", "f16"])
@pytest.mark.parametrize("kernel", KERNELS)
def test_tensor_path(kernel, dtype, k):
    """resident (k <= 128), streaming (k <= 320) and K-chunked (k > 320); each k on another m % 128 and store path"""
    m, n = SHAPES[KS.index(k) % len(SHAPES)]
    x, y = data(m, n, k, dtype, seed=k)
    degree, gamma, coef0 = params_for(kernel, x, y)
    got = gram_matrix(x, y, kernel, degree=degree, gamma=gamma, coef0=coef0)
    assert got.shape == (m, n)
    check(got, x, y, kernel, degree, gamma, coef0, dtype)


@pytest.mark.parametrize("k", [1, 7, 129, 1000])
@pytest.mark.parametrize("kernel", KERNELS)
def test_fp64(kernel, k):
    m, n = SHAPES[[1, 7, 129, 1000].index(k)]
    x, y = data(m, n, k, "f64", seed=k)
    degree, gamma, coef0 = params_for(kernel, x, y)
    got = gram_matrix(x, y, kernel, degree=degree, gamma=gamma, coef0=coef0)
    check(got, x, y, kernel, degree, gamma, coef0, "f64")
    if kernel == "linear":   # the InnerProduct kernel itself
        assert np.array_equal(host(got), host(pairwise_distance(x, y, metric="inner_product")))


@pytest.mark.parametrize("kernel", KERNELS)
def test_store_paths_padding_and_fortran_order(kernel):
    m, n, k = 193, 300, 96
    x, y = data(m, n, k, seed=3)
    degree, gamma, coef0 = params_for(kernel, x, y)
    dense = host(gram_matrix(x, y, kernel, degree=degree, gamma=gamma, coef0=coef0))   # TMA stores (aligned, n % 4 == 0)
    # an out one float past 16-byte alignment: the register stores, the same values
    buf = torch.full((m * n + 1,), -7.0, device=DEV)
    gram_matrix(x, y, kernel, degree=degree, gamma=gamma, coef0=coef0, out=buf[1:].view(m, n))
    assert np.array_equal(host(buf[1:]).reshape(m, n), dense) and float(buf[0]) == -7.0
    # padded leading dimension: the padding is left as it was
    pad = torch.full((m, n + 5), -3.0, device=DEV)
    gram_matrix(x, y, kernel, degree=degree, gamma=gamma, coef0=coef0, out=pad[:, :n])
    assert np.array_equal(host(pad[:, :n]), dense) and (host(pad[:, n:]) == -3.0).all()
    # Fortran order (the operands exchanged inside: K(x, y) = K(y, x)), padded too
    xf, yf = x.t().contiguous().t(), y.t().contiguous().t()
    got = gram_matrix(xf, yf, kernel, degree=degree, gamma=gamma, coef0=coef0)
    assert not got.tensor.is_contiguous() and got.tensor.t().is_contiguous()
    u = pairwise_distance(xf, yf, metric=gram_ref.base_metric(kernel))
    check(got, x, y, kernel, degree, gamma, coef0, u=u)
    padf = torch.full((n + 3, m + 7), -5.0, device=DEV)   # [n + 3, m + 7] row-major = [m, n] column-major with ld m + 7
    view = padf[:n, :m].t()
    gram_matrix(xf, yf, kernel, degree=degree, gamma=gamma, coef0=coef0, out=view)
    assert np.array_equal(host(view), host(got)) and (host(padf[:, m:]) == -5.0).all() and (host(padf[n:]) == -5.0).all()


@pytest.mark.parametrize("dtype", ["f32", "f16", "f64"])
@pytest.mark.parametrize("fortran", [False, True])
def test_aliased_inputs_rbf_diagonal_is_one(dtype, fortran):
    x, _ = data(300, 1, 72, dtype, seed=5)
    if fortran:
        x = x.t().contiguous().t()
    for kernel in KERNELS:
        degree, gamma, coef0 = params_for(kernel, x, x)
        got = host(gram_matrix(x, x, kernel, degree=degree, gamma=gamma, coef0=coef0))
        if kernel == "rbf":
            assert (np.diag(got) == 1.0).all()
        if dtype != "f64":
            assert_all(gram_ref.oracle_check(got, x.double().cpu().numpy(), x.double().cpu().numpy(), kernel, degree, gamma,
                                             coef0), "aliased %s" % kernel)


@pytest.mark.parametrize("kernel", KERNELS)
def test_nan_rows_propagate_and_stay_local(kernel):
    x, y = data(300, 260, 96, seed=7)
    x[7, 13] = float("nan")
    y[201, 95] = float("nan")
    degree, gamma, coef0 = params_for(kernel, x, y)
    got = host(gram_matrix(x, y, kernel, degree=degree, gamma=gamma, coef0=coef0))
    assert np.isnan(got[7]).all() and np.isnan(got[:, 201]).all()
    keep_r, keep_c = np.arange(300) != 7, np.arange(260) != 201
    sub = got[keep_r][:, keep_c]
    assert np.isfinite(sub).all()
    u = host(base(x, y, kernel))[keep_r][:, keep_c]
    assert_all(gram_ref.transform_check(sub, u, kernel, degree, gamma, coef0), "%s transform" % kernel)
    xh, yh = x.double().cpu().numpy()[keep_r], y.double().cpu().numpy()[keep_c]
    assert_all(gram_ref.oracle_check(sub, xh, yh, kernel, degree, gamma, coef0), "%s vs oracle" % kernel)
    # degree 0: 1 everywhere, NaN rows included
    ones = host(gram_matrix(x, y, "polynomial", degree=0, gamma=gamma, coef0=coef0))
    assert (ones == 1.0).all()


@pytest.mark.parametrize("kernel", KERNELS)
def test_outlier_rows_do_not_degrade_ordinary_rows(kernel):
    rng = np.random.default_rng(21)
    x = rng.standard_normal((300, 72)).astype(np.float32)
    y = rng.standard_normal((520, 72)).astype(np.float32)
    x[17] = 1.0e9 * rng.standard_normal(72).astype(np.float32)
    y[333] = 3.0e8 * rng.standard_normal(72).astype(np.float32)
    y[5, 11] = -7.0e7
    xd, yd = torch.from_numpy(x).to(DEV), torch.from_numpy(y).to(DEV)
    degree, gamma, coef0 = 2, 0.05, 0.25
    got = gram_matrix(xd, yd, kernel, degree=degree, gamma=gamma, coef0=coef0)
    u = host(base(xd, yd, kernel))
    g = host(got)
    assert_all(gram_ref.transform_check(g, u, kernel, degree, gamma, coef0), "%s transform" % kernel)
    # the ordinary pairs keep the pairwise bound, carried through the transform
    keep_r, keep_c = np.arange(300) != 17, ~np.isin(np.arange(520), [5, 333])
    xs, ys = x[keep_r], y[keep_c]
    du = None
    if kernel != "rbf":   # the bound test_pairwise_gpu.py's outlier test holds for the inner product
        du = 2e-5 * np.sqrt(oracle.row_norm_sq(xs))[:, None] * np.sqrt(oracle.row_norm_sq(ys))[None, :] + 1e-6
    assert_all(gram_ref.oracle_check(g[keep_r][:, keep_c], xs, ys, kernel, degree, gamma, coef0, du=du),
               "%s ordinary rows" % kernel)


@pytest.mark.parametrize("degree", [0, 1, 5])
@pytest.mark.parametrize("dtype", ["f32", "f16", "f64"])
def test_polynomial_degrees_and_negative_parameters(degree, dtype):
    x, y = data(129, 257, 40, dtype, seed=degree)
    for gamma, coef0 in ((-0.03, -0.4), (0.03, -1.5), (-0.01, 0.0)):
        got = gram_matrix(x, y, "polynomial", degree=degree, gamma=gamma, coef0=coef0)
        if degree == 0:
            assert (host(got) == 1.0).all()
        check(got, x, y, "polynomial", degree, gamma, coef0, dtype)
    got = gram_matrix(x, y, "tanh", gamma=-0.02, coef0=-0.3)
    check(got, x, y, "tanh", 0, -0.02, -0.3, dtype)


def test_empty_and_argument_errors():
    x, y = data(10, 20, 8)
    assert gram_matrix(x[:0], y).shape == (0, 20)
    assert gram_matrix(x, y[:0]).shape == (10, 0)
    with pytest.raises(ValueError):
        gram_matrix(x, y, "sigmoid")
    with pytest.raises(ValueError):
        gram_matrix(x, y, "polynomial", degree=-1)
    with pytest.raises(ValueError):
        gram_matrix(x, y, "rbf", gamma=float("nan"))
    with pytest.raises(LogicError):
        gram_matrix(x, y, "rbf", gamma=1e300)   # not finite as the float the fp32 path uses
    with pytest.raises(ValueError):
        gram_matrix(x, y[:, :7])


def test_cuda_graph_capture():
    m, n, k = 600, 2048, 64
    x, y = data(m, n, k, seed=8)
    L = _lib.lib()
    out = torch.empty((m, n), device=DEV)
    ws = torch.empty(L.b2d_gram_matrix_workspace_bytes(_lib.B2D_KERNEL_RBF, _lib.B2D_F32, m, n, k), dtype=torch.uint8,
                     device=DEV)
    ref = host(gram_matrix(x, y, "rbf", gamma=0.01))
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        _lib.check(L.b2d_gram_matrix(s.cuda_stream, _lib.B2D_KERNEL_RBF, 0, 0.01, 0.0, _lib.B2D_F32, x.data_ptr(), k,
                                     y.data_ptr(), k, out.data_ptr(), n, m, n, k, 1, ws.data_ptr(), ws.numel()))
    for _ in range(2):
        out.fill_(-1.0)
        g.replay()
        torch.cuda.synchronize()
        assert np.array_equal(host(out), ref)


def test_output_conversion_and_handle():
    x, y = data(64, 48, 16)
    h = DeviceResources()
    set_output_as("torch")
    try:
        out = gram_matrix(x, y, "tanh", gamma=0.1, handle=h)
        h.sync()
        assert isinstance(out, torch.Tensor)
    finally:
        set_output_as("raft")
    out = gram_matrix(device_ndarray(x.cpu().numpy()), device_ndarray(y.cpu().numpy()), "tanh", gamma=0.1)
    assert isinstance(out, device_ndarray)
    check(out, x, y, "tanh", 0, 0.1, 0.0)
    from pylibraft.distance import gram_matrix as pl_gram
    assert pl_gram is gram_matrix


def test_full_size_sampled():
    """100000 x 100000 x 128 (40 GB of output): a sample of pairs and the tiles' corners re-evaluated in fp64 on the
    device, every kernel into the same output buffer"""
    from oracle.device_check import sample_pairs
    m = n = 100000
    k = 128
    g = torch.Generator(device=DEV).manual_seed(3)
    x = torch.randn((m, k), device=DEV, generator=g)
    y = torch.randn((n, k), device=DEV, generator=g)
    out = torch.empty((m, n), device=DEV)
    i, j = sample_pairs(m, n, 200_000, 11, DEV)
    a, b = x[i].double(), y[j].double()
    ip = (a * b).sum(1)
    sq = ((a - b) ** 2).sum(1)
    du_ip = 1e-5 * a.norm(dim=1) * b.norm(dim=1) + 1e-6
    for kernel in KERNELS:
        degree, gamma, coef0 = {"linear": (0, 1.0, 0.0), "polynomial": (3, 0.05, 1.0), "rbf": (0, 1.0 / 256, 0.0),
                                "tanh": (0, 0.05, -0.5)}[kernel]
        gram_matrix(x, y, kernel, degree=degree, gamma=gamma, coef0=coef0, out=out)
        got = out[i, j].double()
        gm, c0 = float(np.float32(gamma)), float(np.float32(coef0))
        if kernel == "linear":
            bad = (got - ip).abs() > du_ip
        else:
            u = sq if kernel == "rbf" else ip
            du = 1e-4 * torch.clamp(u.abs() * (1 + 1e-4), min=1.0) if kernel == "rbf" else du_ip
            t = gm * u + (0.0 if kernel == "rbf" else c0)
            dt = abs(gm) * du
            if kernel == "rbf":
                ref, worst = torch.exp(-t), torch.exp(-(t - dt))
            elif kernel == "tanh":
                ref = torch.tanh(t)
                worst = torch.where((t - dt <= 0) & (t + dt >= 0), torch.ones_like(t),
                                    torch.maximum(1 - torch.tanh(t - dt) ** 2, 1 - torch.tanh(t + dt) ** 2))
            else:
                ref = t ** degree
                worst = degree * torch.maximum((t - dt).abs(), (t + dt).abs()) ** (degree - 1)
            ulp = lambda v: torch.clamp(torch.abs(v).float().nextafter(torch.tensor(float("inf"), device=DEV)).double()
                                        - torch.abs(v).float().double(), min=2.0 ** -149)
            c = 2.0 * degree if kernel == "polynomial" else 2.0
            bad = (got - ref).abs() > worst * dt + worst * ulp(t) + c * ulp(ref)
        assert int(bad.sum()) == 0, (kernel, int(bad.sum()))
    del out
    torch.cuda.empty_cache()
