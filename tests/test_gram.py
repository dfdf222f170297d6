"""gram_matrix without a GPU: the fp64 reference (tests/gram_ref.py) against scikit-learn, the workspace query, every
argument check of the C ABI, B2D_ERR_CUDA without a device, and the C++ shim's compile (its run on the GPU is marked
gpu)."""
import os
import subprocess

import numpy as np
import pytest
import torch

import cpp_build
import gram_ref
from raft_b200 import _lib


SIZE_MAX = 2 ** 64 - 1
P = 1 << 12   # a non-null pointer that is never dereferenced (every call below fails before any work)
KID = {"linear": 0, "polynomial": 1, "rbf": 2, "tanh": 3}


def call(kernel=2, degree=3, gamma=0.5, coef0=1.0, dtype=0, x=P, ldx=8, y=P, ldy=8, out=P, ldo=100, m=10, n=100, k=8,
         row_major=1, ws=P * 256, wsb=1 << 40):
    return _lib.lib().b2d_gram_matrix(None, kernel, degree, gamma, coef0, dtype, x, ldx, y, ldy, out, ldo, m, n, k,
                                      row_major, ws, wsb)


def test_reference_matches_sklearn():
    pw = pytest.importorskip("sklearn.metrics.pairwise")
    rng = np.random.default_rng(4)
    x = rng.normal(size=(40, 11))
    y = rng.normal(size=(30, 11))
    np.testing.assert_allclose(gram_ref.gram_matrix(x, y, "linear"), pw.linear_kernel(x, y), rtol=1e-12, atol=1e-12)
    for degree, gamma, coef0 in ((3, 0.3, 1.0), (1, 0.7, -0.2), (5, 0.1, -0.5)):   # (degree 0: test_reference_conventions)
        np.testing.assert_allclose(gram_ref.gram_matrix(x, y, "polynomial", degree, gamma, coef0),
                                   pw.polynomial_kernel(x, y, degree=degree, gamma=gamma, coef0=coef0), rtol=1e-12, atol=1e-12)
    for gamma in (0.05, 1.0):
        np.testing.assert_allclose(gram_ref.gram_matrix(x, y, "rbf", gamma=gamma), pw.rbf_kernel(x, y, gamma=gamma),
                                   rtol=1e-12, atol=1e-14)
    for gamma, coef0 in ((0.2, 0.0), (0.4, -0.7)):
        np.testing.assert_allclose(gram_ref.gram_matrix(x, y, "tanh", gamma=gamma, coef0=coef0),
                                   pw.sigmoid_kernel(x, y, gamma=gamma, coef0=coef0), rtol=1e-12, atol=1e-14)


def test_reference_conventions():
    x = np.array([[1.0, 2.0], [np.nan, 0.0], [0.5, -1.0]])
    y = np.array([[0.0, 1.0], [3.0, np.nan]])
    for kernel in gram_ref.KERNELS:
        g = gram_ref.gram_matrix(x, y, kernel, degree=3, gamma=0.5, coef0=1.0)
        # a NaN row poisons its own row and column only
        assert np.isnan(g[1]).all() and np.isnan(g[:, 1]).all()
        assert np.isfinite(g[[0, 2]][:, [0]]).all()
    # degree 0: 1 everywhere, NaN included (x ** 0 == 1)
    assert (gram_ref.gram_matrix(x, y, "polynomial", degree=0, gamma=0.5, coef0=1.0) == 1.0).all()
    # rbf of a matrix with itself: exactly 1 on the diagonal (difference form)
    z = np.random.default_rng(1).normal(size=(20, 7))
    assert (np.diag(gram_ref.gram_matrix(z, z, "rbf", gamma=3.0)) == 1.0).all()


def test_bounds_accept_rounding_and_reject_errors():
    rng = np.random.default_rng(9)
    u = rng.normal(size=(50, 60)).astype(np.float32)
    for kernel, degree in (("rbf", 0), ("tanh", 0), ("polynomial", 5), ("polynomial", 0), ("linear", 0)):
        g, c0 = np.float32(0.7), np.float32(-0.3)
        uu = np.abs(u) if kernel == "rbf" else u
        t = gram_ref.affine(kernel, uu.astype(np.float64), float(g), float(c0))
        exact = uu.copy() if kernel == "linear" else gram_ref.f(kernel, t, degree).astype(np.float32)
        assert gram_ref.transform_check(exact, uu, kernel, degree, g, c0).all()
        if kernel == "polynomial" and degree == 0:
            continue
        off = exact.copy()
        off[3, 4] = np.nextafter(np.nextafter(np.nextafter(np.float32(exact[3, 4] * (1 + 1e-4)), np.inf), np.inf), np.inf)
        assert not gram_ref.transform_check(off, uu, kernel, degree, g, c0)[3, 4]


def test_workspace_query():
    L = _lib.lib()
    for kernel in range(4):
        base = 0 if kernel == KID["rbf"] else 6   # L2Expanded / InnerProduct
        for dt in (0, 1, 2):
            for m, n, k in ((1000, 2000, 32), (37, 29, 321), (0, 5, 3)):
                assert L.b2d_gram_matrix_workspace_bytes(kernel, dt, m, n, k) == L.b2d_pairwise_workspace_bytes(base, dt, m, n, k)
    assert L.b2d_gram_matrix_workspace_bytes(4, 0, 5, 5, 5) == SIZE_MAX
    assert L.b2d_gram_matrix_workspace_bytes(-1, 0, 5, 5, 5) == SIZE_MAX
    assert L.b2d_gram_matrix_workspace_bytes(0, 3, 5, 5, 5) == SIZE_MAX
    assert L.b2d_gram_matrix_workspace_bytes(2, 0, -1, 5, 5) == SIZE_MAX
    assert L.b2d_gram_matrix_workspace_bytes(2, 0, 5, 5, -1) == SIZE_MAX


def test_argument_errors():
    E = _lib.B2D_ERR_INVALID_ARG
    assert call(kernel=4) == E and call(kernel=-1) == E
    assert call(gamma=float("nan")) == E and call(coef0=float("inf")) == E
    assert call(gamma=1e300) == E                    # finite as a double, infinite as the float the fp32 path uses
    assert call(gamma=1e300, dtype=2, wsb=10) == _lib.B2D_ERR_WORKSPACE   # fp64 uses it as a double: accepted
    assert call(kernel=1, degree=-1) == E
    assert call(kernel=2, degree=-1, wsb=10) == _lib.B2D_ERR_WORKSPACE   # degree is read for POLYNOMIAL only
    assert call(dtype=3) == _lib.B2D_ERR_UNSUPPORTED
    assert call(m=-1) == E and call(k=-1) == E
    assert call(k=0) == E
    assert call(x=None) == E and call(y=None) == E and call(out=None) == E
    assert call(ldx=7) == E and call(ldy=7) == E and call(ldo=99) == E
    assert call(row_major=0, ldx=9, ldy=100, ldo=10) == E and call(row_major=0, ldx=10, ldy=99, ldo=10) == E
    assert call(row_major=0, ldx=10, ldy=100, ldo=9) == E
    assert call(wsb=10) == _lib.B2D_ERR_WORKSPACE and call(ws=None) == _lib.B2D_ERR_WORKSPACE
    assert call(ws=P * 256 + 16) == E
    assert call(dtype=2, wsb=10) == _lib.B2D_ERR_WORKSPACE
    # nothing to do: OK without touching anything
    assert call(m=0, x=None, y=None, out=None) == _lib.B2D_OK
    assert call(n=0, k=0) == _lib.B2D_OK
    with pytest.raises(_lib.LogicError):
        _lib.check(call(kernel=7))


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the error without a device")
@pytest.mark.parametrize("kernel", [0, 1, 2, 3])
@pytest.mark.parametrize("dtype", [0, 1, 2])
def test_cuda_error_without_device(kernel, dtype):
    assert call(kernel=kernel, dtype=dtype) == _lib.B2D_ERR_CUDA


@pytest.fixture(scope="module")
def build_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("gram_cpp"))


def compile_shim(build_dir, mock_raft):
    exe = os.path.join(build_dir, "gram_shim_mockraft" if mock_raft else "gram_shim")
    return cpp_build.build("gram_shim_test.cu", exe, mock_raft)


@pytest.mark.parametrize("mock_raft", [False, True])
def test_shim_compiles(build_dir, mock_raft):
    assert os.path.exists(compile_shim(build_dir, mock_raft))


@pytest.mark.gpu
@pytest.mark.parametrize("mock_raft", [False, True])
def test_shim_runs_on_gpu_and_matches_python(build_dir, mock_raft):
    from raft_b200.distance import gram_matrix
    exe = compile_shim(build_dir, mock_raft)
    rng = np.random.default_rng(23)
    m, n, k = 300, 250, 40
    x = rng.normal(size=(m, k)).astype(np.float32)
    y = rng.normal(size=(n, k)).astype(np.float32)
    inp, out = os.path.join(build_dir, "in.bin"), os.path.join(build_dir, "out.bin")
    with open(inp, "wb") as f:
        f.write(np.array([m, n, k], np.int64).tobytes() + x.tobytes() + y.tobytes())
    res = subprocess.run([exe, inp, out], capture_output=True, text=True, timeout=120)
    assert res.returncode == 0 and "PASS" in res.stdout, res.stdout + res.stderr
    got = np.fromfile(out, np.float32).reshape(4, m, n)
    xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    # the kernels and parameters of gram_shim_test.cu, in its order
    for i, (kernel, degree, gamma, coef0) in enumerate((("linear", 0, 1.0, 0.0), ("polynomial", 3, 0.05, 1.0),
                                                        ("rbf", 0, 0.02, 0.0), ("tanh", 0, 0.03, -0.5))):
        ref = gram_matrix(xd, yd, kernel, degree=degree, gamma=gamma, coef0=coef0).copy_to_host()
        assert np.array_equal(got[i], ref), kernel
