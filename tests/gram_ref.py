"""The fp64 reference of gram_matrix and the error bounds its tests hold (tests/test_gram.py, tests/test_gram_gpu.py).

gram_matrix(x, y, kernel, ...) is the kernel matrix in fp64 from the inputs as given (fp32 / fp16 inputs exactly
widened).  The bounds:
  transform  the engine's own pre-transform value u (pairwise_distance InnerProduct, or L2Expanded for rbf) against the
             transformed one: with u* = gamma u + coef0 in fp64 (gamma u for rbf), gamma and coef0 rounded to fp32,
             |got - f(u*)| <= |f'(u*)| ulp32(u*) + c ulp32(f(u*)), c = 2 for exp and tanh, 2 degree for the power;
             ulp32 is never below the spacing at FLT_MIN (2^-149).
  oracle     the bound the pairwise tests hold for u (InnerProduct: 1e-5 |x||y| + 1e-6; L2Expanded: CompareApprox 1e-4),
             carried through the largest |f'| over the interval it allows, plus the transform term.
"""
import numpy as np

KERNELS = ("linear", "polynomial", "rbf", "tanh")
ULP_FLOOR = 2.0 ** -149


def base_metric(kernel):
    """the pairwise_distance metric whose value the kernel transforms"""
    return "sqeuclidean" if kernel == "rbf" else "inner_product"


def base_value(x, y, kernel):
    """u in fp64: the inner products, or (rbf) the squared distances in the difference form"""
    a, b = np.asarray(x, np.float64), np.asarray(y, np.float64)
    if kernel == "rbf":
        out = np.empty((a.shape[0], b.shape[0]))
        for j0 in range(0, b.shape[0], 32):
            out[:, j0:j0 + 32] = ((a[:, None, :] - b[None, j0:j0 + 32, :]) ** 2).sum(-1)
        return out
    return a @ b.T


def affine(kernel, u, gamma, coef0):
    """u* = gamma u + coef0 (gamma u for rbf)"""
    return gamma * u if kernel == "rbf" else gamma * u + coef0


def f(kernel, t, degree):
    """the transform of u* (linear: u itself)"""
    with np.errstate(over="ignore", invalid="ignore"):
        if kernel == "rbf":
            return np.exp(-t)
        if kernel == "tanh":
            return np.tanh(t)
        if kernel == "polynomial":
            return np.ones_like(t) if degree == 0 else t ** degree   # (degree 0: 1 everywhere, NaN included)
        return t


def fprime(kernel, t, degree):
    """|f'(u*)|"""
    with np.errstate(over="ignore", invalid="ignore"):
        if kernel == "rbf":
            return np.exp(-t)
        if kernel == "tanh":
            return 1.0 - np.tanh(t) ** 2
        if kernel == "polynomial":
            return np.zeros_like(t) if degree == 0 else degree * np.abs(t) ** (degree - 1)
        return np.ones_like(t)


def gram_matrix(x, y, kernel="rbf", degree=3, gamma=1.0, coef0=0.0):
    """the kernel matrix in fp64 (gamma and coef0 as given)"""
    u = base_value(x, y, kernel)
    return u if kernel == "linear" else f(kernel, affine(kernel, u, gamma, coef0), degree)


def ulp32(v):
    v = np.abs(np.asarray(v, np.float64))
    with np.errstate(over="ignore", invalid="ignore"):
        s = np.spacing(v.astype(np.float32)).astype(np.float64)
    return np.maximum(s, ULP_FLOOR)


def c_transform(kernel, degree):
    return 2.0 * degree if kernel == "polynomial" else 2.0


def transform_check(got, u, kernel, degree, gamma, coef0):
    """boolean matrix: got (the engine's kernel values) against its own pre-transform values u, both fp32 on the host"""
    got = np.asarray(got, np.float64)
    u = np.asarray(u, np.float64)
    if kernel == "linear":
        return got.view(np.uint64) == u.view(np.uint64)    # bit for bit
    g, c0 = float(np.float32(gamma)), float(np.float32(coef0))
    t = affine(kernel, u, g, c0)
    ref = f(kernel, t, degree)
    bound = fprime(kernel, t, degree) * ulp32(t) + c_transform(kernel, degree) * ulp32(ref)
    with np.errstate(invalid="ignore"):
        ok = np.abs(got - ref) <= bound
    return ok | (np.isnan(got) & np.isnan(ref)) | (got == ref)


def base_error(x, y, kernel, u_ref):
    """the bound the pairwise tests hold for u: InnerProduct 1e-5 |x||y| + 1e-6, L2Expanded CompareApprox 1e-4"""
    if kernel == "rbf":
        return 1e-4 * np.maximum(np.abs(u_ref) * (1 + 1e-4), 1.0)
    nx = np.sqrt((np.asarray(x, np.float64) ** 2).sum(1))
    ny = np.sqrt((np.asarray(y, np.float64) ** 2).sum(1))
    return 1e-5 * nx[:, None] * ny[None, :] + 1e-6


def oracle_check(got, x, y, kernel, degree, gamma, coef0, du=None):
    """boolean matrix: got against the fp64 oracle on the same (fp32 / fp16-rounded) inputs, gamma and coef0 rounded to
    fp32 as the engine uses them.  du: the bound on the pre-transform value (default base_error)."""
    got = np.asarray(got, np.float64)
    u = base_value(x, y, kernel)
    if du is None:
        du = base_error(x, y, kernel, u)
    g, c0 = float(np.float32(gamma)), float(np.float32(coef0))
    if kernel == "linear":
        bound = du
        ref = u
    else:
        t = affine(kernel, u, g, c0)
        ref = f(kernel, t, degree)
        dt = abs(g) * du
        lo, hi = t - dt, t + dt
        worst = np.maximum(fprime(kernel, lo, degree), fprime(kernel, hi, degree))
        if kernel == "tanh":
            worst = np.where((lo <= 0) & (hi >= 0), 1.0, worst)
        bound = worst * dt + fprime(kernel, t, degree) * ulp32(t) + c_transform(kernel, degree) * ulp32(ref)
    with np.errstate(invalid="ignore"):
        ok = np.abs(got - ref) <= bound
    return ok | (np.isnan(got) & np.isnan(ref)) | (got == ref)
