"""fp64 model of kernel_density (b2d_kde_score_samples), from the raw inputs or from a given matrix of squared distances:
out[i] = log(sum_j w_j K(d_ij; h)) - log(sum_j w_j) + log_norm(kernel, h, d), the compact kernels over d^2_ij <
fp32(h h) only, and the normalisation of sklearn's _log_kernel_norm with the exact cosine term."""
import math

import numpy as np
from scipy.special import logsumexp

KERNELS = ("gaussian", "tophat", "epanechnikov", "exponential", "linear", "cosine")
COMPACT = ("tophat", "epanechnikov", "linear", "cosine")


def _log_vn(n):
    return 0.5 * n * math.log(math.pi) - math.lgamma(0.5 * n + 1)


def log_sphere(d):
    """log S_(d-1), the surface of the unit sphere in d dimensions (sklearn's logSn(d - 1))"""
    return math.log(2 * math.pi) + _log_vn(d - 2)


def log_cos_moment(d):
    """log of the integral of t^(d-1) cos(pi t / 2) over [0, 1], from the alternating series in u = 1 - t whose terms fall
    by at least (pi/2)^2 / 12 per step"""
    q, s, t = (math.pi / 2) ** 2, 0.0, 1.0
    for k in range(64):
        s += -t if k % 2 else t
        t *= q / ((d + 2 * k + 2) * (d + 2 * k + 3))
    return math.log(math.pi / 2) - math.log(d) - math.log(d + 1) + math.log(s)


def log_norm(kernel, h, d):
    """-log of the integral of K(|x|; h) over R^d"""
    if kernel == "gaussian":
        f = 0.5 * d * math.log(2 * math.pi)
    elif kernel == "tophat":
        f = _log_vn(d)
    elif kernel == "epanechnikov":
        f = _log_vn(d) + math.log(2.0 / (d + 2.0))
    elif kernel == "exponential":
        f = log_sphere(d) + math.lgamma(d)
    elif kernel == "linear":
        f = _log_vn(d) - math.log(d + 1.0)
    elif kernel == "cosine":
        f = log_sphere(d) + log_cos_moment(d)
    else:
        raise ValueError(kernel)
    return -f - d * math.log(h)


def h2_of(h):
    """the support bound of the compact kernels: fp32(h h), the product formed in fp64"""
    return float(np.float32(h * h))


def log_sum_from_d2(d2, kernel, h, w=None):
    """log(sum_j w_j K) per row of d2 [m, n] (squared distances, any float dtype, evaluated in fp64)"""
    d2 = np.asarray(d2, np.float64)
    w = np.ones(d2.shape[1]) if w is None else np.asarray(w, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        if kernel in ("gaussian", "exponential"):
            logk = -d2 / (2 * h * h) if kernel == "gaussian" else -np.sqrt(d2) / h
            out = logsumexp(logk, axis=1, b=np.broadcast_to(w, d2.shape))
        else:
            t = np.sqrt(d2) / h
            k = {"tophat": np.ones_like(d2), "epanechnikov": 1 - d2 / (h * h), "linear": 1 - t,
                 "cosine": np.cos(0.5 * np.pi * t)}[kernel]
            k = np.where(d2 < h2_of(h), k, 0.0)
            out = np.log((k * w).sum(axis=1))
    out[np.isnan(d2).any(axis=1)] = np.nan
    return out


def score_from_d2(d2, kernel, h, w=None):
    """the model on given squared distances d2 [m, n] without the normalisation (the caller adds log_norm(kernel, h, d))"""
    wsum = d2.shape[1] if w is None else float(np.asarray(w, np.float64).sum())
    return log_sum_from_d2(d2, kernel, h, w) - math.log(wsum)


def d2_64(queries, dataset):
    """exact fp64 squared distances [m, n] (difference form)"""
    q, x = np.asarray(queries, np.float64), np.asarray(dataset, np.float64)
    return ((q[:, None, :] - x[None, :, :]) ** 2).sum(-1)


def score64(dataset, queries, kernel, h, w=None):
    """the model on the raw inputs"""
    d = np.asarray(dataset).shape[1]
    return score_from_d2(d2_64(queries, dataset), kernel, h, w) + log_norm(kernel, h, d)
