"""fp64 reference of the epsilon neighbourhood, shared by the CPU and GPU tests of eps_neighbors_l2sq."""
import numpy as np


def sqdist64(x, y):
    """squared L2 distances in fp64 in the expanded form, clamped at 0, and the scale |x_i|^2 + |y_j|^2 (at least 1) that
    bounds the fp32 error of the tensor path"""
    x64, y64 = np.asarray(x, np.float64), np.asarray(y, np.float64)
    nx, ny = (x64 ** 2).sum(1)[:, None], (y64 ** 2).sum(1)[None, :]
    return np.maximum(nx + ny - 2 * x64 @ y64.T, 0), np.maximum(nx + ny, 1.0)


def ref_eps(x, y, eps):
    """adjacency, per-column degrees with the total appended, and the mask of pairs outside the band
    |d - eps| <= 1e-5 * scale, where the fp32 result may fall either way"""
    d, scale = sqdist64(x, y)
    adj = d <= eps
    cnt = adj.sum(0)
    return adj, np.concatenate([cnt, [cnt.sum()]]), np.abs(d - eps) > 1e-5 * scale
