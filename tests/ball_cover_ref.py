"""The oracle of the ball-cover tests: a brute force on the device that evaluates the contract's distance term by term,
as separate elementwise float32 ops with explicit column adds (each rounded on its own), and orders neighbours by the
int64 key (distance bits << 32) | index.  A pair at a NaN distance is never a neighbour."""
import torch

KEY_NONE = 2 ** 63 - 1
METRIC_IDS = {"sqeuclidean": 4, "euclidean": 5}


def dist(q, x, metric):
    """float32 [m, n]: s = ((q0-x0)*(q0-x0) + (q1-x1)*(q1-x1)) + (q2-x2)*(q2-x2), sqrt(s) for "euclidean"."""
    s = None
    for c in range(q.shape[1]):
        t = q[:, c:c + 1] - x[:, c][None, :]
        t = t * t
        s = t if s is None else s + t
    return torch.sqrt(s) if metric == "euclidean" else s


def keys(d):
    """int64 keys of a distance block (distances >= 0 or NaN), KEY_NONE for NaN"""
    idx = torch.arange(d.shape[1], device=d.device, dtype=torch.int64)
    k = (d.contiguous().view(torch.int32).to(torch.int64) << 32) | idx[None, :]
    return torch.where(torch.isnan(d), torch.full_like(k, KEY_NONE), k)


def split(k):
    """keys -> (indices int64, distances float32), KEY_NONE -> (-1, +inf)"""
    none = k == KEY_NONE
    idx = torch.where(none, torch.full_like(k, -1), k & 0xFFFFFFFF)
    d = (k >> 32).to(torch.int32).view(torch.float32)
    return idx, torch.where(none, torch.full_like(d, float("inf")), d)


def knn(q, x, k, metric, chunk=None):
    """(indices int64 [m, k], distances float32 [m, k]) of the k smallest keys of every query row"""
    chunk = chunk or max(1, (1 << 27) // max(1, x.shape[0]))
    out_i, out_d = [], []
    for a in range(0, q.shape[0], chunk):
        kk = torch.topk(keys(dist(q[a:a + chunk], x, metric)), k, dim=1, largest=False, sorted=True).values
        i, d = split(kk)
        out_i.append(i)
        out_d.append(d)
    return torch.cat(out_i), torch.cat(out_d)


def eps_csr(q, x, eps, metric):
    """(indptr, indices, distances) of every pair with distance <= eps, rows in key order"""
    d = dist(q, x, metric)
    k = keys(d)
    hit = d <= eps
    k = torch.where(hit, k, torch.full_like(k, KEY_NONE))
    k = torch.sort(k, dim=1).values
    cnt = hit.sum(dim=1)
    indptr = torch.zeros(q.shape[0] + 1, dtype=torch.int64, device=q.device)
    indptr[1:] = torch.cumsum(cnt, 0)
    flat = k[torch.arange(k.shape[1], device=q.device)[None, :] < cnt[:, None]]
    i, dd = split(flat)
    return indptr, i, dd
