"""DBSCAN on the GPU: labels, core_sample_indices and n_clusters equal tests/dbscan_ref.py applied to the adjacency of
one public eps_neighbors_l2sq(x, x, e) call (cosine: pairwise_distance(x, x, "cosine") <= e, the diagonal 0), bit for
bit; the batch plan, repeated runs and a CUDA-graph replay give identical bytes; sklearn.cluster.DBSCAN agrees exactly
where no pair distance is near eps; and a 10^5-row case against the edge-list reference."""
import ctypes

import numpy as np
import pytest

from dbscan_ref import dbscan_ref, dbscan_ref_edges

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
pytest.importorskip("scipy.sparse.csgraph")

from raft_b200 import _lib  # noqa: E402

METRIC_IDS = {"sqeuclidean": 0, "euclidean": 1, "cosine": 2}


def make_data(kind, m, d, seed):
    """blobs of several spreads with uniform noise around them, uniform points, blobs of exact duplicates, or the integer
    lattice 1 .. sqrt(m) in 2-D (every distance exact, massive ties: deep union-find trees; no zero row for cosine)"""
    rng = np.random.default_rng(seed)
    if kind == "lattice":
        side = int(round(m ** 0.5))
        g = np.arange(1, side + 1)
        return np.stack(np.meshgrid(g, g, indexing="ij"), -1).reshape(m, d).astype(np.float32)
    if kind == "uniform":
        return rng.uniform(-1, 1, (m, d)).astype(np.float32)
    centers = rng.uniform(-10, 10, (max(1, m // 150), d))
    lab = rng.integers(0, len(centers), m)
    if kind == "dups":   # few distinct rows, each repeated many times
        base = centers[lab] + rng.standard_normal((m, d))
        return base[rng.integers(0, max(1, m // 20), m)].astype(np.float32)
    spread = rng.choice([0.3, 1.0, 2.0], len(centers))[lab][:, None]
    x = centers[lab] + spread * rng.standard_normal((m, d))
    noise = rng.random(m) < 0.1
    x[noise] = rng.uniform(-12, 12, (int(noise.sum()), d))
    return x.astype(np.float32)


def threshold(metric, eps):
    if not eps >= 0:
        return -1.0
    return float(np.float32(np.float64(eps) ** 2)) if metric == "euclidean" else float(np.float32(eps))


def adjacency(xd, metric, eps):
    """A of the contract, on the device"""
    from raft_b200.distance import pairwise_distance
    from raft_b200.neighbors.epsilon_neighborhood import eps_neighbors_l2sq
    e = threshold(metric, eps)
    if metric != "cosine":
        adj, _ = eps_neighbors_l2sq(xd, xd, e)
        return adj
    m = xd.shape[0]
    dist = torch.empty((m, m), dtype=torch.float32, device="cuda")
    pairwise_distance(xd, xd, out=dist, metric="cosine")
    adj = dist <= e
    adj.fill_diagonal_(e >= 0)
    return adj


def pick_eps(x, metric, density):
    """an eps that makes about `density` of the pairs adjacent"""
    sub = x[:: max(1, len(x) // 400)].astype(np.float64)
    if metric == "cosine":
        n = np.linalg.norm(sub, axis=1)
        n[n == 0] = 1
        dist = 1 - (sub @ sub.T) / np.outer(n, n)
    else:
        dist = ((sub[:, None, :] - sub[None, :, :]) ** 2).sum(-1)
    q = float(np.quantile(dist[~np.eye(len(sub), dtype=bool)], density)) if len(sub) > 1 else 1.0
    return np.sqrt(q) if metric == "euclidean" else q


def run(xd, eps, min_samples, metric, **kw):
    from raft_b200.cluster import dbscan
    o = dbscan(xd, eps, min_samples=min_samples, metric=metric, **kw)
    torch.cuda.synchronize()
    return o.labels.cpu().numpy(), o.core_sample_indices.cpu().numpy(), o.n_clusters


def check(got, want):
    lab, csi, nc = got
    wl, wc, wn = want
    assert lab.tobytes() == wl.tobytes()
    n = int((wc >= 0).sum())
    assert csi.tobytes() == wc[:n].tobytes()
    assert nc == wn


def raw_fit(xp, ldx, m, d, eps, min_samples, metric, max_bytes=0, stream=None):
    """b2d_dbscan_fit on a device pointer with pitch ldx; returns (labels, core_sample_indices [m], n_clusters)"""
    L = _lib.lib()
    lab = torch.full((m,), -7, dtype=torch.int32, device="cuda")
    csi = torch.full((m,), -7, dtype=torch.int32, device="cuda")
    ncl = torch.full((1,), -7, dtype=torch.int32, device="cuda")
    ws = torch.empty(L.b2d_dbscan_workspace_bytes(m, d, max_bytes), dtype=torch.uint8, device="cuda")
    _lib.check(L.b2d_dbscan_fit(stream, METRIC_IDS[metric], xp, ldx, m, d, float(eps), min_samples, max_bytes,
                                lab.data_ptr(), csi.data_ptr(), ncl.data_ptr(), ws.data_ptr(), ws.numel()))
    torch.cuda.synchronize()
    return lab.cpu().numpy(), csi.cpu().numpy(), int(ncl.item())


CASES = [("blobs", 1000, 32), ("blobs", 2049, 3), ("blobs", 1537, 128), ("blobs", 333, 320), ("uniform", 777, 2),
         ("uniform", 1200, 33), ("uniform", 500, 1), ("dups", 900, 31), ("blobs", 1, 5), ("blobs", 2, 1), ("blobs", 17, 3),
         ("lattice", 2500, 2)]


@pytest.mark.parametrize("metric", ["euclidean", "sqeuclidean", "cosine"])
@pytest.mark.parametrize("kind,m,d", CASES)
def test_equals_reference_on_device_adjacency(kind, m, d, metric):
    x = make_data(kind, m, d, seed=m + d)
    xd = torch.from_numpy(x).cuda()
    eps = pick_eps(x, metric, 0.03)
    A = adjacency(xd, metric, eps).cpu().numpy()
    for ms in sorted({1, 2, 5, 50, m + 1}):
        check(run(xd, eps, ms, metric), dbscan_ref(A, ms))


@pytest.mark.parametrize("metric", ["euclidean", "sqeuclidean", "cosine"])
def test_eps_zero_and_negative(metric):
    x = make_data("dups", 700, 9, seed=3)
    xd = torch.from_numpy(x).cuda()
    A = adjacency(xd, metric, 0.0).cpu().numpy()
    for ms in (1, 2, 5):
        check(run(xd, 0.0, ms, metric), dbscan_ref(A, ms))
    for eps in (-0.5, float("nan")):
        lab, csi, nc = run(xd, eps, 1, metric)
        assert (lab == -1).all() and csi.size == 0 and nc == 0


@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
def test_nan_row_is_noise(metric):
    m, d = 1500, 16
    x = make_data("blobs", m, d, seed=9)
    eps = pick_eps(x, metric, 0.03)
    xn = x.copy()
    xn[5, 3] = np.nan
    xd = torch.from_numpy(xn).cuda()
    with pytest.raises(ValueError):
        run(xd, eps, 5, metric)
    A = adjacency(xd, metric, eps).cpu().numpy()
    rest = torch.from_numpy(np.delete(x, 5, axis=0)).cuda()
    for ms in (2, 5):
        got = raw_fit(xd.data_ptr(), d, m, d, eps, ms, metric)
        check((got[0], got[1][got[1] >= 0], got[2]), dbscan_ref(A, ms))
        assert got[0][5] == -1
        other = raw_fit(rest.data_ptr(), d, m - 1, d, eps, ms, metric)
        assert (np.delete(got[0], 5) == other[0]).all() and got[2] == other[2]


def test_padded_leading_dimension():
    m, d, pad = 1100, 20, 7
    x = make_data("blobs", m, d, seed=12)
    xp = torch.full((m, d + pad), float("nan"), device="cuda")
    xp[:, :d] = torch.from_numpy(x).cuda()
    eps = pick_eps(x, "euclidean", 0.03)
    want = run(torch.from_numpy(x).cuda(), eps, 5, "euclidean")
    check(run(xp[:, :d], eps, 5, "euclidean"), (want[0], np.concatenate([want[1], np.int32([-1])]), want[2]))
    lab, csi, nc = raw_fit(xp.data_ptr(), d + pad, m, d, eps, 5, "euclidean")
    assert lab.tobytes() == want[0].tobytes() and nc == want[2]
    assert (csi[:len(want[1])] == want[1]).all() and (csi[len(want[1]):] == -1).all()


@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
def test_batch_plan_and_repeat_give_identical_bytes(metric):
    m, d = 3001, 16
    x = make_data("blobs", m, d, seed=21)
    xd = torch.from_numpy(x).cuda()
    eps = pick_eps(x, metric, 0.03)
    # one batch; 256 columns (a last batch of 185); 1280 (last 441); 768 (last 697)
    plans = [0, m * 256, m * 256 * 5, m * 1000]
    outs = [raw_fit(xd.data_ptr(), d, m, d, eps, 5, metric, mb) for mb in plans]
    outs.append(raw_fit(xd.data_ptr(), d, m, d, eps, 5, metric, plans[1]))
    for o in outs[1:]:
        assert o[0].tobytes() == outs[0][0].tobytes() and o[1].tobytes() == outs[0][1].tobytes() and o[2] == outs[0][2]
    A = adjacency(xd, metric, eps).cpu().numpy()
    want = dbscan_ref(A, 5)
    assert outs[0][0].tobytes() == want[0].tobytes() and outs[0][1].tobytes() == want[1].tobytes()
    # the Python batch size in MiB
    check(run(xd, eps, 5, metric, max_mbytes_per_batch=1), want)


def test_equals_sklearn_with_margin():
    cluster = pytest.importorskip("sklearn.cluster")
    m, d = 240, 3
    rng = np.random.default_rng(5)
    centers = rng.uniform(-6, 6, (6, d))
    x = (centers[rng.integers(0, 6, m)] + rng.standard_normal((m, d)) * rng.choice([0.4, 0.8], m)[:, None])
    x = x.astype(np.float32)
    x64 = x.astype(np.float64)
    d2 = ((x64[:, None, :] - x64[None, :, :]) ** 2).sum(-1)
    # eps^2 in the middle of the widest relative gap between pair distances in the 1 % - 15 % range
    v = np.sort(d2[np.triu_indices(m, 1)])
    seg = v[int(0.01 * v.size):int(0.15 * v.size)]
    g = int(np.argmax(seg[1:] / seg[:-1]))
    eps = float(np.sqrt(np.sqrt(seg[g] * seg[g + 1])))
    rel = np.abs(d2 - eps * eps) / (eps * eps)
    assert rel.min() > 1e-3, rel.min()
    xd = torch.from_numpy(x).cuda()
    mixed = 0
    for ms in (1, 4, 10, 30):
        sk = cluster.DBSCAN(eps=eps, min_samples=ms).fit(x64)
        lab, csi, nc = run(xd, eps, ms, "euclidean")
        assert (lab == sk.labels_).all() and (csi == sk.core_sample_indices_).all()
        assert nc == len(set(sk.labels_.tolist()) - {-1})
        mixed += bool((lab >= 0).any() and (lab == -1).any() and csi.size < (lab >= 0).sum())   # core, border, noise
    assert mixed


def test_large_against_edge_list_reference():
    from raft_b200.neighbors.epsilon_neighborhood import eps_neighbors_l2sq
    m, d = 100000, 32
    x = make_data("blobs", m, d, seed=77)
    xd = torch.from_numpy(x).cuda()
    eps = pick_eps(x, "euclidean", 0.001)
    adj, vd = eps_neighbors_l2sq(xd, xd, threshold("euclidean", eps))   # one call: the whole m x m adjacency
    rows, cols = [], []
    for r0 in range(0, m, 10000):   # its entries, a block of rows at a time
        nz = torch.nonzero(adj[r0:r0 + 10000])
        rows.append((nz[:, 0] + r0).cpu().numpy())
        cols.append(nz[:, 1].cpu().numpy())
    del adj
    rows, cols = np.concatenate(rows), np.concatenate(cols)
    for ms in (5, 50):
        want = dbscan_ref_edges(rows, cols, m, ms)
        got = run(xd, eps, ms, "euclidean")
        check(got, want)
        assert want[2] > 1 and (got[0] == -1).any() and (got[0] >= 0).any()


def test_cuda_graph_replay():
    m, d = 5000, 24
    x = make_data("blobs", m, d, seed=31)
    xd = torch.from_numpy(x).cuda()
    eps = pick_eps(x, "euclidean", 0.03)
    want = raw_fit(xd.data_ptr(), d, m, d, eps, 5, "euclidean", m * 512)
    L = _lib.lib()
    lab = torch.full((m,), -7, dtype=torch.int32, device="cuda")
    csi = torch.full((m,), -7, dtype=torch.int32, device="cuda")
    ncl = torch.full((1,), -7, dtype=torch.int32, device="cuda")
    ws = torch.empty(L.b2d_dbscan_workspace_bytes(m, d, m * 512), dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(g, stream=s):
        _lib.check(L.b2d_dbscan_fit(ctypes.c_void_p(s.cuda_stream), 1, xd.data_ptr(), d, m, d, float(eps), 5, m * 512,
                                    lab.data_ptr(), csi.data_ptr(), ncl.data_ptr(), ws.data_ptr(), ws.numel()))
    lab.fill_(-7)
    csi.fill_(-7)
    ncl.fill_(-7)
    g.replay()
    torch.cuda.synchronize()
    assert lab.cpu().numpy().tobytes() == want[0].tobytes() and csi.cpu().numpy().tobytes() == want[1].tobytes()
    assert int(ncl.item()) == want[2]


def test_empty_and_single_row():
    from raft_b200.cluster import dbscan
    o = dbscan(torch.empty((0, 4), device="cuda"), 1.0)
    assert o.labels.numel() == 0 and o.core_sample_indices.numel() == 0 and o.n_clusters == 0
    o = dbscan(torch.zeros((1, 4), device="cuda"), 1.0, min_samples=1)
    assert o.labels.tolist() == [0] and o.core_sample_indices.tolist() == [0] and o.n_clusters == 1
    with pytest.raises(ValueError):
        dbscan(torch.full((3, 2), float("inf"), device="cuda"), 1.0)
