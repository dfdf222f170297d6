"""neighbors.ball_cover on the GPU against the term-by-term brute force of tests/ball_cover_ref.py: index and distance
outputs equal bit for bit across shapes, k, both metrics, pitched inputs, landmark counts, seeds, query orders and
adversarial data (ties, duplicates, points on a ball's radius, cancellation, subnormal squares, one huge ball, far
queries, NaN and inf), and the epsilon CSR byte for byte at every eps edge."""
import numpy as np
import pytest
import torch

import ball_cover_ref as ref
from raft_b200 import _lib

pytestmark = pytest.mark.gpu

METRICS = ["sqeuclidean", "euclidean"]


def bc():
    from raft_b200.neighbors import ball_cover
    return ball_cover


def cuda(a):
    return torch.as_tensor(np.ascontiguousarray(a, np.float32)).cuda()


def same(a, b):
    """bit-for-bit equality of two tensors (floats compared as their bits)"""
    a, b = a.contiguous(), b.contiguous()
    if a.dtype == torch.float32:
        a, b = a.view(torch.int32), b.view(torch.int32)
    return a.shape == b.shape and torch.equal(a, b)


def check_knn(index, q, x, k, metric):
    dist, idx = bc().knn_query(index, q, k)
    ri, rd = ref.knn(q, x, k, metric)
    assert same(idx, ri), (idx[:2], ri[:2])
    assert same(dist, rd)
    return dist, idx


def check_eps(index, q, x, eps, metric):
    got = bc().eps_nn(index, q, eps)
    want = ref.eps_csr(q, x, eps, metric)
    for g, w in zip(got, want):
        assert same(g, w), (g[:10], w[:10])
    return got


def rng_points(n, d, seed, kind="uniform"):
    r = np.random.default_rng(seed)
    if kind == "uniform":
        return r.random((n, d), dtype=np.float32)
    centers = r.random((8, d)) * 10
    return (centers[r.integers(0, 8, n)] + r.normal(0, 0.3, (n, d))).astype(np.float32)


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("d", [2, 3])
@pytest.mark.parametrize("n", [1, 2, 63, 1000, 100003])
def test_knn_shapes(n, d, metric):
    x = cuda(rng_points(n, d, n + d, "uniform" if n % 2 else "blobs"))
    q = cuda(rng_points(300, d, 7) * 1.2 - 0.1)
    index = bc().build_index(x, metric=metric)
    ks = sorted({k for k in (1, 2, 31, 32, 33, 64, n) if k <= min(64, n)})
    for k in ks:
        check_knn(index, q, x, k, metric)
    # all-kNN: every row finds itself at 0 first unless an equal row has a smaller index
    k = ks[-1]
    dist, idx = bc().all_knn_query(index, k)
    if n <= 20000:
        ri, rd = ref.knn(x, x, k, metric)
    else:
        sel = torch.randperm(n, device="cuda")[:3000]
        ri, rd = ref.knn(x[sel], x, k, metric)
        dist, idx = dist[sel], idx[sel]
    assert same(idx, ri) and same(dist, rd)
    assert (dist[:, 0] == 0).all()


@pytest.mark.parametrize("d", [2, 3])
def test_all_knn_million(d):
    n = 1000000
    x = cuda(rng_points(n, d, 11 + d, "uniform" if d == 2 else "blobs"))
    metric = METRICS[d - 2]
    index = bc().build_index(x, metric=metric)
    for k in (1, 32, 64):
        dist, idx = bc().all_knn_query(index, k)
        sel = torch.randperm(n, device="cuda", generator=torch.Generator("cuda").manual_seed(k))[:2048]
        ri, rd = ref.knn(x[sel], x, k, metric, chunk=128)
        assert same(idx[sel], ri) and same(dist[sel], rd)


def test_pitched_inputs_through_the_c_abi():
    L = _lib.lib()
    n, d, m, k = 5000, 3, 700, 20
    q = cuda(rng_points(m, 5, 4))[:, 1:1 + d]   # pitch 5, offset by one column
    s = torch.cuda.current_stream().cuda_stream
    for metric in METRICS:
        mid = ref.METRIC_IDS[metric]
        wide = cuda(rng_points(n, 7, 3 + mid))
        x = wide[:, :d].contiguous()
        buf = torch.empty(L.b2d_ball_cover_index_bytes(n, d, 0), dtype=torch.uint8, device="cuda")
        ws = torch.empty(L.b2d_ball_cover_build_workspace_bytes(n, d, 0), dtype=torch.uint8, device="cuda")
        _lib.check(L.b2d_ball_cover_build(s, buf.data_ptr(), wide.data_ptr(), 7, n, d, mid, 0, 5, ws.data_ptr(),
                                          ws.numel()))
        wide.fill_(float("nan"))   # the index holds its own copy of the points
        oi = torch.empty((m, k), dtype=torch.int64, device="cuda")
        od = torch.empty((m, k), dtype=torch.float32, device="cuda")
        _lib.check(L.b2d_ball_cover_knn(s, oi.data_ptr(), od.data_ptr(), buf.data_ptr(), n, d, mid, 0, q.data_ptr(), 5, m,
                                        k))
        ri, rd = ref.knn(q.contiguous(), x, k, metric)
        assert same(oi, ri) and same(od, rd)


def test_independent_of_landmarks_seed_and_query_order():
    n, d, k = 20000, 2, 16
    x = cuda(rng_points(n, d, 21, "blobs"))
    q = cuda(rng_points(4000, d, 22) * 10)
    outs = []
    for nl in (1, None, n):
        for seed in (0, 1, 12345678901):
            index = bc().build_index(x, metric="euclidean", n_landmarks=nl, seed=seed)
            outs.append(bc().knn_query(index, q, k) + bc().eps_nn(index, q, 0.25))
    for o in outs[1:]:
        assert all(same(a, b) for a, b in zip(o, outs[0]))
    ri, rd = ref.knn(q, x, k, "euclidean")
    assert same(outs[0][1], ri) and same(outs[0][0], rd)
    index = bc().build_index(x, metric="euclidean")
    perm = torch.randperm(q.shape[0], device="cuda")
    dist, idx = bc().knn_query(index, q[perm].contiguous(), k)
    assert same(idx, outs[0][1][perm]) and same(dist, outs[0][0][perm])
    for _ in range(3):
        again = bc().knn_query(index, q, k)
        assert same(again[0], outs[0][0]) and same(again[1], outs[0][1])


def adversarial(kind, d):
    r = np.random.default_rng(5)
    if kind == "lattice":
        g = np.stack(np.meshgrid(*[np.arange(12 if d == 3 else 40)] * d, indexing="ij"), -1).reshape(-1, d)
        return g.astype(np.float32), (g[r.integers(0, len(g), 500)] + 0.5 * r.integers(0, 2, (500, d))).astype(np.float32)
    if kind == "identical":
        return np.full((3000, d), 0.3, np.float32), np.concatenate([np.full((5, d), 0.3), r.random((100, d))]).astype(np.float32)
    if kind == "duplicates":
        base = r.random((37, d)).astype(np.float32)
        return base[r.integers(0, 37, 5000)], base[r.integers(0, 37, 300)]
    if kind == "on_radius":
        # rings around a centre row: with one landmark at the centre, a ring's members share (nearly) one s, and the
        # outer ring lies on the ball's radius
        ang = np.arange(64) * (2 * np.pi / 64)
        ring = np.stack([np.cos(ang), np.sin(ang)] + [np.zeros(64)] * (d - 2), -1).astype(np.float32)
        rows = [np.zeros((1, d), np.float32)] + [(ring * np.float32(rr)).astype(np.float32) for rr in (1, 2, 4, 8)]
        pts = np.concatenate(rows)
        return pts, (r.random((300, d)) * 16 - 8).astype(np.float32)
    if kind == "cancellation":
        return (1e4 + 1e-2 * r.random((5000, d))).astype(np.float32), (1e4 + 1e-2 * r.random((300, d))).astype(np.float32)
    if kind == "subnormal":
        return (1e-20 * r.random((5000, d))).astype(np.float32), (1e-20 * r.random((300, d))).astype(np.float32)
    if kind == "huge_ball":
        dense = 1e-3 * r.random((20000, d))
        out = 1e3 * r.random((50, d))
        return np.concatenate([dense, out]).astype(np.float32), np.concatenate([1e-3 * r.random((200, d)),
                                                                               1e3 * r.random((100, d))]).astype(np.float32)
    if kind == "far_queries":
        return r.random((5000, d)).astype(np.float32), (1e6 + r.random((300, d)) * 1e5).astype(np.float32)
    raise ValueError(kind)


KINDS = ["lattice", "identical", "duplicates", "on_radius", "cancellation", "subnormal", "huge_ball", "far_queries"]


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("d", [2, 3])
@pytest.mark.parametrize("kind", KINDS)
def test_adversarial(kind, d, metric):
    xn, qn = adversarial(kind, d)
    x, q = cuda(xn), cuda(qn)
    n = x.shape[0]
    dd = ref.dist(q, x, metric)
    typical = float(torch.quantile(dd[:, :min(n, 4000)].flatten().float(), 0.01))
    for nl in (None, 1, max(1, n // 3)):
        index = bc().build_index(x, metric=metric, n_landmarks=nl, seed=nl or 0)
        for k in (1, 16, min(64, n)):
            check_knn(index, q, x, k, metric)
        check_knn(index, x, x, min(64, n), metric)
        check_eps(index, q, x, typical, metric)
        check_eps(index, q, x, 0.0, metric)


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("d", [2, 3])
def test_nan_and_inf_rows_and_queries(d, metric):
    r = np.random.default_rng(9)
    xn = r.random((3000, d)).astype(np.float32)
    xn[r.integers(0, 3000, 40), r.integers(0, d, 40)] = np.nan
    xn[r.integers(0, 3000, 10), r.integers(0, d, 10)] = np.inf
    xn[5, :] = np.nan
    qn = r.random((200, d)).astype(np.float32)
    qn[3, 0] = np.nan
    qn[7, :] = np.nan
    qn[11, 1] = -np.inf
    x, q = cuda(xn), cuda(qn)
    index = bc().build_index(x, metric=metric)
    dist, idx = check_knn(index, q, x, 64, metric)
    assert (idx[3] == -1).all() and (idx[7] == -1).all() and torch.isinf(dist[3]).all()
    check_knn(index, x, x, 33, metric)
    indptr, _, _ = check_eps(index, q, x, 0.05, metric)
    assert indptr[4] == indptr[3] and indptr[8] == indptr[7]
    check_eps(index, q, x, float("inf"), metric)
    # every landmark NaN but one row: the finite rows still find each other
    few = np.full((50, d), np.nan, np.float32)
    few[17] = 0.5
    few[30] = 0.25
    x2 = cuda(few)
    index = bc().build_index(x2, metric=metric, n_landmarks=50)
    check_knn(index, q, x2, 5, metric)


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("d", [2, 3])
def test_eps_edges(d, metric):
    x = cuda(rng_points(2000, d, 31, "blobs"))
    q = cuda(rng_points(400, d, 32) * 10)
    dd = ref.dist(x, x, metric)
    smallest = float(dd[dd > 0].min())
    diameter = float(dd.max())
    typical = float(torch.quantile(dd.flatten()[:1000000], 0.02))
    index = bc().build_index(x, metric=metric)
    for eps in (0.0, smallest, typical, diameter * 1.01, float("inf"), float("nan"), -1.0):
        check_eps(index, q, x, eps, metric)
        check_eps(index, x, x, eps, metric)


def test_agrees_with_brute_force_knn():
    # The expanded form's error is relative to the squared norms, not to the distances: within 1e-6 (|q|^2 + max |x|^2)
    # the two agree, and every row brute_force.knn returns is, measured exactly, within that of our k-th distance.
    from raft_b200.neighbors import brute_force
    for kind, d in (("blobs", 3), ("uniform", 2)):
        x = cuda(rng_points(50000, d, 41, kind))
        q = cuda(rng_points(2000, d, 42) * 10)
        index = bc().build_index(x, metric="sqeuclidean")
        dist, idx = bc().knn_query(index, q, 16)
        bd, bi = brute_force.knn(x, q, 16, metric="sqeuclidean")
        tol = 1e-6 * ((q * q).sum(1, keepdim=True) + (x * x).sum(1).max())
        assert ((dist - bd).abs() <= tol).all()
        exact = torch.gather(ref.dist(q, x, "sqeuclidean"), 1, bi)
        assert (exact <= dist[:, -1:] + tol).all()
        assert (idx == bi).float().mean() > 0.9


def test_argument_errors_raise():
    x = cuda(rng_points(100, 2, 1))
    with pytest.raises(ValueError):
        bc().build_index(x, metric="cosine")
    index = bc().build_index(x)
    with pytest.raises(_lib.LogicError):
        bc().knn_query(index, x, 65)
    with pytest.raises(_lib.LogicError):
        bc().build_index(cuda(rng_points(100, 4, 1)))
