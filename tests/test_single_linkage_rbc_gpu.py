"""Exact single linkage on the random ball cover on the GPU: the EMST edges and the single-linkage outputs equal the
oracle (tests/emst_ref.py: Kruskal over every pair in the contract's order, on the fp32 term-by-term pair value) byte for
byte.  Covered: m from 1 to 5000, both d and both metrics; the ball cover tests' hard data (an integer lattice with
massive ties, exact duplicates, rows on a ball's radius, a 1e4 offset with a 1e-2 spread, 1e-20 coordinates, one dense
ball with far outliers, well-separated blobs); independence from n_landmarks and the seed; a pitched x, repeated calls
and a CUDA-graph replay of b2d_emst_rbc; a non-finite x; agreement with linkage="knn_graph" where that graph is
complete; and 2 10^5 rows against Kruskal over the pairs ball_cover.eps_nn finds within the tree's longest edge."""
import ctypes

import numpy as np
import pytest

import emst_ref
from single_linkage_ref import _find, edge_order

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

from raft_b200 import _lib  # noqa: E402

METRICS = ["sqeuclidean", "euclidean"]
METRIC_IDS = {"sqeuclidean": 4, "euclidean": 5}


def cuda(a):
    return torch.as_tensor(np.ascontiguousarray(a, np.float32)).cuda()


def points(m, d, seed, kind="uniform"):
    r = np.random.default_rng(seed)
    if kind == "uniform":
        return r.random((m, d), dtype=np.float32)
    if kind == "lattice":   # every axis pair at s = 1: ties everywhere
        side = int(np.ceil(m ** (1 / d)))
        g = np.stack(np.meshgrid(*[np.arange(side)] * d, indexing="ij"), -1).reshape(-1, d)
        return g[:m].astype(np.float32)
    if kind == "duplicates":   # s = 0 between distinct rows
        return r.random((max(1, m // 8), d)).astype(np.float32)[r.integers(0, max(1, m // 8), m)]
    if kind == "ring":   # rows on circles / spheres around a few centres: many on a ball's radius
        c = r.random((4, d)) * 10
        v = r.normal(size=(m, d))
        v /= np.linalg.norm(v, axis=1, keepdims=True)
        return (c[r.integers(0, 4, m)] + v).astype(np.float32)
    if kind == "cancellation":
        return (1e4 + 1e-2 * r.random((m, d))).astype(np.float32)
    if kind == "subnormal":
        return (1e-20 * r.random((m, d))).astype(np.float32)
    if kind == "dense_ball":
        return np.concatenate([1e-3 * r.random((m - 20, d)), 1e3 * r.random((20, d))]).astype(np.float32)
    if kind == "blobs":   # well separated: the late rounds have a few large components
        c = r.random((6, d)) * 1000
        return (c[r.integers(0, 6, m)] + r.normal(0, 1, (m, d))).astype(np.float32)
    raise ValueError(kind)


def run_emst(x, metric, **kw):
    from raft_b200.cluster import emst
    o = emst(x, metric=metric, **kw)
    torch.cuda.synchronize()
    return o.src.cpu().numpy(), o.dst.cpu().numpy(), o.weights.cpu().numpy()


def run_sl(x, nc, metric, **kw):
    from raft_b200.cluster import single_linkage
    o = single_linkage(x, nc, metric=metric, linkage="pairwise", **kw)
    assert o.n_connected_components == 1
    return o.children.cpu().numpy(), o.deltas.cpu().numpy(), o.sizes.cpu().numpy(), o.labels.cpu().numpy()


def same(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        g, w = np.asarray(g), np.asarray(w)
        assert g.dtype == w.dtype and g.shape == w.shape and g.tobytes() == w.tobytes(), (g[:8], w[:8])


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("d", [2, 3])
@pytest.mark.parametrize("m", [1, 2, 3, 33, 257, 1000, 5000])
def test_shapes(m, d, metric):
    xn = points(m, d, 10 * m + d)
    x = cuda(xn)
    want = emst_ref.emst(xn, metric)
    same(run_emst(x, metric), want)
    for nc in sorted({1, min(m, 2), min(m, 7), m}):
        same(run_sl(x, nc, metric), emst_ref.linkage(want, nc, metric))


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("d", [2, 3])
@pytest.mark.parametrize("kind", ["lattice", "duplicates", "ring", "cancellation", "subnormal", "dense_ball", "blobs"])
def test_adversarial(kind, d, metric):
    xn = points(1500, d, 5, kind)
    x = cuda(xn)
    want = emst_ref.emst(xn, metric)
    for nl in (None, 1, 40):
        same(run_emst(x, metric, n_landmarks=nl, seed=nl or 0), want)
    same(run_sl(x, 6, metric), emst_ref.linkage(want, 6, metric))


def test_independent_of_landmarks_and_seed():
    m, d = 4000, 2
    xn = points(m, d, 21, "blobs")
    x = cuda(xn)
    want = emst_ref.emst(xn, "euclidean")
    for nl in (1, 2, int(np.ceil(np.sqrt(m))), m):
        for seed in (0, 1, 12345678901):
            same(run_emst(x, "euclidean", n_landmarks=nl, seed=seed), want)
    ch = emst_ref.linkage(want, 6, "euclidean")
    for nl in (1, m):
        same(run_sl(x, 6, "euclidean", n_landmarks=nl, seed=3), ch)


def raw_emst(xp, ldx, m, d, metric, nl=0, seed=0, stream=None):
    L = _lib.lib()
    src = torch.full((m - 1,), -7, dtype=torch.int32, device="cuda")
    dst = torch.full((m - 1,), -7, dtype=torch.int32, device="cuda")
    w = torch.full((m - 1,), -7, dtype=torch.float32, device="cuda")
    ws = torch.empty(L.b2d_emst_rbc_workspace_bytes(m, d, nl), dtype=torch.uint8, device="cuda")
    _lib.check(L.b2d_emst_rbc(stream, METRIC_IDS[metric], xp, ldx, m, d, nl, seed, src.data_ptr(), dst.data_ptr(),
                              w.data_ptr(), ws.data_ptr(), ws.numel()))
    torch.cuda.synchronize()
    return src.cpu().numpy(), dst.cpu().numpy(), w.cpu().numpy()


def test_pitched_input_through_the_c_abi():
    m, d = 3000, 3
    wide = cuda(points(m, 6, 4))
    xn = wide[:, 1:1 + d].cpu().numpy()
    for metric in METRICS:
        same(raw_emst(wide.data_ptr() + 4, 6, m, d, metric, nl=17, seed=3), emst_ref.emst(xn, metric))
    from raft_b200.cluster import single_linkage
    o = single_linkage(wide[:, 1:1 + d], 5, linkage="pairwise")   # a strided view through Python
    same((o.children.cpu().numpy(), o.deltas.cpu().numpy(), o.sizes.cpu().numpy(), o.labels.cpu().numpy()),
         emst_ref.single_linkage(xn, 5, "euclidean"))


def test_repeat_and_cuda_graph_replay():
    m, d = 5000, 2
    xn = points(m, d, 41, "blobs")
    x = cuda(xn)
    want = raw_emst(x.data_ptr(), d, m, d, "euclidean")
    same(raw_emst(x.data_ptr(), d, m, d, "euclidean"), want)
    same(want, emst_ref.emst(xn, "euclidean"))
    L = _lib.lib()
    src = torch.full((m - 1,), -7, dtype=torch.int32, device="cuda")
    dst = torch.full((m - 1,), -7, dtype=torch.int32, device="cuda")
    w = torch.full((m - 1,), -7, dtype=torch.float32, device="cuda")
    ws = torch.empty(L.b2d_emst_rbc_workspace_bytes(m, d, 0), dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(g, stream=s):
        _lib.check(L.b2d_emst_rbc(ctypes.c_void_p(s.cuda_stream), 5, x.data_ptr(), d, m, d, 0, 0, src.data_ptr(),
                                  dst.data_ptr(), w.data_ptr(), ws.data_ptr(), ws.numel()))
    for _ in range(2):
        for t in (src, dst, w):
            t.fill_(-7)
        g.replay()
        torch.cuda.synchronize()
        same((src.cpu().numpy(), dst.cpu().numpy(), w.cpu().numpy()), want)


def test_non_finite_input():
    from raft_b200.cluster import emst, single_linkage
    for bad in (float("nan"), float("inf")):
        x = cuda(points(300, 2, 3))
        x[17, 1] = bad
        with pytest.raises(_lib.LogicError, match="non-finite"):
            single_linkage(x, 3, linkage="pairwise")
        with pytest.raises(ValueError):
            emst(x)
        # the C ABI's EMST states finiteness as a precondition: the call is safe, its output unspecified
        raw_emst(x.data_ptr(), 2, 300, 2, "euclidean")


def test_single_row():
    from raft_b200.cluster import emst, single_linkage
    o = emst(torch.zeros((1, 3), device="cuda"))
    assert o.src.numel() == 0 and o.dst.numel() == 0 and o.weights.numel() == 0
    o = single_linkage(torch.zeros((1, 2), device="cuda"), 1, linkage="pairwise")
    assert o.children.shape == (0, 2) and o.labels.tolist() == [0]


@pytest.mark.parametrize("d", [2, 3])
def test_agrees_with_knn_graph_where_it_is_complete(d):
    # small integers: the squared distances are exact in the expanded and the unexpanded form, and with m <= 64 and c
    # large enough n_nb = m, so the kNN graph is complete and both linkages are exact
    from raft_b200.cluster import single_linkage
    r = np.random.default_rng(60 + d)
    for m in (9, 40, 64):
        xn = r.integers(0, 50, (m, d)).astype(np.float32)
        x = cuda(xn)
        a = single_linkage(x, 3, metric="sqeuclidean", linkage="pairwise")
        b = single_linkage(x, 3, metric="sqeuclidean", c=64)
        assert torch.equal(a.deltas, b.deltas)
        # where the weights are distinct, the merges are forced: the trees agree
        w = a.deltas.cpu().numpy()
        if len(np.unique(w)) == len(w):
            assert torch.equal(a.children, b.children) and torch.equal(a.sizes, b.sizes)
            assert torch.equal(a.labels, b.labels)


def test_scale_against_eps_nn_kruskal():
    # the tree lies in the graph of the pairs within its longest edge, so Kruskal over ball_cover.eps_nn at that eps,
    # in the contract's order, must give the tree edge for edge
    from raft_b200.neighbors import ball_cover
    m, d = 200000, 2
    x = torch.rand((m, d), generator=torch.Generator("cuda").manual_seed(7), device="cuda")
    src, dst, w = run_emst(x, "sqeuclidean")
    eps = float(w.max())
    index = ball_cover.build_index(x, metric="sqeuclidean")
    indptr, indices, dist = ball_cover.eps_nn(index, x, eps)
    rows = torch.repeat_interleave(torch.arange(m, device="cuda"), indptr[1:] - indptr[:-1])
    keep = rows < indices
    a, b, s = rows[keep].cpu().numpy(), indices[keep].cpu().numpy(), dist[keep].cpu().numpy()
    # positions in (min row, max row) order, then Kruskal's (w, position) order is the contract's
    o = np.lexsort((b, a))
    a, b, s = a[o], b[o], s[o]
    p = list(range(m))
    chosen = []
    for e in edge_order(s):
        ra, rb = _find(p, int(a[e])), _find(p, int(b[e]))
        if ra != rb:
            p[max(ra, rb)] = min(ra, rb)
            chosen.append(int(e))
            if len(chosen) == m - 1:
                break
    chosen = np.array(chosen)
    same((src, dst, w), (a[chosen].astype(np.int32), b[chosen].astype(np.int32), s[chosen]))
