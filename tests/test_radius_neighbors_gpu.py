"""GPU tier: radius_neighbors (the fused radius query as CSR) is bit for bit the composition it replaces --
D = pairwise_distance(q, x, metric), D <= r, each row sorted by oracle.pack_minloc(D, j) -- for every metric, ragged
shapes on both kernel variants, radii at and around the edge cases, ties, self pairs, rows that never match, rows longer
than any shared-memory sort tile and several work items per CTA; plus the fp64 check outside the rounding band,
reproducibility, graph capture and the nnz guard of the C ABI."""
import numpy as np
import pytest
import torch

import oracle
from radius_ref import METRIC_IDS, composition, dist64
from raft_b200 import _lib
from raft_b200.distance import pairwise_distance
from raft_b200.neighbors import radius_neighbors

pytestmark = pytest.mark.gpu
DEV = "cuda"
METRICS = ["sqeuclidean", "euclidean", "cosine", "correlation"]


def blobs(m, n, k, seed=0):
    q, _, c = oracle.make_blobs(m, k, seed=411 + seed)
    x, _, _ = oracle.make_blobs(n, k, seed=877 + seed, centers=c)
    return torch.from_numpy(q).to(DEV), torch.from_numpy(x).to(DEV)


def pdist(q, x, metric):
    out = torch.empty((q.shape[0], x.shape[0]), dtype=torch.float32, device=DEV)
    pairwise_distance(q, x, out=out, metric=metric)
    return out


def r_at(d, frac):
    """a radius that is itself one of the distances (so '<=' is tested at equality), about a fraction frac of the pairs"""
    flat = d.flatten()
    flat = flat[~torch.isnan(flat)]
    return float(flat.kthvalue(max(1, int(frac * flat.numel()))).values)


def host(csr):
    return tuple(t.cpu().numpy() for t in csr)


def assert_csr_equal(got, want):
    gp, gi, gd = got
    wp, wi, wd = want
    assert np.array_equal(gp, wp)
    assert np.array_equal(gi, wi)
    assert np.array_equal(np.asarray(gd, np.float32).view(np.int32), np.asarray(wd, np.float32).view(np.int32))


def check(x, q, r, metric):
    """the fused call against the composition; returns the fused CSR (host arrays)"""
    got = host(radius_neighbors(x, q, r, metric=metric))
    assert_csr_equal(got, composition(pdist(q, x, metric).cpu().numpy(), r))
    return got


def raw(q, x, r, metric, m=None, n=None, k=None, ldq=None, ldx=None, stream=0, nnz=None, indices=None, distances=None):
    """both C calls; q / x torch tensors whose rows may be padded (ldq / ldx).  Returns (indptr, indices, distances, ws)."""
    L = _lib.lib()
    m = q.shape[0] if m is None else m
    n = x.shape[0] if n is None else n
    k = q.shape[1] if k is None else k
    ldq = q.shape[1] if ldq is None else ldq
    ldx = x.shape[1] if ldx is None else ldx
    mid = METRIC_IDS[metric]
    indptr = torch.full((m + 1,), -5, dtype=torch.int64, device=DEV)
    ws = torch.empty(L.b2d_radius_neighbors_workspace_bytes(m, n, k, 0) + 256, dtype=torch.uint8, device=DEV)
    _lib.check(L.b2d_radius_neighbors_count(stream, indptr.data_ptr(), mid, q.data_ptr(), ldq, x.data_ptr(), ldx, m, n, k,
                                            r, ws.data_ptr(), ws.numel()))
    torch.cuda.synchronize()
    total = int(indptr[m])
    nnz = total if nnz is None else nnz
    if indices is None:
        indices = torch.empty(nnz, dtype=torch.int64, device=DEV)
        distances = torch.empty(nnz, dtype=torch.float32, device=DEV)
    ws = torch.empty(L.b2d_radius_neighbors_workspace_bytes(m, n, k, nnz) + 256, dtype=torch.uint8, device=DEV)
    _lib.check(L.b2d_radius_neighbors_fill(stream, indptr.data_ptr(), nnz, indices.data_ptr(), distances.data_ptr(), mid,
                                           q.data_ptr(), ldq, x.data_ptr(), ldx, m, n, k, r, ws.data_ptr(), ws.numel()))
    torch.cuda.synchronize()
    return indptr, indices, distances


# m % 128 in {1, 64, 65, 127} with n % 256 in {1, 128, 129, 255}
SHAPES = [(129, 513), (192, 384), (193, 385), (255, 511)]


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("k", [24, 128, 129, 320])
@pytest.mark.parametrize("m,n", SHAPES)
def test_equals_composition(m, n, k, metric):
    q, x = blobs(m, n, k, seed=k + m)
    r = r_at(pdist(q, x, metric), 0.01)
    got = check(x, q, r, metric)
    assert got[0][-1] >= int(0.01 * m * n)   # the radius is the int(0.01 m n)-th smallest distance
    assert (got[2] == np.float32(r)).any()   # the pair at exactly the radius is in


@pytest.mark.parametrize("metric", METRICS)
def test_radius_edge_values(metric):
    m, n, k = 193, 385, 40
    q, x = blobs(m, n, k, seed=3)
    d = pdist(q, x, metric)
    for r in (-1e-3, -0.0, float("nan"), float("inf"), 0.0, r_at(d, 0.3)):
        got = check(x, q, r, metric)
        if not (r >= 0):
            assert got[0].tolist() == [0] * (m + 1) and len(got[1]) == 0
    inf = host(radius_neighbors(x, q, float("inf"), metric=metric))
    assert inf[0][-1] == m * n   # blobs have no NaN distance


@pytest.mark.parametrize("metric", METRICS)
def test_duplicate_rows_ties_ordered_by_index(metric):
    m, k = 130, 33
    q, base = blobs(m, 40, k, seed=5)
    rng = np.random.default_rng(9)
    x = base[torch.from_numpy(rng.integers(0, 40, size=1000)).to(DEV)].contiguous()   # every row about 25 times
    d = pdist(q, x, metric)
    got = check(x, q, r_at(d, 0.2), metric)
    # (the composition orders equal distances by ascending index) and there are many of them
    rows = np.repeat(np.arange(m), np.diff(got[0]))
    same = (got[2][1:] == got[2][:-1]) & (rows[1:] == rows[:-1])
    assert same.sum() > 1000


@pytest.mark.parametrize("metric", ["sqeuclidean", "euclidean"])
def test_self_pairs_only_for_the_same_matrix(metric):
    n, k = 300, 50
    _, x = blobs(10, n, k, seed=7)
    got = check(x, x, 0.0, metric)   # x is x: the diagonal is at exactly 0
    rows = np.repeat(np.arange(n), np.diff(got[0]))
    diag = got[1] == rows
    assert diag.sum() == n and (got[2][diag] == 0).all()
    y = x.clone()   # a copy gets no such rule: the composition of pairwise_distance(y, x) again
    check(x, y, r_at(pdist(y, x, metric), 0.05), metric)


@pytest.mark.parametrize("metric", METRICS)
def test_rows_that_never_match(metric):
    m, n, k = 150, 400, 16
    q, x = blobs(m, n, k, seed=11)
    q[3, 5] = float("nan")
    x[7, 2] = float("nan")
    if metric == "cosine":
        q[10] = 0.0
        x[20] = 0.0
    if metric == "correlation":
        q[10] = 1.5
        x[20] = -2.0
    got = check(x, q, float("inf"), metric)
    assert got[0][4] == got[0][3]           # the NaN query row has no pair
    assert not (got[1] == 7).any()          # the NaN dataset row is in no row
    if metric in ("cosine", "correlation"):
        assert got[0][11] == got[0][10] and not (got[1] == 20).any()


def test_rows_longer_than_a_sort_tile():
    m, n, k = 5, 70001, 24
    q, x = blobs(m, n, k, seed=13)
    got = check(x, q, float("inf"), "sqeuclidean")
    assert np.diff(got[0]).tolist() == [n] * m


def test_several_items_per_cta():
    m, n, k = 40000, 1000, 32
    q, x = blobs(m, n, k, seed=17)
    check(x, q, r_at(pdist(q[:2000], x, "euclidean"), 0.01), "euclidean")


@pytest.mark.parametrize("metric", METRICS)
def test_membership_agrees_with_fp64_outside_band(metric):
    m, n, k = 300, 700, 96
    q, x = blobs(m, n, k, seed=19)
    r = r_at(pdist(q, x, metric), 0.05)
    indptr, indices, _ = host(radius_neighbors(x, q, r, metric=metric))
    d64 = dist64(q.cpu().numpy(), x.cpu().numpy(), metric)
    hit = np.zeros((m, n), bool)
    hit[np.repeat(np.arange(m), np.diff(indptr)), indices] = True
    clear = np.abs(d64 - r) > 1e-4 * max(1.0, abs(r))
    assert clear.mean() > 0.95
    assert np.array_equal(hit[clear], (d64 <= r)[clear])


def test_reproducible_bytes():
    q, x = blobs(700, 3000, 128, seed=23)
    r = r_at(pdist(q, x, "cosine"), 0.02)
    a = host(radius_neighbors(x, q, r, metric="cosine"))
    b = host(radius_neighbors(x, q, r, metric="cosine"))
    assert_csr_equal(a, b)


def test_padded_leading_dimension_through_the_c_abi():
    m, n, k = 193, 385, 129
    q, x = blobs(m, n, k, seed=29)
    qp = torch.zeros((m, k + 7), dtype=torch.float32, device=DEV)
    xp = torch.zeros((n, k + 3), dtype=torch.float32, device=DEV)
    qp[:, :k] = q
    xp[:, :k] = x
    for metric in METRICS:
        r = r_at(pdist(q, x, metric), 0.03)
        got = host(raw(qp, xp, r, metric, k=k, ldq=k + 7, ldx=k + 3))
        assert_csr_equal(got, composition(pdist(q, x, metric).cpu().numpy(), r))


def test_cuda_graph_capture():
    m, n, k, metric = 600, 2048, 64, "euclidean"
    q, x = blobs(m, n, k, seed=31)
    r = r_at(pdist(q, x, metric), 0.02)
    want = composition(pdist(q, x, metric).cpu().numpy(), r)
    nnz = int(want[0][-1])
    L = _lib.lib()
    mid = METRIC_IDS[metric]
    indptr = torch.empty(m + 1, dtype=torch.int64, device=DEV)
    indices = torch.empty(nnz, dtype=torch.int64, device=DEV)
    distances = torch.empty(nnz, dtype=torch.float32, device=DEV)
    ws = torch.empty(L.b2d_radius_neighbors_workspace_bytes(m, n, k, nnz), dtype=torch.uint8, device=DEV)
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        _lib.check(L.b2d_radius_neighbors_count(s.cuda_stream, indptr.data_ptr(), mid, q.data_ptr(), k, x.data_ptr(), k, m,
                                                n, k, r, ws.data_ptr(), ws.numel()))
        _lib.check(L.b2d_radius_neighbors_fill(s.cuda_stream, indptr.data_ptr(), nnz, indices.data_ptr(),
                                               distances.data_ptr(), mid, q.data_ptr(), k, x.data_ptr(), k, m, n, k, r,
                                               ws.data_ptr(), ws.numel()))
    for _ in range(2):
        indptr.fill_(-1)
        indices.fill_(-1)
        distances.fill_(-1)
        g.replay()
        torch.cuda.synchronize()
        assert_csr_equal(host((indptr, indices, distances)), want)


def test_fill_never_writes_past_nnz():
    m, n, k, metric = 257, 1000, 48, "sqeuclidean"
    q, x = blobs(m, n, k, seed=37)
    r = r_at(pdist(q, x, metric), 0.05)
    want = composition(pdist(q, x, metric).cpu().numpy(), r)
    total = int(want[0][-1])
    nnz = total // 2
    guard = 4096
    ibuf = torch.full((nnz + guard,), -7, dtype=torch.int64, device=DEV)
    dbuf = torch.full((nnz + guard,), -7.0, dtype=torch.float32, device=DEV)
    indptr, _, _ = raw(q, x, r, metric, nnz=nnz, indices=ibuf, distances=dbuf)
    assert int(indptr[m]) == total
    assert (ibuf[nnz:] == -7).all() and (dbuf[nnz:] == -7.0).all()
    # the rows that end at or before nnz are complete and exact
    full = int(np.searchsorted(want[0], nnz, side="right")) - 1
    e = int(want[0][full])
    assert full > 10
    assert np.array_equal(ibuf[:e].cpu().numpy(), want[1][:e])
    assert np.array_equal(dbuf[:e].cpu().numpy().view(np.int32), want[2][:e].view(np.int32))


@pytest.mark.parametrize("metric", METRICS)
def test_empty_inputs(metric):
    q, x = blobs(70, 90, 8, seed=41)
    p, i, d = radius_neighbors(x, q[:0], 1.0, metric=metric)
    assert p.tolist() == [0] and i.numel() == 0 and d.numel() == 0
    p, i, d = radius_neighbors(x[:0], q, 1.0, metric=metric)
    assert p.tolist() == [0] * 71 and i.numel() == 0 and d.numel() == 0
