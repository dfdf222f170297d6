"""GPU tier: eps_neighbors_l2sq (the fused epsilon neighbourhood) is bit for bit the composition it replaces,
pairwise_distance(x, y, "sqeuclidean") <= eps with per-column sums, on both adjacency store paths, both kernel variants
and ragged shapes; plus the fp64 check outside the rounding band, self pairs, counts and the C ABI's modes."""
import numpy as np
import pytest
import torch

import oracle
from eps_ref import ref_eps, sqdist64
from raft_b200 import LogicError, _lib
from raft_b200.distance import pairwise_distance
from raft_b200.neighbors import eps_neighbors_l2sq

pytestmark = pytest.mark.gpu
DEV = "cuda"


def blobs(m, n, k, seed=0):
    x, _, c = oracle.make_blobs(m, k, seed=311 + seed)
    y, _, _ = oracle.make_blobs(n, k, seed=733 + seed, centers=c)
    return torch.from_numpy(x).to(DEV), torch.from_numpy(y).to(DEV)


def sqeuclidean(x, y):
    out = torch.empty((x.shape[0], y.shape[0]), dtype=torch.float32, device=DEV)
    pairwise_distance(x, y, out=out, metric="sqeuclidean")
    return out


def eps_at(d, q):
    """an eps that is itself one of the distances (so '<=' is tested at equality), about a fraction q adjacent"""
    flat = d.flatten()
    return float(flat.kthvalue(max(1, int(q * flat.numel()))).values)


def composition(d, eps):
    adj = d <= eps
    cnt = adj.sum(0, dtype=torch.int64)
    return adj, torch.cat([cnt, cnt.sum().reshape(1)])


def raw(x, y, eps, adj=None, ld_adj=None, vd=None, init_vd=1, m=None, n=None, x_ptr=None, y_ptr=None, ldx=None, ldy=None,
        stream=0):
    """the C ABI call; adj / vd are torch tensors (or None), pointers may be offset"""
    L = _lib.lib()
    m = x.shape[0] if m is None else m
    n = y.shape[0] if n is None else n
    k = x.shape[1]
    ws = torch.empty(max(L.b2d_eps_neighbors_l2sq_workspace_bytes(m, n, k), 256), dtype=torch.uint8, device=DEV)
    rc = L.b2d_eps_neighbors_l2sq(stream, None if adj is None else adj.data_ptr(), n if ld_adj is None else ld_adj,
                                  None if vd is None else vd.data_ptr(), 1 if vd is not None and vd.dtype == torch.int64 else 0,
                                  init_vd, x.data_ptr() if x_ptr is None else x_ptr, k if ldx is None else ldx,
                                  y.data_ptr() if y_ptr is None else y_ptr, k if ldy is None else ldy, m, n, k, eps,
                                  ws.data_ptr(), ws.numel())
    _lib.check(rc)
    return ws


SHAPES = [(129, 300), (192, 511), (193, 257), (255, 1000), (1000, 129), (1, 2049)]   # m % 128 in {1, 64, 65, 127}


@pytest.mark.parametrize("k", [1, 3, 32, 96, 128, 129, 200, 320])
@pytest.mark.parametrize("m,n", SHAPES)
def test_equals_composition(m, n, k):
    x, y = blobs(m, n, k, seed=k)
    d = sqeuclidean(x, y)
    eps = eps_at(d, 0.05)
    radj, rvd = composition(d, eps)
    adj, vd = eps_neighbors_l2sq(x, y, eps)
    assert torch.equal(adj, radj)
    assert torch.equal(vd, rvd)
    # the register store path (n % 16 != 0 already takes it; an adj one byte off any alignment forces it): same bytes
    buf = torch.zeros(m * n + 1, dtype=torch.uint8, device=DEV)
    vd2 = torch.empty(n + 1, dtype=torch.int64, device=DEV)
    ws = raw(x, y, eps, adj=buf[1:], vd=vd2)
    torch.cuda.synchronize()
    del ws
    assert torch.equal(buf[1:].view(m, n).bool(), radj) and int(buf[0]) == 0
    assert torch.equal(vd2, rvd)


@pytest.mark.parametrize("k", [16, 128, 200])
def test_tma_and_register_paths_identical(k):
    m, n = 1000, 4096   # n % 16 == 0: the aligned call stores through TMA
    x, y = blobs(m, n, k, seed=5)
    eps = eps_at(sqeuclidean(x, y), 0.02)
    a1, v1 = eps_neighbors_l2sq(x, y, eps)
    buf = torch.zeros(m * n + 1, dtype=torch.uint8, device=DEV)
    v2 = torch.empty(n + 1, dtype=torch.int64, device=DEV)
    raw(x, y, eps, adj=buf[1:], vd=v2)
    torch.cuda.synchronize()
    assert torch.equal(buf[1:].view(m, n).bool(), a1) and torch.equal(v1, v2)


def test_outlier_rows():
    x, y = blobs(300, 700, 40, seed=9)
    x[7] *= 1e6      # rows far above the rest take their own exponent in the operand preparation
    y[11] *= 1e-5
    y[600] *= 3e5
    d = sqeuclidean(x, y)
    eps = eps_at(d, 0.1)
    radj, rvd = composition(d, eps)
    adj, vd = eps_neighbors_l2sq(x, y, eps)
    assert torch.equal(adj, radj) and torch.equal(vd, rvd)


@pytest.mark.parametrize("k", [32, 200])
def test_fp64_outside_band(k):
    x, y = blobs(500, 900, k, seed=21)
    xh, yh = x.cpu().numpy(), y.cpu().numpy()
    eps = float(np.quantile(sqdist64(xh, yh)[0], 0.03))
    radj, rvd, clear = ref_eps(xh, yh, eps)
    adj, vd = eps_neighbors_l2sq(x, y, eps)
    adj, vd = adj.cpu().numpy(), vd.cpu().numpy()
    assert (adj[clear] == radj[clear]).all()
    cols = clear.all(0)   # columns without a pair in the band: exact counts
    assert cols.sum() > 0
    assert (vd[:-1][cols] == rvd[:-1][cols]).all()


@pytest.mark.parametrize("k", [32, 200])           # resident and streaming kernel
@pytest.mark.parametrize("n", [4096, 4100])         # adjacency by TMA and by the copy-out
def test_many_items_per_cta(n, k):
    """m = 40000: 848 work items of 6 x tiles each on 132 SMs, so every CTA flushes the counts of several y blocks,
    accumulates several tiles per item and reuses each staging slot many times"""
    m = 40000
    x, y = blobs(m, n, k, seed=40 + k)
    d = sqeuclidean(x, y)
    eps = eps_at(d, 0.01)
    radj, rvd = composition(d, eps)
    del d
    adj, vd = eps_neighbors_l2sq(x, y, eps)
    assert torch.equal(adj, radj) and torch.equal(vd, rvd)
    _, vc = eps_neighbors_l2sq(x, y, eps, return_adj=False)
    assert torch.equal(vc, rvd)
    for dt in (torch.int32, torch.int64):   # init_vd = 0, twice: the counts add up
        acc = torch.zeros(n + 1, dtype=dt, device=DEV)
        a2 = torch.zeros((m, n), dtype=torch.uint8, device=DEV)
        raw(x, y, eps, adj=a2, vd=acc, init_vd=0)
        raw(x, y, eps, vd=acc, init_vd=0)
        torch.cuda.synchronize()
        assert torch.equal(acc.long(), 2 * rvd) and torch.equal(a2.bool(), radj)


@pytest.mark.parametrize("n_pad", [4096, 1000])
def test_padded_ld_adj_untouched(n_pad):
    m, n, k = 300, n_pad, 24
    x, y = blobs(m, n, k, seed=2)
    eps = eps_at(sqeuclidean(x, y), 0.05)
    radj, rvd = composition(sqeuclidean(x, y), eps)
    ld = n + 32
    buf = torch.full((m, ld), 0xA5, dtype=torch.uint8, device=DEV)
    vd = torch.empty(n + 1, dtype=torch.int64, device=DEV)
    raw(x, y, eps, adj=buf, ld_adj=ld, vd=vd)
    torch.cuda.synchronize()
    assert torch.equal(buf[:, :n].bool(), radj) and torch.equal(vd, rvd)
    assert bool((buf[:, n:] == 0xA5).all())


def test_self_pairs():
    x, _ = blobs(1000, 1, 16, seed=3)
    x = x + 1000.0   # far from the origin: the tensor form of a row against itself is not 0 here
    adj, vd = eps_neighbors_l2sq(x, x, 0.0)
    assert bool(adj.diagonal().all())
    off, n = 130, 500
    ywin = x[off:off + n]   # a view: the same memory
    adj, vd = eps_neighbors_l2sq(x, ywin, 0.0)
    j = torch.arange(n, device=DEV)
    assert bool(adj[j + off, j].all())
    d = sqeuclidean(x, ywin)
    d[j + off, j] = 0.0
    radj, rvd = composition(d, 0.0)
    assert torch.equal(adj, radj) and torch.equal(vd, rvd)
    # negative eps: nothing, self pairs included
    adj, vd = eps_neighbors_l2sq(x, ywin, -1.0)
    assert not bool(adj.any()) and int(vd.sum()) == 0
    # a copy in other memory has no self-pair rule: it is exactly the composition
    yc = ywin.clone()
    adj, vd = eps_neighbors_l2sq(x, yc, 0.0)
    radj, rvd = composition(sqeuclidean(x, yc), 0.0)
    assert torch.equal(adj, radj) and torch.equal(vd, rvd)


def test_count_only_and_modes():
    m, n, k = 777, 1500, 48
    x, y = blobs(m, n, k, seed=4)
    eps = eps_at(sqeuclidean(x, y), 0.05)
    adj, vd = eps_neighbors_l2sq(x, y, eps)
    none, vd_c = eps_neighbors_l2sq(x, y, eps, return_adj=False)
    assert none is None and torch.equal(vd_c, vd)
    v32 = torch.empty(n + 1, dtype=torch.int32, device=DEV)
    _, v32 = eps_neighbors_l2sq(x, y, eps, vd=v32)
    assert v32.dtype == torch.int32 and torch.equal(v32.long(), vd)
    # init_vd = 0 adds: twice gives double, int32 and int64
    for dt in (torch.int32, torch.int64):
        acc = torch.zeros(n + 1, dtype=dt, device=DEV)
        raw(x, y, eps, vd=acc, init_vd=0)
        raw(x, y, eps, vd=acc, init_vd=0)
        torch.cuda.synchronize()
        assert torch.equal(acc.long(), 2 * vd)
    # adjacency only
    a2 = torch.zeros((m, n), dtype=torch.uint8, device=DEV)
    raw(x, y, eps, adj=a2)
    torch.cuda.synchronize()
    assert torch.equal(a2.bool(), adj)
    # two calls: identical bytes
    adj2, vd2 = eps_neighbors_l2sq(x, y, eps)
    assert torch.equal(adj, adj2) and torch.equal(vd, vd2)


def test_nan():
    x, y = blobs(300, 400, 20, seed=6)
    x[5, 3] = float("nan")
    y[17, 0] = float("nan")
    eps = 1e30
    adj, vd = eps_neighbors_l2sq(x, y, eps)
    assert not bool(adj[5].any()) and not bool(adj[:, 17].any())
    radj, rvd = composition(sqeuclidean(x, y), eps)
    assert torch.equal(adj, radj) and torch.equal(vd, rvd)
    for e in (float("nan"), -0.5):
        adj, vd = eps_neighbors_l2sq(x, y, e)
        assert not bool(adj.any()) and int(vd.abs().sum()) == 0


def test_empty():
    x, y = blobs(10, 10, 8)
    adj, vd = eps_neighbors_l2sq(x[:0], y, 1.0)
    assert adj.shape == (0, 10) and torch.equal(vd, torch.zeros(11, dtype=torch.int64, device=DEV))
    adj, vd = eps_neighbors_l2sq(x, y[:0], 1.0)
    assert adj.shape == (10, 0) and torch.equal(vd, torch.zeros(1, dtype=torch.int64, device=DEV))


def test_k_limit():
    x, y = blobs(10, 10, 321)
    with pytest.raises(LogicError, match="320"):
        eps_neighbors_l2sq(x, y, 1.0)


def test_cuda_graph_capture():
    m, n, k = 600, 2048, 64
    x, y = blobs(m, n, k, seed=8)
    eps = eps_at(sqeuclidean(x, y), 0.05)
    radj, rvd = composition(sqeuclidean(x, y), eps)
    L = _lib.lib()
    adj = torch.zeros((m, n), dtype=torch.uint8, device=DEV)
    vd = torch.empty(n + 1, dtype=torch.int64, device=DEV)
    ws = torch.empty(L.b2d_eps_neighbors_l2sq_workspace_bytes(m, n, k), dtype=torch.uint8, device=DEV)
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        _lib.check(L.b2d_eps_neighbors_l2sq(s.cuda_stream, adj.data_ptr(), n, vd.data_ptr(), 1, 1, x.data_ptr(), k,
                                            y.data_ptr(), k, m, n, k, eps, ws.data_ptr(), ws.numel()))
    for _ in range(2):
        adj.zero_()
        vd.fill_(-7)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(adj.bool(), radj) and torch.equal(vd, rvd)
