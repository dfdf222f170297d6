"""DBSCAN on the random ball cover on the GPU: labels, core_sample_indices and n_clusters equal the oracle byte for byte,
the oracle being tests/dbscan_ref.py on A = (tests/ball_cover_ref.dist(x, x) <= fp32(eps)), the contract's pair value
term by term.  Covered: d in {2, 3}, both metrics, m from 1 to 20000, min_samples from 1 to m + 1, the ball cover tests'
adversarial data (a lattice with eps at a lattice distance, duplicates, a 1e4 offset with a 1e-2 spread, 1e-20
coordinates, one dense ball with outliers), every eps edge, independence from n_landmarks and the seed, a pitched x,
repeated runs and a CUDA-graph replay, agreement with the brute fit where both forms are exact, 10^6 rows against the
edge list of ball_cover.eps_nn, and the C++ shim against the Python call."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import ball_cover_ref as bref
import cpp_build
from dbscan_ref import dbscan_ref, dbscan_ref_edges

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
pytest.importorskip("scipy.sparse.csgraph")

from raft_b200 import _lib  # noqa: E402

METRICS = ["sqeuclidean", "euclidean"]
METRIC_IDS = {"sqeuclidean": 4, "euclidean": 5}


def cuda(a):
    return torch.as_tensor(np.ascontiguousarray(a, np.float32)).cuda()


def points(m, d, seed, kind="blobs"):
    r = np.random.default_rng(seed)
    if kind == "uniform":
        return r.random((m, d), dtype=np.float32)
    centers = r.random((max(1, m // 200), d)) * 10
    x = centers[r.integers(0, len(centers), m)] + r.normal(0, 0.3, (m, d))
    noise = r.random(m) < 0.1
    x[noise] = r.random((int(noise.sum()), d)) * 10
    return x.astype(np.float32)


def oracle(x, eps, min_samples, metric, block=4096):
    """dbscan_ref on A = dist(x, x) <= fp32(eps), formed on the device: the dense reference for small m, the edge-list
    one (the same rules, tests/test_dbscan.py) for large m or dense A"""
    m = x.shape[0]
    e = float(np.float32(eps)) if eps == eps else float("nan")
    if m <= 1000:
        A = (bref.dist(x, x, metric) <= e).cpu().numpy()
        return dbscan_ref(A, min_samples)
    rows, cols = [], []
    for r0 in range(0, m, block):
        nz = torch.nonzero(bref.dist(x[r0:r0 + block], x, metric) <= e)
        rows.append((nz[:, 0] + r0).cpu().numpy())
        cols.append(nz[:, 1].cpu().numpy())
    return dbscan_ref_edges(np.concatenate(rows), np.concatenate(cols), m, min_samples)


def run(x, eps, min_samples, metric, **kw):
    from raft_b200.cluster import dbscan
    o = dbscan(x, eps, min_samples=min_samples, metric=metric, algorithm="rbc", **kw)
    torch.cuda.synchronize()
    return o.labels.cpu().numpy(), o.core_sample_indices.cpu().numpy(), o.n_clusters


def check(got, want):
    lab, csi, nc = got
    wl, wc, wn = want
    assert lab.tobytes() == wl.tobytes(), (lab[:20], wl[:20])
    n = int((wc >= 0).sum())
    assert csi.tobytes() == wc[:n].tobytes()
    assert nc == wn


def eps_for(x, metric, neighbours):
    """an eps giving about `neighbours` rows within it per row (from a sample of rows)"""
    m = x.shape[0]
    if m < 2:
        return 1.0
    rows = max(64, min(512, (1 << 26) // m))
    sel = x[torch.randperm(m, device=x.device, generator=torch.Generator("cuda").manual_seed(m))[:rows]]
    dd = bref.dist(sel, x, metric)
    k = min(m - 1, neighbours)
    return float(torch.kthvalue(dd, k + 1, dim=1).values.median())


def raw_fit(xp, ldx, m, d, eps, min_samples, metric, nl=0, seed=0, stream=None):
    """b2d_dbscan_rbc_fit on a device pointer with pitch ldx; returns (labels, core_sample_indices [m], n_clusters)"""
    L = _lib.lib()
    lab = torch.full((m,), -7, dtype=torch.int32, device="cuda")
    csi = torch.full((m,), -7, dtype=torch.int32, device="cuda")
    ncl = torch.full((1,), -7, dtype=torch.int32, device="cuda")
    ws = torch.empty(L.b2d_dbscan_rbc_workspace_bytes(m, d, nl), dtype=torch.uint8, device="cuda")
    _lib.check(L.b2d_dbscan_rbc_fit(stream, METRIC_IDS[metric], xp, ldx, m, d, float(eps), min_samples, nl, seed,
                                    lab.data_ptr(), csi.data_ptr(), ncl.data_ptr(), ws.data_ptr(), ws.numel()))
    torch.cuda.synchronize()
    return lab.cpu().numpy(), csi.cpu().numpy(), int(ncl.item())


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("d", [2, 3])
@pytest.mark.parametrize("m", [1, 2, 63, 1000, 20000])
def test_shapes_and_min_samples(m, d, metric):
    x = cuda(points(m, d, m + d, "blobs" if m % 2 == 0 else "uniform"))
    eps = eps_for(x, metric, 12)
    mixed = False
    for ms in (1, 2, 5, 20, m + 1):
        got = run(x, eps, ms, metric)
        check(got, oracle(x, eps, ms, metric))
        mixed |= bool((got[0] >= 0).any() and (got[0] == -1).any())
    assert m < 1000 or mixed


def adversarial(kind, d):
    """the ball cover tests' data (tests/test_ball_cover_gpu.py)"""
    r = np.random.default_rng(5)
    if kind == "lattice":
        g = np.stack(np.meshgrid(*[np.arange(14 if d == 3 else 50)] * d, indexing="ij"), -1).reshape(-1, d)
        return g.astype(np.float32)
    if kind == "duplicates":
        base = r.random((37, d)).astype(np.float32)
        return base[r.integers(0, 37, 5000)]
    if kind == "cancellation":
        return (1e4 + 1e-2 * r.random((5000, d))).astype(np.float32)
    if kind == "subnormal":
        return (1e-20 * r.random((5000, d))).astype(np.float32)
    if kind == "dense_ball":
        dense = 1e-3 * r.random((20000, d))
        out = 1e3 * r.random((50, d))
        return np.concatenate([dense, out]).astype(np.float32)
    raise ValueError(kind)


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("d", [2, 3])
@pytest.mark.parametrize("kind", ["lattice", "duplicates", "cancellation", "subnormal", "dense_ball"])
def test_adversarial(kind, d, metric):
    x = cuda(adversarial(kind, d))
    if kind == "lattice":   # eps exactly at a lattice distance: every axis neighbour (and the diagonal one) on it
        eps_list = [1.0, 2.0] if metric == "sqeuclidean" else [1.0, float(torch.sqrt(torch.tensor(2.0)))]
    elif kind == "duplicates":
        eps_list = [0.0, eps_for(x, metric, 400)]
    else:
        eps_list = [eps_for(x, metric, 8), eps_for(x, metric, 40)]
    for eps in eps_list:
        for ms in (1, 5, 20):
            for nl in (None, 1):
                check(run(x, eps, ms, metric, n_landmarks=nl, seed=nl or 0), oracle(x, eps, ms, metric))


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("d", [2, 3])
def test_eps_edges(d, metric):
    x = cuda(points(1500, d, 31))
    dd = bref.dist(x, x, metric)
    smallest = float(dd[dd > 0].min())
    below = float(np.nextafter(np.float32(smallest), np.float32(0)))
    diameter = float(dd.max())
    for eps in (0.0, smallest, below, diameter * 1.01, float("inf"), float("nan"), -1.0):
        for ms in (1, 2, 5):
            got = run(x, eps, ms, metric)
            check(got, oracle(x, eps, ms, metric))
            if not eps >= 0:   # every row noise
                assert (got[0] == -1).all() and got[1].size == 0 and got[2] == 0
            if eps == float("inf"):   # every pair linked
                assert (got[0] == 0).all() and got[2] == 1


def test_independent_of_landmarks_and_seed():
    m, d = 20000, 2
    x = cuda(points(m, d, 21))
    eps = eps_for(x, "euclidean", 15)
    want = oracle(x, eps, 10, "euclidean")
    outs = []
    for nl in (1, 2, int(np.ceil(np.sqrt(m))), m):
        for seed in (0, 1, 12345678901):
            outs.append(run(x, eps, 10, "euclidean", n_landmarks=nl, seed=seed))
    for o in outs:
        check(o, want)
    assert want[2] > 1


def test_pitched_input_through_the_c_abi():
    m, d = 4000, 3
    wide = cuda(points(m, 6, 4))
    x = wide[:, 1:1 + d].contiguous()
    for metric in METRICS:
        eps = eps_for(x, metric, 10)
        got = raw_fit(wide.data_ptr() + 4, 6, m, d, eps, 5, metric, nl=17, seed=3)
        check((got[0], got[1][got[1] >= 0], got[2]), oracle(x, eps, 5, metric))
        assert (got[1][(got[1] >= 0).sum():] == -1).all()


def test_repeat_and_cuda_graph_replay():
    m, d = 20000, 3
    x = cuda(points(m, d, 41))
    eps = eps_for(x, "euclidean", 20)
    want = raw_fit(x.data_ptr(), d, m, d, eps, 8, "euclidean")
    again = raw_fit(x.data_ptr(), d, m, d, eps, 8, "euclidean")
    assert all(np.asarray(a).tobytes() == np.asarray(b).tobytes() for a, b in zip(want, again))
    L = _lib.lib()
    lab = torch.full((m,), -7, dtype=torch.int32, device="cuda")
    csi = torch.full((m,), -7, dtype=torch.int32, device="cuda")
    ncl = torch.full((1,), -7, dtype=torch.int32, device="cuda")
    ws = torch.empty(L.b2d_dbscan_rbc_workspace_bytes(m, d, 0), dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(g, stream=s):
        _lib.check(L.b2d_dbscan_rbc_fit(ctypes.c_void_p(s.cuda_stream), 5, x.data_ptr(), d, m, d, float(eps), 8, 0, 0,
                                        lab.data_ptr(), csi.data_ptr(), ncl.data_ptr(), ws.data_ptr(), ws.numel()))
    for _ in range(2):
        lab.fill_(-7)
        csi.fill_(-7)
        ncl.fill_(-7)
        g.replay()
        torch.cuda.synchronize()
        assert lab.cpu().numpy().tobytes() == want[0].tobytes() and csi.cpu().numpy().tobytes() == want[1].tobytes()
        assert int(ncl.item()) == want[2]


@pytest.mark.parametrize("d", [2, 3])
def test_agrees_with_brute_fit_on_small_integers(d):
    # integer coordinates below 64: the squared distances are small integers, exact in both the expanded and the
    # unexpanded form, and eps sits between them
    from raft_b200.cluster import dbscan
    r = np.random.default_rng(50 + d)
    x = cuda(r.integers(0, 64 if d == 2 else 16, (6000, d)))
    for metric, eps in (("sqeuclidean", 2.5), ("sqeuclidean", 8.5), ("euclidean", 1.5), ("euclidean", 2.9)):
        for ms in (2, 6):
            a = dbscan(x, eps, min_samples=ms, metric=metric, algorithm="rbc")
            b = dbscan(x, eps, min_samples=ms, metric=metric, algorithm="brute")
            assert torch.equal(a.labels, b.labels) and torch.equal(a.core_sample_indices, b.core_sample_indices)
            assert a.n_clusters == b.n_clusters


@pytest.mark.parametrize("d,kind,metric", [(2, "uniform", "euclidean"), (3, "blobs", "sqeuclidean")])
def test_million_points_against_eps_nn_edges(d, kind, metric):
    from raft_b200.neighbors import ball_cover
    m = 1000000
    if kind == "uniform":
        x = torch.rand((m, d), generator=torch.Generator("cuda").manual_seed(7), device="cuda")
    else:
        x = cuda(points(m, d, 8))
    eps = eps_for(x, metric, 30)
    index = ball_cover.build_index(x, metric=metric)
    indptr, indices, _ = ball_cover.eps_nn(index, x, eps)
    rows = torch.repeat_interleave(torch.arange(m, device="cuda"), indptr[1:] - indptr[:-1]).cpu().numpy()
    cols = indices.cpu().numpy()
    del indices
    for ms in (10, 40):
        want = dbscan_ref_edges(rows, cols, m, ms)
        got = run(x, eps, ms, metric)
        check(got, want)
        assert want[2] >= 1 and (got[0] >= 0).any()


def test_empty_single_row_and_non_finite():
    from raft_b200.cluster import dbscan
    o = dbscan(torch.empty((0, 2), device="cuda"), 1.0, algorithm="rbc")
    assert o.labels.numel() == 0 and o.core_sample_indices.numel() == 0 and o.n_clusters == 0
    o = dbscan(torch.zeros((1, 3), device="cuda"), 1.0, min_samples=1, algorithm="rbc")
    assert o.labels.tolist() == [0] and o.core_sample_indices.tolist() == [0] and o.n_clusters == 1
    with pytest.raises(ValueError):
        dbscan(torch.full((3, 2), float("nan"), device="cuda"), 1.0, algorithm="rbc")


@pytest.mark.parametrize("mock_raft", [False, True])
def test_shim_runs_on_gpu_and_matches_python(tmp_path, mock_raft):
    from raft_b200.cluster import dbscan
    exe = cpp_build.build("dbscan_rbc_shim_test.cu", str(tmp_path / "shim"), mock_raft)
    m, d, ms, nl = 5000, 2, 10, 40
    xn = points(m, d, 8)
    x = cuda(xn)
    eps = np.float32(eps_for(x, "euclidean", 15))
    inp, out = os.path.join(tmp_path, "in.bin"), os.path.join(tmp_path, "out.bin")
    with open(inp, "wb") as f:
        f.write(np.array([m, d, ms, nl], np.int64).tobytes() + eps.tobytes() + xn.tobytes())
    res = subprocess.run([exe, inp, out], capture_output=True, text=True, timeout=120)
    assert res.returncode == 0 and "PASS" in res.stdout, res.stdout + res.stderr
    raw = np.fromfile(out, np.int32)
    o = dbscan(x, float(eps), min_samples=ms, algorithm="rbc")
    lab = o.labels.cpu().numpy()
    assert raw[:m].tobytes() == lab.tobytes()
    n = o.core_sample_indices.numel()
    assert raw[m:m + n].tobytes() == o.core_sample_indices.cpu().numpy().tobytes() and (raw[m + n:2 * m] == -1).all()
    assert o.n_clusters > 1 and (lab == -1).any()
    brute = dbscan(x, float(eps), min_samples=ms, algorithm="brute")
    assert raw[2 * m:].tobytes() == brute.labels.cpu().numpy().tobytes()
