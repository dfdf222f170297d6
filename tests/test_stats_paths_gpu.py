"""GPU tier: silhouette_score and trustworthiness_score on every slab, label and neighbour path, against fp64.

Exact cases use small-integer coordinates in both spaces: the operands are fp16-exact and every squared distance is an
integer below 2^24, so the tensor path computes it exactly, the fused kNN and the rank count break ties by index, and
trustworthiness must equal the fp64 oracle to 1e-12.  Silhouette sums floats atomically in shared memory; it is held
to the bars of test_stats_gpu.py (score 2e-4, per sample 5e-4).  Cases that Python cannot reach (padded leading
dimensions, NaN per sample, CUDA-graph capture, error statuses) go through the C ABI."""
import ctypes

import numpy as np
import pytest
import torch

import oracle
from oracle import DistanceType as DT
from raft_b200 import LogicError, _lib
from raft_b200.stats import silhouette_score, trustworthiness_score

pytestmark = pytest.mark.gpu
DEV = "cuda"
SCORE_TOL, SAMPLE_TOL = 2e-4, 5e-4
NO_WS = 2 ** 64 - 1


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def sil_reference(x, labels, n_labels, metric=DT.L2Unexpanded, p=2.0, rows=None):
    """fp64 per-sample silhouette of `rows` (default: every row) by oracle.silhouette_score's definition, blocked over
    rows so that no n x n matrix is formed: per-cluster sums of a row are segment sums of its distances with the
    columns grouped by label.  d(i, i) is 0 by definition, as in sil_row_kernel: that matters where the metric does not
    give 0 (inner product, Russell-Rao) or gives 0 only up to rounding (Hellinger)."""
    x64 = np.asarray(x, dtype=np.float64)
    labels = np.asarray(labels, dtype=np.int64)
    n = len(labels)
    rows = np.arange(n) if rows is None else np.asarray(rows)
    counts = np.bincount(labels, minlength=n_labels)
    cnt = counts.astype(np.float64)
    present = np.flatnonzero(counts)
    perm = np.argsort(labels, kind="stable")
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]])[present]
    block = max(1, min(256, (1 << 24) // n))
    out = np.empty(len(rows))
    for r0 in range(0, len(rows), block):
        rr = rows[r0:r0 + block]
        at = np.arange(len(rr))
        d = oracle.pairwise_distance(x64[rr], x64, metric, p)
        d[at, rr] = 0.0                                      # d(i, i) = 0 by definition
        sums = np.zeros((len(rr), n_labels))
        sums[:, present] = np.add.reduceat(d[:, perm], starts, axis=1)
        own = labels[rr]
        a = np.where(counts[own] > 1, sums[at, own] / np.maximum(cnt[own] - 1, 1), -1.0)
        with np.errstate(divide="ignore", invalid="ignore"):
            mean = np.where(counts > 0, sums / np.maximum(cnt, 1), np.inf)
            mean[at, own] = np.inf
            b = mean.min(axis=1)
            s = np.where((a == -1.0) | (a == b), 0.0,
                         np.where(a > b, (b - a) / np.where(a == 0, 1, a), (b - a) / np.where(b == 0, 1, b)))
        out[r0:r0 + len(rr)] = s
    return out


def sil_abi(x, labels, n_labels, metric=DT.L2Unexpanded, p=2.0, chunk=0, ldx=None, k=None, stream=None, ws=None,
            score=None, per=None):
    """b2d_silhouette_score through ctypes on device tensors; returns (status, score [1], per-sample [n])."""
    L = _lib.lib()
    n = labels.shape[0]
    k = x.shape[1] if k is None else k
    ldx = x.stride(0) if ldx is None else ldx
    if ws is None:
        need = L.b2d_silhouette_score_workspace_bytes(n, k, n_labels, int(metric), chunk)
        ws = torch.empty(256 if need == NO_WS else max(need, 256), dtype=torch.uint8, device=DEV)
    score = torch.full((1,), -7.0, device=DEV) if score is None else score
    per = torch.full((n,), -7.0, device=DEV) if per is None else per
    rc = L.b2d_silhouette_score(ctypes.c_void_p(stream), score.data_ptr(), per.data_ptr(), x.data_ptr(), ldx,
                                labels.data_ptr(), n, k, int(n_labels), int(metric), float(p), int(chunk), ws.data_ptr(),
                                ws.numel())
    return rc, score, per


def trust_abi(x, e, n_neighbors, metric=DT.L2Expanded, batch=0, ldx=None, lde=None, m=None, d=None, stream=None,
              ws=None, out=None):
    """b2d_trustworthiness_score through ctypes on device tensors; returns (status, score [1] float64)."""
    L = _lib.lib()
    n = x.shape[0]
    m = x.shape[1] if m is None else m
    d = e.shape[1] if d is None else d
    ldx = x.stride(0) if ldx is None else ldx
    lde = e.stride(0) if lde is None else lde
    if ws is None:
        need = L.b2d_trustworthiness_score_workspace_bytes(n, m, d, n_neighbors, int(metric), batch)
        ws = torch.empty(256 if need == NO_WS else max(need, 256), dtype=torch.uint8, device=DEV)
    out = torch.full((1,), -7.0, dtype=torch.float64, device=DEV) if out is None else out
    rc = L.b2d_trustworthiness_score(ctypes.c_void_p(stream), out.data_ptr(), x.data_ptr(), ldx, e.data_ptr(), lde, n,
                                     m, d, int(n_neighbors), int(metric), int(batch), ws.data_ptr(), ws.numel())
    return rc, out


def int_data(n, m, d, x_dups, e_groups, seed):
    """Integer coordinates in [-16, 16]: X [n, m], embedding [n, d].  x_dups: groups of identical rows in X;
    e_groups: coincident groups in the embedding, up to 220 points (more than n_neighbors + 1 for every n_neighbors)."""
    rng = np.random.default_rng(seed)
    x = rng.integers(-16, 17, (n, m)).astype(np.float32)
    e = rng.integers(-16, 17, (n, d)).astype(np.float32)
    if x_dups:
        for g in np.split(rng.permutation(n)[:300], [3, 6, 46, 86, 126]):
            x[g] = x[g[0]]
    if e_groups:
        for g in np.split(rng.permutation(n)[:min(n, 400)], [2, 7, 40, 110, 180]):
            if len(g):
                e[g] = e[g[0]]
    return x, e


# ---------------------------------------------------------------------------------------------------------------
# trustworthiness: exact cases


@pytest.mark.parametrize("n_neighbors", [1, 31, 32, 33, 62, 63])
@pytest.mark.parametrize("dups", ["x", "emb", "both"])
def test_trustworthiness_exact_with_ties(dups, n_neighbors):
    """Duplicate rows in X, coincident groups in the embedding, and both: ties in either space are broken by index in
    the kNN and in the rank count, so the score is the oracle's to 1e-12.  n_neighbors 31 / 32 / 33 / 62 / 63 cover
    both halves of the rank counters (neighbour q < 32 and q >= 32).  A sample with n_neighbors + 1 or more coincident
    mates of smaller index is missing from its own kNN list: it still counts exactly n_neighbors neighbours."""
    x, e = int_data(700, 24, 3, dups in ("x", "both"), dups in ("emb", "both"), seed=n_neighbors)
    ref = oracle.trustworthiness_score(x, e, n_neighbors, metric=DT.L2Expanded)
    xt, et = dev(x), dev(e)
    for metric in ("sqeuclidean", "sqeuclidean_unexpanded"):
        got = trustworthiness_score(xt, et, n_neighbors=n_neighbors, metric=metric)
        assert got == pytest.approx(ref, abs=1e-12), (metric, got, ref)


@pytest.mark.parametrize("n", [129, 1025, 1027, 1100])
def test_trustworthiness_slab_plans_are_exact_and_identical(n):
    """Slabs of 128 rows (the last one holds 1 or 3 rows for n = 129 / 1025 / 1027), n - 1 rows (rounded down to a
    multiple of 128) and the default; ld = n rounded up to 4 is padded for n = 129 / 1025 / 1027.  The penalty is an
    integer atomic: every plan and every repeat gives the same score, the oracle's to 1e-12."""
    x, e = int_data(n, 20, 2, True, True, seed=n)
    xt, et = dev(x), dev(e)
    for k in (5, 40):
        ref = oracle.trustworthiness_score(x, e, k, metric=DT.L2Expanded)
        got = [trustworthiness_score(xt, et, n_neighbors=k, metric="sqeuclidean", batch_size=b)
               for b in (128, n - 1, 0, 128)]
        assert got == [got[0]] * 4, (k, got)
        assert got[0] == pytest.approx(ref, abs=1e-12), (k, got[0], ref)


@pytest.mark.parametrize("k", [1, 2, 32, 63])
def test_trustworthiness_of_the_identity_with_tied_neighbours(k):
    """Points on a line: every inner sample has two neighbours at each distance, and the embedding is X itself (then
    X shifted).  One tie rule in both spaces keeps every embedded neighbour inside the original-space top k: 1 exactly.
    Pairs of coincident points (x // 2): a sample never lacks itself from a list of k + 1, the score is the oracle's."""
    x = np.arange(200, dtype=np.float32)[:, None]
    for e in (x, x + 5.0):
        assert trustworthiness_score(dev(x), dev(e), n_neighbors=k, metric="sqeuclidean") == 1.0
    e = np.floor(x / 2)
    got = trustworthiness_score(dev(x), dev(e), n_neighbors=k, metric="sqeuclidean_unexpanded", batch_size=128)
    assert got == pytest.approx(oracle.trustworthiness_score(x, e, k, metric=DT.L2Expanded), abs=1e-12)


# ---------------------------------------------------------------------------------------------------------------
# trustworthiness: metrics


@pytest.mark.parametrize("metric,dt", [("euclidean", DT.L2SqrtExpanded), ("sqeuclidean", DT.L2Expanded),
                                       ("l2_unexpanded", DT.L2SqrtUnexpanded),
                                       ("sqeuclidean_unexpanded", DT.L2Unexpanded),
                                       ("cosine", DT.CosineExpanded), ("correlation", DT.CorrelationExpanded)])
@pytest.mark.parametrize("k", [1, 7, 45])
def test_trustworthiness_metrics(metric, dt, k):
    """Every metric of the L2 and cosine families on float data; the cosine rows have norms spanning 10^4, so an L2
    neighbourhood would differ from the cosine one."""
    rng = np.random.default_rng(100 + k)
    n, m, d = 1500, 40, 5
    x = rng.standard_normal((n, m)).astype(np.float32)
    if dt == DT.CosineExpanded:
        x *= (10.0 ** rng.uniform(-2, 2, (n, 1))).astype(np.float32)
    e = (x @ rng.standard_normal((m, d)).astype(np.float32) + 0.3 * rng.standard_normal((n, d))).astype(np.float32)
    ref = oracle.trustworthiness_score(x, e, k, metric=dt)
    got = trustworthiness_score(dev(x), dev(e), n_neighbors=k, metric=metric, batch_size=384)
    assert abs(got - ref) < 1e-4, (got, ref)


# ---------------------------------------------------------------------------------------------------------------
# silhouette: metrics, slab plans, labels


def family_data(metric, n, k, n_labels, seed):
    """The data families of test_distribution_and_boolean_metrics: probability rows for KL / JS / Hellinger, 0/1 rows for
    the boolean metrics, counts for Bray-Curtis; separated normal blobs (positive ones for the inner product)."""
    rng = np.random.default_rng(seed)
    labels = rng.integers(0, n_labels, n).astype(np.int32)
    labels[:n_labels] = np.arange(n_labels)
    if metric in (DT.KLDivergence, DT.JensenShannon, DT.HellingerExpanded):
        x = rng.random((n, k)) + 0.5 * (labels[:, None] == np.arange(k)[None, :] % n_labels)
        x /= x.sum(1, keepdims=True)
    elif metric in (DT.HammingUnexpanded, DT.RusselRaoExpanded, DT.JaccardExpanded, DT.DiceExpanded):
        x = rng.random((n, k)) < 0.3 + 0.4 * (labels[:, None] == np.arange(k)[None, :] % n_labels)
    elif metric == DT.BrayCurtis:
        x = rng.random((n, k)) * 9 + 3 * labels[:, None]
    elif metric == DT.InnerProduct:
        x = rng.uniform(0.5, 1.5, (n, k)) + 0.3 * labels[:, None]
    else:
        x = rng.standard_normal((n, k)) + 1.5 * labels[:, None]
    return x.astype(np.float32), labels


SIL_METRICS = [DT.L2Expanded, DT.L2SqrtExpanded, DT.CosineExpanded, DT.CorrelationExpanded, DT.InnerProduct,
               DT.HellingerExpanded, DT.RusselRaoExpanded, DT.JaccardExpanded, DT.DiceExpanded, DT.L1, DT.L2Unexpanded,
               DT.L2SqrtUnexpanded, DT.Linf, DT.Canberra, DT.LpUnexpanded, DT.HammingUnexpanded, DT.KLDivergence,
               DT.JensenShannon, DT.BrayCurtis]


@pytest.mark.parametrize("k", [1, 3, 321, 784])
@pytest.mark.parametrize("metric", SIL_METRICS, ids=[m.name for m in SIL_METRICS])
def test_silhouette_every_metric(metric, k):
    """Every fp32 metric of pairwise_distance (p = 3 for Lp); k = 321 / 784 take the K-chunked tensor path, k = 1 / 3
    the unvectorised loads.  Not run at k = 1: correlation (undefined for one feature, 0 / 0) and cosine (every
    distance is 0 or 2, so on most rows a and b are both 0 up to rounding and (b - a) / max(a, b) is rounding noise)."""
    if metric in (DT.CorrelationExpanded, DT.CosineExpanded) and k == 1:
        pytest.skip("ill-posed for one feature")
    x, labels = family_data(metric, 400, k, 4, seed=k)
    ref = sil_reference(x, labels, 4, metric, 3.0)
    got, per = silhouette_score(dev(x), dev(labels), 4, metric=int(metric), p=3.0, return_samples=True)
    assert abs(got - ref.mean()) < SCORE_TOL, (got, ref.mean())
    err = np.abs(per.cpu().numpy() - ref)
    assert err.max() < SAMPLE_TOL, (err.max(), int(err.argmax()))


@pytest.mark.parametrize("n", [129, 1025, 1027, 1100])
def test_silhouette_slab_plans(n):
    """Slabs of 128 rows (the last one holds 1 or 3 rows), n - 1 rows and the default, over a padded ld."""
    x, labels = family_data(DT.L2Unexpanded, n, 13, 3, seed=n)
    ref = sil_reference(x, labels, 3)
    xt, lt = dev(x), dev(labels)
    for chunk in (128, n - 1, 0):
        got, per = silhouette_score(xt, lt, 3, chunk=chunk, return_samples=True)
        assert abs(got - ref.mean()) < SCORE_TOL, (chunk, got, ref.mean())
        assert np.abs(per.cpu().numpy() - ref).max() < SAMPLE_TOL, chunk


@pytest.mark.parametrize("n,n_labels", [(3000, 2), (3000, 300), (13000, 12000)])
def test_silhouette_label_counts(n, n_labels):
    """2, 300 and 12000 labels: the last fills 48000 bytes of shared memory with per-cluster sums.  12001 labels are
    rejected with UNSUPPORTED."""
    rng = np.random.default_rng(n_labels)
    labels = np.concatenate([np.arange(n_labels), rng.integers(0, n_labels, n - n_labels)]).astype(np.int32)
    labels = labels[rng.permutation(n)]
    centres = rng.standard_normal((n_labels, 8)) * 3
    x = (centres[labels] + rng.standard_normal((n, 8))).astype(np.float32)
    ref = sil_reference(x, labels, n_labels)
    xt, lt = dev(x), dev(labels)
    got, per = silhouette_score(xt, lt, n_labels, return_samples=True)
    assert abs(got - ref.mean()) < SCORE_TOL, (got, ref.mean())
    assert np.abs(per.cpu().numpy() - ref).max() < SAMPLE_TOL
    if n_labels == 12000:
        rc, _, _ = sil_abi(xt, lt, 12001)
        assert rc == _lib.B2D_ERR_UNSUPPORTED
        with pytest.raises(LogicError):
            silhouette_score(xt, lt, 12001)


def test_silhouette_mostly_unused_label_ids_and_an_identical_cluster():
    """Four label ids used out of 1500; cluster 700 is one point repeated, so its rows score exactly 1 (a = 0)."""
    rng = np.random.default_rng(5)
    n = 2000
    pick = rng.integers(0, 4, n)
    labels = np.array([0, 17, 700, 1499])[pick].astype(np.int32)
    x = rng.integers(-16, 17, (n, 10)).astype(np.float32) + 2.0 * pick[:, None].astype(np.float32)
    x[labels == 700] = x[np.flatnonzero(labels == 700)[0]]
    xt, lt = dev(x), dev(labels)
    for metric, dt in (("sqeuclidean_unexpanded", DT.L2Unexpanded), ("sqeuclidean", DT.L2Expanded),
                       ("euclidean", DT.L2SqrtExpanded)):
        ref = sil_reference(x, labels, 1500, dt)
        got, per = silhouette_score(xt, lt, 1500, metric=metric, return_samples=True)
        per = per.cpu().numpy()
        assert abs(got - ref.mean()) < SCORE_TOL, (metric, got, ref.mean())
        assert np.abs(per - ref).max() < SAMPLE_TOL, metric
        assert (per[labels == 700] == 1.0).all() and (ref[labels == 700] == 1.0).all(), metric
    assert silhouette_score(xt, lt) == pytest.approx(silhouette_score(xt, lt, 1500), abs=1e-6)   # n_labels inferred


def test_silhouette_giant_cluster_next_to_singletons():
    """n = 200000: one cluster of 190000 rows, one of 8000 and 2000 singletons -- many slabs and fp32 segment sums over
    190000 columns.  About 1000 sampled rows against the blocked fp64 reference; the score is the mean of the
    per-sample values."""
    rng = np.random.default_rng(200000)
    n, k = 200000, 16
    labels = np.zeros(n, dtype=np.int32)
    labels[190000:198000] = 1
    labels[198000:] = np.arange(2, 2002)
    labels = labels[rng.permutation(n)]
    x = (rng.standard_normal((n, k)) + 2.0 * (labels == 1)[:, None]).astype(np.float32)
    got, per = silhouette_score(dev(x), dev(labels), 2002, return_samples=True)
    per = per.cpu().numpy().astype(np.float64)
    rows = np.concatenate([rng.choice(n, 990, replace=False), np.flatnonzero(labels == 1)[:5],
                           np.flatnonzero(labels >= 2)[:5]])
    ref = sil_reference(x, labels, 2002, rows=rows)
    err = np.abs(per[rows] - ref)
    assert err.max() < SAMPLE_TOL, (err.max(), int(rows[err.argmax()]))
    assert (per[labels >= 2] == 0.0).all()                      # singletons score 0
    assert abs(got - per.mean()) < 1e-5, (got, per.mean())


def test_silhouette_one_non_empty_cluster_is_nan():
    """Fewer than two non-empty clusters: every b would be FLT_MAX and s ~ 1.  The C ABI returns NaN, Python raises,
    whether n_labels is declared or inferred."""
    rng = np.random.default_rng(3)
    x = dev(rng.standard_normal((300, 6)).astype(np.float32))
    zeros = torch.zeros(300, dtype=torch.int32, device=DEV)
    rc, score, _ = sil_abi(x, zeros, 3)
    torch.cuda.synchronize()
    assert rc == _lib.B2D_OK and torch.isnan(score).all()
    with pytest.raises(LogicError, match="non-empty"):
        silhouette_score(x, zeros, 3)
    with pytest.raises(LogicError, match="non-empty"):
        silhouette_score(x, zeros + 2)                          # n_labels inferred as 3
    two = zeros.clone()
    two[7] = 2                                                  # two non-empty clusters: defined again
    got = silhouette_score(x, two, 3)
    ref = sil_reference(x.cpu().numpy(), two.cpu().numpy(), 3)
    assert abs(got - ref.mean()) < SCORE_TOL


# ---------------------------------------------------------------------------------------------------------------
# C ABI


def test_padded_leading_dimensions():
    """ldx / lde larger than the row length: the same results as the packed inputs."""
    x, e = int_data(1027, 20, 3, True, True, seed=77)
    xp = torch.zeros((1027, 27), device=DEV)
    ep = torch.zeros((1027, 5), device=DEV)
    xp[:, :20] = dev(x)
    ep[:, :3] = dev(e)
    for k in (1, 33):
        ref = oracle.trustworthiness_score(x, e, k, metric=DT.L2Expanded)
        for metric in (DT.L2Expanded, DT.L2Unexpanded):
            rc, out = trust_abi(xp, ep, k, metric, batch=128, m=20, d=3)
            assert rc == _lib.B2D_OK, _lib.lib().b2d_last_error()
            torch.cuda.synchronize()
            assert out.item() == pytest.approx(ref, abs=1e-12), (k, metric)
    labels = (np.arange(1027) % 5).astype(np.int32)
    lt = dev(labels)
    ref = sil_reference(x, labels, 5)
    for metric in (DT.L2Unexpanded, DT.L2Expanded, DT.L1):
        want = sil_reference(x, labels, 5, metric) if metric != DT.L2Unexpanded else ref
        rc, score, per = sil_abi(xp, lt, 5, metric, chunk=128, k=20)
        assert rc == _lib.B2D_OK, _lib.lib().b2d_last_error()
        torch.cuda.synchronize()
        assert abs(score.item() - want.mean()) < SCORE_TOL, metric
        assert np.abs(per.cpu().numpy() - want).max() < SAMPLE_TOL, metric


def test_invalid_labels_poison_exactly_their_rows():
    """Labels outside [0, n_labels) make the score NaN and the per-sample values of exactly those rows NaN; the other
    rows are scored over the valid rows alone."""
    x, labels = family_data(DT.L2Unexpanded, 1000, 12, 4, seed=9)
    bad = np.array([3, 400, 401, 999])
    labels[bad] = [-1, 4, 1000, -7]
    rc, score, per = sil_abi(dev(x), dev(labels), 4, chunk=256)
    assert rc == _lib.B2D_OK
    torch.cuda.synchronize()
    per = per.cpu().numpy()
    assert np.isnan(score.item())
    assert (np.flatnonzero(np.isnan(per)) == bad).all()
    ok = np.setdiff1d(np.arange(1000), bad)
    ref = sil_reference(x[ok], labels[ok], 4)
    assert np.abs(per[ok] - ref).max() < SAMPLE_TOL
    with pytest.raises(LogicError, match="n_labels"):
        silhouette_score(dev(x), dev(labels), 4)


def test_both_calls_replay_in_a_cuda_graph():
    """Captured in a CUDA graph with preallocated buffers and replayed: the calls enqueue work and never synchronise
    the host.  Trustworthiness equals the direct call exactly, silhouette within tolerance."""
    L = _lib.lib()
    x, e = int_data(1025, 24, 3, True, True, seed=31)
    labels = (np.arange(1025) % 7).astype(np.int32)
    xt, et, lt = dev(x), dev(e), dev(labels)
    k, n = 33, 1025
    tws = torch.empty(L.b2d_trustworthiness_score_workspace_bytes(n, 24, 3, k, int(DT.L2Expanded), 256),
                      dtype=torch.uint8, device=DEV)
    sws = torch.empty(L.b2d_silhouette_score_workspace_bytes(n, 24, 7, int(DT.L2Unexpanded), 256), dtype=torch.uint8,
                      device=DEV)
    tout = torch.empty(1, dtype=torch.float64, device=DEV)
    sout, sper = torch.empty(1, device=DEV), torch.empty(n, device=DEV)

    def calls(stream):
        rc, _ = trust_abi(xt, et, k, DT.L2Expanded, batch=256, stream=stream, ws=tws, out=tout)
        assert rc == _lib.B2D_OK, L.b2d_last_error()
        rc, _, _ = sil_abi(xt, lt, 7, DT.L2Unexpanded, chunk=256, stream=stream, ws=sws, score=sout, per=sper)
        assert rc == _lib.B2D_OK, L.b2d_last_error()

    calls(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    t_direct, s_direct, p_direct = tout.clone(), sout.clone(), sper.clone()
    tout.fill_(-7.0)
    sout.fill_(-7.0)
    sper.fill_(-7.0)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        calls(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        assert tout.item() == t_direct.item()
        assert tout.item() == pytest.approx(oracle.trustworthiness_score(x, e, k, metric=DT.L2Expanded), abs=1e-12)
        assert abs(sout.item() - s_direct.item()) < 1e-6
        assert (sper - p_direct).abs().max().item() < 1e-6


def test_trustworthiness_error_statuses():
    """n_neighbors in [1, 63]; 2n - 3k - 1 > 0; a supported metric; leading dimensions at least the row length."""
    def status(n, k, metric=DT.L2Expanded, **kw):
        x, e = int_data(n, 6, 2, False, False, seed=n + k)
        rc, out = trust_abi(dev(x), dev(e), k, metric, **kw)
        torch.cuda.synchronize()
        return rc, out.item(), x, e

    assert status(200, 0)[0] == _lib.B2D_ERR_UNSUPPORTED
    assert status(200, 64)[0] == _lib.B2D_ERR_UNSUPPORTED
    assert status(200, 5, DT.L1)[0] == _lib.B2D_ERR_UNSUPPORTED
    assert status(200, 5, ldx=5)[0] == _lib.B2D_ERR_INVALID_ARG
    assert status(200, 5, lde=1)[0] == _lib.B2D_ERR_INVALID_ARG
    for k in (1, 32, 33, 63):
        n_min = (3 * k + 1) // 2 + 1                            # the smallest n with 2n - 3k - 1 > 0
        assert status(n_min - 1, k)[0] == _lib.B2D_ERR_INVALID_ARG, k
        rc, got, x, e = status(n_min, k)
        assert rc == _lib.B2D_OK, (k, _lib.lib().b2d_last_error())
        assert got == pytest.approx(oracle.trustworthiness_score(x, e, k, metric=DT.L2Expanded), abs=1e-12), k
    with pytest.raises(LogicError):
        trustworthiness_score(torch.zeros((95, 4), device=DEV), torch.zeros((95, 2), device=DEV), n_neighbors=63)


def test_silhouette_error_statuses():
    """2 <= n_labels <= n - 1 (INVALID_ARG), n_labels <= 12000 (UNSUPPORTED), ldx >= k, chunk >= 0."""
    x, labels = family_data(DT.L2Unexpanded, 50, 4, 3, seed=1)
    xt, lt = dev(x), dev(labels)
    assert sil_abi(xt, lt, 1)[0] == _lib.B2D_ERR_INVALID_ARG
    assert sil_abi(xt, lt, 50)[0] == _lib.B2D_ERR_INVALID_ARG
    assert sil_abi(xt, lt, 3, ldx=3)[0] == _lib.B2D_ERR_INVALID_ARG
    assert sil_abi(xt, lt, 3, chunk=-1)[0] == _lib.B2D_ERR_INVALID_ARG
    rc, score, _ = sil_abi(xt, lt, 49)
    assert rc == _lib.B2D_OK
    torch.cuda.synchronize()
    assert abs(score.item() - sil_reference(x, labels, 49).mean()) < SCORE_TOL
