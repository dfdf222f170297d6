"""CPU tier: the oracle against the committed golden vectors and the reference's surviving pins."""
import numpy as np
import pytest

import oracle
from oracle import DistanceType as DT
from oracle import coracle

METRICS = ["L2Expanded", "L2SqrtExpanded", "CosineExpanded", "L1", "L2Unexpanded", "L2SqrtUnexpanded",
           "Linf", "Canberra", "CorrelationExpanded", "InnerProduct"]


@pytest.mark.parametrize("case", ["small", "cfg1"])
@pytest.mark.parametrize("metric", METRICS)
def test_numpy_oracle_matches_golden(golden, case, metric):
    x, y = golden[f"{case}_x"], golden[f"{case}_y"]
    got = oracle.pairwise_distance(x, y, DT[metric])
    np.testing.assert_allclose(got, golden[f"{case}_{metric}"], rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("name", ["prob_KLDivergence", "prob_JensenShannon", "prob_HellingerExpanded",
                                  "bool_HammingUnexpanded", "bool_RusselRaoExpanded"])
def test_distribution_and_boolean_metrics_golden(golden, name):
    pre, metric = name.split("_")
    x, y = golden[f"{pre}_x"], golden[f"{pre}_y"]
    for impl in (oracle.pairwise_distance, coracle.pairwise_distance):
        got = impl(x, y, DT[metric])
        ref = golden[name]
        fin = np.isfinite(ref)
        np.testing.assert_allclose(got[fin], ref[fin], rtol=1e-9, atol=1e-9)
        assert (np.isinf(got) == np.isinf(ref)).all()


@pytest.mark.parametrize("case", ["small", "cfg1"])
def test_minkowski_golden(golden, case):
    got = oracle.pairwise_distance(golden[f"{case}_x"], golden[f"{case}_y"], DT.LpUnexpanded, 3.0)
    np.testing.assert_allclose(got, golden[f"{case}_LpUnexpanded_p3"], rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("metric", METRICS + ["LpUnexpanded"])
def test_c_oracle_matches_numpy_oracle(golden, metric):
    x, y = golden["small_x"], golden["small_y"]
    a = oracle.pairwise_distance(x, y, DT[metric], 3.0)
    b = coracle.pairwise_distance(x, y, DT[metric], 3.0, threads=2)
    np.testing.assert_allclose(a, b, rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("case", ["small", "cfg1"])
def test_fused_l2_nn_golden(golden, case):
    x, y = golden[f"{case}_x"], golden[f"{case}_y"]
    for impl in (oracle.fused_l2_nn, coracle.fused_l2_nn):
        idx, val = impl(x, y, sqrt=False)
        assert (idx == golden[f"{case}_nn_idx"]).all()
        np.testing.assert_allclose(val, golden[f"{case}_nn_val"], rtol=1e-9, atol=1e-9)
    idx, val = oracle.fused_l2_nn(x, y, sqrt=True)
    np.testing.assert_allclose(val, np.sqrt(golden[f"{case}_nn_val"]), rtol=1e-9)


def test_reference_argmin_known_answer(golden):
    """cpp/tests/matrix/argmin.cu:71-75."""
    assert (oracle.row_argmin(golden["ref_argmin_in"]) == golden["ref_argmin_out"]).all()


def test_reference_argmin_op_ties():
    """cpp/tests/core/operators_host.cpp:134-152 (kvp = (key, value))."""
    a, b, c = (0, 1.2), (0, 3.4), (1, 1.2)
    assert oracle.argmin_op(a, b) == a and oracle.argmin_op(b, a) == a
    assert oracle.argmin_op(a, c) == a and oracle.argmin_op(c, a) == a
    assert oracle.argmin_op(b, c) == c and oracle.argmin_op(c, b) == c


def test_compare_approx_semantics():
    """cpp/tests/test_utils.h:31-45: relative above eps, absolute below."""
    assert oracle.compare_approx(1000.0, 1000.05, 1e-4).all()       # rel 5e-5
    assert not oracle.compare_approx(1000.0, 1000.2, 1e-4).all()    # rel 2e-4
    assert oracle.compare_approx(0.0, 5e-5, 1e-4).all()             # abs below eps
    assert not oracle.compare_approx(0.0, 5e-3, 1e-4).all()
    assert oracle.compare_approx(np.nan, np.nan, 1e-4).all()


def test_row_norm_spec():
    """L2Norm == sum of squares: cpp/tests/linalg/norm.cu:42-66 naive kernel."""
    rng = np.random.default_rng(0)
    x = rng.uniform(-1, 1, (11, 33)).astype(np.float32)
    ref = np.array([sum(float(v) * float(v) for v in row) for row in x])
    np.testing.assert_allclose(oracle.row_norm_sq(x), ref, rtol=1e-12)


def test_fused_nn_tie_break_smallest_index():
    x = np.zeros((3, 4), np.float32)
    y = np.ones((7, 4), np.float32)
    y[2] = y[5] = 0.0
    idx, val = oracle.fused_l2_nn(x, y)
    assert (idx == 2).all() and (val == 0).all()
    idx2, _ = coracle.fused_l2_nn(x, y)
    assert (idx2 == 2).all()


def test_pack_minloc_is_argmin_op():
    rng = np.random.default_rng(1)
    v = rng.standard_normal(1000).astype(np.float32)
    v[10] = v[500] = v.min() - 1.0
    i = np.arange(1000)
    key = oracle.pack_minloc(v, i).min()
    bv, bi = oracle.unpack_minloc(np.array([key]))
    assert bi[0] == 10 and bv[0] == v[10]
    # order-preserving across signs and zero
    vals = np.array([-3.5, -0.0, 0.0, 1e-30, 2.0, np.inf], np.float32)
    keys = oracle.pack_minloc(vals, np.zeros(6, np.int64))
    assert (np.diff(keys) >= 0).all()


def test_make_blobs_distribution():
    x, lab, c = oracle.make_blobs(20000, 8, seed=3)
    assert x.dtype == np.float32 and c.shape == (5, 8) and np.abs(c).max() <= 10
    resid = x - c[lab]
    assert abs(resid.std() - 1.0) < 0.02 and abs(resid.mean()) < 0.02


def test_knn_oracle_against_brute_force_sort():
    """oracle.knn_l2 (blocked, lexsort by (distance, index)) == full sort of the fp64 distance matrix."""
    rng = np.random.default_rng(4)
    x = rng.standard_normal((37, 9))
    y = rng.standard_normal((211, 9))
    y[[50, 120]] = y[7]                                    # ties -> ascending index
    d = ((x[:, None, :] - y[None, :, :]) ** 2).sum(-1)
    order = np.lexsort((np.broadcast_to(np.arange(211), d.shape), d), axis=1)[:, :13]
    gi, gv = oracle.knn_l2(x, y, 13, block=64)
    assert (gi == order).all()
    assert np.allclose(gv, np.take_along_axis(d, order, axis=1), rtol=1e-12, atol=1e-12)
    gi1, gv1 = oracle.knn_l2(x, y, 1)
    ni, nv = oracle.fused_l2_nn(x, y)
    assert (gi1[:, 0] == ni).all() and np.allclose(gv1[:, 0], nv)
    # oracle.knn (any metric, blocked per 'block' columns) == one sort of the whole row, ties and NaN rows included
    y[33] = np.nan                                         # NaN distances: after every number
    y[150] = 0.0                                           # zero norm: NaN under the cosine family
    x[5] = np.nan                                          # a row of NaN distances: index order
    for mt in (oracle.DistanceType.L2Expanded, oracle.DistanceType.L2SqrtExpanded, oracle.DistanceType.CosineExpanded,
               oracle.DistanceType.CorrelationExpanded):
        d = oracle.pairwise_distance(x, y, mt)
        order = np.lexsort((np.broadcast_to(np.arange(211), d.shape), d), axis=1)
        for kk, block in ((13, 64), (13, 4096), (1, 50), (211, 100)):
            gi, gv = oracle.knn(x, y, kk, mt, block=block)
            assert gi.dtype == np.int64 and gi.shape == (37, kk)
            assert (gi == order[:, :kk]).all(), (mt, kk, block)
            want = np.take_along_axis(d, order[:, :kk], axis=1)
            if block >= 211:   # the same pairwise_distance call as the whole row: bit-identical
                assert np.array_equal(gv, want, equal_nan=True)
            assert np.allclose(gv, want, rtol=1e-12, atol=1e-12, equal_nan=True)
        assert (np.delete(order, 5, axis=0)[:, :209] != 33).all() and (order[5] == np.arange(211)).all()
    gi, gv = oracle.knn(x, y, 13, oracle.DistanceType.L2Expanded, block=64)
    ri, rv = oracle.knn_l2(x, y, 13, block=64)
    assert (gi[x[:, 0] == x[:, 0]] == ri[x[:, 0] == x[:, 0]]).all()


def test_silhouette_oracle_pinned_to_sklearn():
    """The silhouette restatement against scikit-learn's implementation (an independent pin: same
    definition as raft::stats::silhouette_score, incl. score 0 for singleton clusters)."""
    skm = pytest.importorskip("sklearn.metrics")
    rng = np.random.default_rng(8)
    x = rng.standard_normal((300, 7)) + rng.integers(0, 4, 300)[:, None] * 2.5
    labels = rng.integers(0, 5, 300)
    labels[labels == 4] = 3
    labels[0] = 4                                           # a singleton cluster
    for metric, sk in ((oracle.DistanceType.L2SqrtUnexpanded, "euclidean"), (oracle.DistanceType.L2Unexpanded, "sqeuclidean"),
                       (oracle.DistanceType.L1, "cityblock"), (oracle.DistanceType.CosineExpanded, "cosine")):
        got, per = oracle.silhouette_score(x, labels, metric=metric, return_samples=True)
        assert abs(got - skm.silhouette_score(x, labels, metric=sk)) < 1e-9
        assert np.allclose(per, skm.silhouette_samples(x, labels, metric=sk), atol=1e-9)
        assert per[0] == 0.0


def test_trustworthiness_oracle_pinned_to_sklearn():
    skm = pytest.importorskip("sklearn.manifold")
    rng = np.random.default_rng(12)
    x = rng.standard_normal((180, 10))
    w = rng.standard_normal((10, 2))
    good, bad = x @ w + 0.05 * rng.standard_normal((180, 2)), rng.standard_normal((180, 2))
    for emb in (good, bad, x[:, :3]):
        for k in (3, 7):
            assert abs(oracle.trustworthiness_score(x, emb, k) - skm.trustworthiness(x, emb, n_neighbors=k)) < 1e-12
    assert oracle.trustworthiness_score(x, x, 5) == 1.0
    # embeddings of coincident groups of exactly k + 1 points: a sample's k neighbours are its k group mates whichever
    # tied mate a kNN lists first, so sklearn's neighbour sets are the oracle's
    for k in (1, 4, 9):
        groups = np.repeat(rng.standard_normal((180 // (k + 1), 2)), k + 1, axis=0)
        emb = groups[rng.permutation(len(groups))]
        xs = x[: len(emb)]
        got = oracle.trustworthiness_score(xs, emb, k)
        assert abs(got - skm.trustworthiness(xs, emb, n_neighbors=k)) < 1e-12, k
        assert got < 0.9                                    # the embedding is not trustworthy: the check has teeth


def _trustworthiness_by_definition(x, e, k):
    """Trustworthiness by its definition with plain Python sorts: the k samples nearest to i in the embedding (i
    excluded, ties to the smaller index), each ranked among all samples ordered by (original-space distance, index)
    with i itself first."""
    n = len(x)
    dx = ((x[:, None, :] - x[None, :, :]) ** 2).sum(-1)
    de = ((e[:, None, :] - e[None, :, :]) ** 2).sum(-1)
    t = 0
    for i in range(n):
        nbrs = [j for _, j in sorted((de[i, j], j) for j in range(n) if j != i)[:k]]
        order = [i] + [j for _, j in sorted((dx[i, j], j) for j in range(n) if j != i)]
        pos = {j: r for r, j in enumerate(order)}
        t += sum(max(0, pos[j] - k) for j in nbrs)
    return 1.0 - 2.0 / (n * k * (2.0 * n - 3.0 * k - 1.0)) * t


@pytest.mark.parametrize("group", [2, 3, 5, 8])
def test_trustworthiness_oracle_counts_exactly_k_neighbours(group):
    """Coincident groups in the embedding, larger than k + 1 for most k here, and duplicate rows in the original space:
    a sample with k + 1 or more coincident mates of smaller index is not in its own (k + 1)-nearest list, and counting
    the whole list would give it k + 1 neighbours.  Integer coordinates: every distance is exact, so the ties are
    real ties and the tie rule decides."""
    rng = np.random.default_rng(20 + group)
    n = 120
    e = np.repeat(rng.integers(-6, 7, (n // group, 2)), group, axis=0)[rng.permutation(n)].astype(np.float64)
    x = rng.integers(-4, 5, (n, 5)).astype(np.float64)
    x[10:14] = x[3]                                          # duplicate rows in the original space too
    for k in (1, group - 1, group, group + 1):
        if k < 1:
            continue
        want = _trustworthiness_by_definition(x, e, k)
        assert 0.0 <= want <= 1.0                            # k neighbours per row: the normalisation holds
        for metric in (DT.L2SqrtUnexpanded, DT.L2Unexpanded, DT.L2Expanded, DT.L2SqrtExpanded):
            assert abs(oracle.trustworthiness_score(x, e, k, metric=metric) - want) < 1e-12, (k, metric)


def test_silhouette_oracle_is_nan_for_one_non_empty_cluster():
    """sklearn raises 'Number of labels is 1'; the restatement returns NaN (the C ABI's answer), whatever n_labels is
    declared."""
    rng = np.random.default_rng(9)
    x = rng.standard_normal((50, 4))
    with np.errstate(invalid="ignore"):
        for labels, nl in ((np.zeros(50, int), 3), (np.full(50, 2), None), (np.full(50, 1), 2)):
            assert np.isnan(oracle.silhouette_score(x, labels, nl))
        x[:] = x[0]                                           # one cluster of identical points
        assert np.isnan(oracle.silhouette_score(x, np.zeros(50, int), 2))
