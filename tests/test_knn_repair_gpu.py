"""GPU tier: the fused kNN's overflow repair.  When a row's 128-entry candidate list overflows in a way that matters,
knn_merge_kernel puts the row on the pass's dirty list and knn_fix_kernel measures the pass's columns again in fp32; every
repaired row is measured once more over all columns after the last pass.  That path is what makes brute_force.knn exact
for any input order, so these cases make it run: for every metric, in the resident (k <= 128) and the streaming kernel,
with more dirty rows than knn_fix_kernel has blocks, through padded leading dimensions, with outlier, NaN and zero-norm
rows, and with exact ties across passes.

In the adversarial cases the expected indices follow from how the data is built, so only the returned pairs need an fp64
evaluation.  The checker has no mismatch allowance: every row must be a valid k-nearest set (check_knn_strict)."""
import numpy as np
import pytest
import torch

import oracle
from raft_b200 import LogicError, _lib
from raft_b200.distance.distance_type import resolve_metric
from raft_b200.neighbors import brute_force

pytestmark = pytest.mark.gpu

DT = oracle.DistanceType
ORACLE_METRIC = {"sqeuclidean": DT.L2Expanded, "euclidean": DT.L2SqrtExpanded, "cosine": DT.CosineExpanded,
                 "correlation": DT.CorrelationExpanded}
REL = 1e-4     # returned distance against the fp64 distance of the returned index (CompareApprox)
DELTA = 1e-5   # near-tie resolution at the k-th position, relative


def cosine_family(metric):
    return metric in ("cosine", "correlation")


def pair_dist(x, y, idx, metric, rows=256):
    """fp64 distance of query row i to y[idx[i, j]] for every (i, j); idx < 0 gives NaN."""
    out = np.empty(idx.shape)
    for r0 in range(0, idx.shape[0], rows):
        xi = x[r0:r0 + rows].astype(np.float64)[:, None, :]
        ii = idx[r0:r0 + rows]
        yi = y[np.maximum(ii, 0)].astype(np.float64)
        if cosine_family(metric):
            if metric == "correlation":
                xi = xi - xi.mean(-1, keepdims=True)
                yi = yi - yi.mean(-1, keepdims=True)
            with np.errstate(divide="ignore", invalid="ignore"):
                d = 1.0 - (xi * yi).sum(-1) / np.sqrt((xi * xi).sum(-1) * (yi * yi).sum(-1))
        else:
            d = ((xi - yi) ** 2).sum(-1)
            if metric == "euclidean":
                d = np.sqrt(d)
        out[r0:r0 + rows] = np.where(ii >= 0, d, np.nan)
    return out


def check_knn_strict(gd, gi, x, y, kk, metric, ref_i, exact=False):
    """Every row: shape, indices in range and unique, distances ascending; each distance equal to the fp64 distance of
    its index (REL, plus 4e-7 absolute for the cosine family); a valid k-nearest set against the exact top-kk ref_i
    (ascending by fp64 distance, then index): nothing returned is farther than the true k-th distance + tol, and every
    index closer than the true k-th distance - tol is returned (tol = DELTA relative).  exact: the index lists equal
    ref_i (cases built with exact ties)."""
    m, n = x.shape[0], y.shape[0]
    assert gi.shape == (m, kk) and gd.shape == (m, kk) and ref_i.shape == (m, kk)
    assert gi.min() >= 0 and gi.max() < n, (gi.min(), gi.max())
    srt = np.sort(gi, axis=1)
    dup = (np.diff(srt, axis=1) == 0).any(axis=1)
    assert not dup.any(), f"{dup.sum()} rows return an index twice; first row {np.flatnonzero(dup)[0]}"
    bad = (np.diff(gd, axis=1) < 0).any(axis=1)
    assert not bad.any(), f"{bad.sum()} rows not ascending; first row {np.flatnonzero(bad)[0]}"
    floor = 4e-7 if cosine_family(metric) else 0.0
    true_d = pair_dist(x, y, gi, metric)
    err = np.abs(gd - true_d) > REL * np.abs(true_d) + floor
    assert not err.any(), (f"{err.sum()} distances differ from fp64; first at {tuple(np.argwhere(err)[0])}: "
                           f"{gd[err][0]!r} vs {true_d[err][0]!r}")
    ref_d = pair_dist(x, y, ref_i, metric)
    kth = ref_d[:, -1:]
    tol = DELTA * np.abs(kth) + floor
    far = true_d > kth + tol
    assert not far.any(), (f"{far.any(axis=1).sum()} rows return an index beyond the k-th distance; first row "
                           f"{np.flatnonzero(far.any(axis=1))[0]}")
    must = ref_d < kth - tol
    found = (ref_i[:, :, None] == gi[:, None, :]).any(-1)
    miss = (must & ~found).any(axis=1)
    assert not miss.any(), (f"{miss.sum()} of {m} rows miss a neighbour closer than the k-th; first row "
                            f"{np.flatnonzero(miss)[0]}: got {gi[np.flatnonzero(miss)[0]].tolist()}")
    if exact:
        wrong = (gi != ref_i).any(axis=1)
        assert not wrong.any(), (f"{wrong.sum()} of {m} rows differ from the exact index list; first row "
                                 f"{np.flatnonzero(wrong)[0]}: got {gi[np.flatnonzero(wrong)[0]].tolist()}, "
                                 f"want {ref_i[np.flatnonzero(wrong)[0]].tolist()}")


def run_knn(x, y, kk, metric, **kw):
    gd, gi = brute_force.knn(torch.from_numpy(y).cuda(), torch.from_numpy(x).cuda(), k=kk, metric=metric, **kw)
    return gd.cpu().numpy(), gi.cpu().numpy()


def first_by(key, kk, m):
    """The kk smallest entries of key (ties: smaller index), the same for every one of m query rows."""
    order = np.lexsort((np.arange(len(key)), key))[:kk]
    return np.broadcast_to(order, (m, kk)).astype(np.int64)


def line_data(m, n, k, seed, v_at=None):
    """y on a line through the origin, t_j |dir| from 50 down to 1, queries within 0.01 * sqrt(k) of the origin: the
    distance of every query grows with t, so it falls with the index -- every pass improves on all earlier ones and
    overflows.  v_at: from that index on, t rises again (a V: the rest of that pass adds nothing).  Returns x, y, t."""
    rng = np.random.default_rng(seed)
    direction = rng.standard_normal(k)
    direction /= np.linalg.norm(direction)
    if v_at is None:
        t = np.linspace(50.0, 1.0, n)
    else:
        h = 49.0 / (v_at - 1)
        t = np.concatenate([np.linspace(50.0, 1.0, v_at), 1.0 + (np.arange(n - v_at) + 0.5) * h])
    y = (t[:, None] * direction[None, :]).astype(np.float32)
    x = (rng.standard_normal((m, k)) * 0.01).astype(np.float32)
    return x, y, t


def arc_data(m, n, k, seed, center):
    """Cosine / correlation adversarial order: y_j = s_j (cos th_j u + sin th_j v) with th_j falling from 1.5 to 0.5 and
    s_j in [0.5, 2]; queries u + eps w, w orthogonal to u and v.  The distance 1 - cos th_j / sqrt(1 + eps^2) falls with
    the index; neighbouring distances differ by >= 1e-5, far above the kernel's error.  center: u, v, w have zero mean
    and every row of y gets a random constant added (the correlation is unchanged, the cosine is not)."""
    rng = np.random.default_rng(seed)
    basis = rng.standard_normal((k, min(k - 1, 34)))
    if center:
        basis -= basis.mean(axis=0, keepdims=True)
    q, _ = np.linalg.qr(basis)                              # orthonormal columns (zero-mean when centred)
    u, v = q[:, 0], q[:, 1]
    w = rng.standard_normal((m, q.shape[1] - 2)) @ q[:, 2:].T
    w /= np.linalg.norm(w, axis=1, keepdims=True)
    th = np.linspace(1.5, 0.5, n)
    s = rng.uniform(0.5, 2.0, n)
    y = s[:, None] * (np.cos(th)[:, None] * u[None, :] + np.sin(th)[:, None] * v[None, :])
    if center:
        y += (rng.uniform(-2.0, 2.0, n) * s / np.sqrt(k))[:, None]
    eps = rng.uniform(0.0, 0.3, m)
    x = u[None, :] + eps[:, None] * w
    return x.astype(np.float32), y.astype(np.float32), th


# feature dimension -> (n, kk, metric): the resident kernel (k <= 128) and the streaming one, up to the 320-wide xs buffer
# of knn_fix_kernel; m = 2000 dirty rows (> 2 x 132 blocks), passes up to 65536 columns wide, every one repaired
LINE_CASES = [(24, 131072, 1, "sqeuclidean"), (96, 131072, 16, "sqeuclidean"), (128, 65536, 64, "euclidean"),
              (200, 32768, 1, "sqeuclidean"), (320, 16384, 16, "sqeuclidean")]


@pytest.mark.parametrize("k,n,kk,metric", LINE_CASES)
def test_repair_l2_adversarial_order(k, n, kk, metric):
    m = 2000
    x, y, t = line_data(m, n, k, seed=k)
    ref = first_by(t, kk, m)
    ri, _ = oracle.knn(x[:3], y, kk, ORACLE_METRIC[metric])           # the construction, checked on three rows
    assert (ri == ref[:3]).all()
    gd, gi = run_knn(x, y, kk, metric)
    check_knn_strict(gd, gi, x, y, kk, metric, ref)
    assert (gi[:, 0] == n - 1).all()


@pytest.mark.parametrize("k,kk", [(128, 64), (200, 16)])
def test_repair_v_shape(k, kk):
    """The order turns round in the middle of the last pass [n/2, n): the pass is repaired, and its tail after the turn
    adds no candidate, so knn_fix_kernel runs many chunks without a sort."""
    m, n = 1000, 32768
    x, y, t = line_data(m, n, k, seed=k + 1, v_at=n // 2 + n // 4)
    ref = first_by(t, kk, m)
    gd, gi = run_knn(x, y, kk, "sqeuclidean")
    check_knn_strict(gd, gi, x, y, kk, "sqeuclidean", ref)


@pytest.mark.parametrize("k,kk", [(64, 16), (200, 64)])
@pytest.mark.parametrize("metric", ["cosine", "correlation"])
def test_repair_cosine_family_adversarial_order(metric, k, kk):
    m, n = 600, 32768
    x, y, th = arc_data(m, n, k, seed=k + kk, center=metric == "correlation")
    ref = first_by(th, kk, m)
    ri, _ = oracle.knn(x[:3], y, kk, ORACLE_METRIC[metric])
    assert (ri == ref[:3]).all()
    gd, gi = run_knn(x, y, kk, metric)
    check_knn_strict(gd, gi, x, y, kk, metric, ref)


def dup_layout(n, rng):
    """Positions of the exact duplicates of the nearest row: two in the first passes, 20 in [256, 512), 200 scattered
    over the pass [2048, 4096), two in the last pass [4096, n)."""
    wide = np.sort(rng.choice(np.arange(2048, 4096), 200, replace=False))
    mid = np.sort(rng.choice(np.arange(256, 512), 20, replace=False))
    return np.concatenate([[3, 200], mid, wide, [5000, n - 1]])


@pytest.mark.parametrize("kk", [16, 64])
@pytest.mark.parametrize("metric", ["sqeuclidean", "cosine"])
def test_repair_ties_across_passes(metric, kk):
    """More than 128 exact duplicates of the nearest row inside one pass, and duplicates before and after it.  kk = 16:
    the 16 nearest are known before that pass, so it overflows only with ties at the threshold and needs no repair.
    kk = 64: it overflows with rows that enter the result and is repaired, while duplicates from earlier passes are in
    the top-k.  Either way the result is the kk smallest duplicate indices, in index order."""
    m, n, k = 300, 8192, 64
    rng = np.random.default_rng(kk)
    y = rng.standard_normal((n, k)).astype(np.float32)
    z = rng.standard_normal(k).astype(np.float32)
    pos = dup_layout(n, rng)
    y[pos] = z
    x = (z[None, :] + 0.3 * rng.standard_normal((m, k))).astype(np.float32)
    ref = np.broadcast_to(pos[:kk], (m, kk)).astype(np.int64)
    ri, _ = oracle.knn(x[:3], y, kk, ORACLE_METRIC[metric])
    assert (ri == ref[:3]).all()
    gd, gi = run_knn(x, y, kk, metric)
    check_knn_strict(gd, gi, x, y, kk, metric, ref, exact=True)
    assert (gd == gd[:, :1]).all(), "duplicates of one row must get one distance"


@pytest.mark.parametrize("metric", ["sqeuclidean", "correlation"])
def test_repair_padded_leading_dimensions(metric):
    """The C ABI with ldx = k + 3 and ldy = k + 5 (NaN in the padding, which no kernel may read), adversarial order."""
    m, n, k, kk = 700, 16384, 96, 16
    if metric == "sqeuclidean":
        x, y, key = line_data(m, n, k, seed=11)
    else:
        x, y, key = arc_data(m, n, k, seed=12, center=True)
    ref = first_by(key, kk, m)
    xp = torch.full((m, k + 3), float("nan"), device="cuda")
    yp = torch.full((n, k + 5), float("nan"), device="cuda")
    xp[:, :k] = torch.from_numpy(x).cuda()
    yp[:, :k] = torch.from_numpy(y).cuda()
    idx = torch.empty((m, kk), dtype=torch.int64, device="cuda")
    dist = torch.empty((m, kk), dtype=torch.float32, device="cuda")
    L = _lib.lib()
    ws = torch.empty(L.b2d_knn_l2_workspace_bytes(m, n, k, kk), dtype=torch.uint8, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    _lib.check(L.b2d_knn(stream, idx.data_ptr(), dist.data_ptr(), int(resolve_metric(metric)), xp.data_ptr(), k + 3,
                         yp.data_ptr(), k + 5, m, n, k, kk, ws.data_ptr(), ws.numel()))
    torch.cuda.synchronize()
    check_knn_strict(dist.cpu().numpy(), idx.cpu().numpy(), x, y, kk, metric, ref)


@pytest.mark.parametrize("order", ["random", "adversarial"])
def test_outlier_rows(order):
    """One x row and one y row at 1e9, one y row at 2e8: per-row exponents in the tensor kernel (EPI_TOPK).  Every row,
    ordinary or not, must stay a valid k-nearest set."""
    m, k, kk = 300, 96, 32
    rng = np.random.default_rng(3)
    if order == "random":
        n = 20000
        x = rng.standard_normal((m, k)).astype(np.float32)
        y = (rng.standard_normal((n, k)) + 0.2).astype(np.float32)
    else:
        n = 8192
        x, y, _ = line_data(m, n, k, seed=5)
    for arr, row, scale in ((x, 7, 1e9), (y, 100, 1e9), (y, n - 5, 2e8)):
        d = rng.standard_normal(k)
        arr[row] = (scale * d / np.linalg.norm(d)).astype(np.float32)
    ref, _ = oracle.knn(x, y, kk, DT.L2Expanded)
    gd, gi = run_knn(x, y, kk, "sqeuclidean")
    check_knn_strict(gd, gi, x, y, kk, "sqeuclidean", ref)
    assert not np.isin(gi[np.arange(m) != 7], [100, n - 5]).any()


@pytest.mark.parametrize("offset", [0, 1000])
@pytest.mark.parametrize("metric", ["sqeuclidean", "cosine", "correlation"])
def test_nan_and_zero_norm_rows(metric, offset):
    """Rows of y with a NaN distance (a NaN element; zero norm under cosine, a constant row under correlation) never
    appear in a result, also where they would be the nearest; every other query gets the result of the data without
    them.  A query without any candidate gets index -1 and +inf in every slot, with or without global_id_offset.
    Adversarial order, so the repair meets the bad rows too."""
    m, n, k, kk = 400, 4096, 48, 16
    if metric == "sqeuclidean":
        x, y, _ = line_data(m, n, k, seed=21)
    else:
        x, y, _ = arc_data(m, n, k, seed=22, center=metric == "correlation")
    y[[10, 2000]] = np.nan                 # whole rows
    y[n - 1, 5] = np.nan                   # the would-be nearest row
    x[3, 0] = np.nan
    x[4] = np.nan
    bad_y = [10, 2000, n - 1]
    if metric != "sqeuclidean":
        y[n - 2] = 0.0 if metric == "cosine" else 1.5     # the next nearest: no direction
        x[5] = 0.0 if metric == "cosine" else -2.0
        bad_y.append(n - 2)
    bad_x = [3, 4] if metric == "sqeuclidean" else [3, 4, 5]
    keep_y = np.setdiff1d(np.arange(n), bad_y)
    keep_x = np.setdiff1d(np.arange(m), bad_x)
    ri, _ = oracle.knn(x[keep_x], y[keep_y], kk, ORACLE_METRIC[metric])
    gd, gi = run_knn(x, y, kk, metric, global_id_offset=offset)
    assert (gi[bad_x] == -1).all() and np.isposinf(gd[bad_x]).all(), (gi[bad_x], gd[bad_x])
    gi_ok = gi[keep_x] - offset
    check_knn_strict(gd[keep_x], gi_ok, x[keep_x], y, kk, metric, keep_y[ri])
    assert not np.isin(gi_ok, bad_y).any()


@pytest.mark.parametrize("kk", [1, 63, 64])
@pytest.mark.parametrize("n", ["kk", 128, 129, 256, 257, 513])
def test_pass_boundaries(n, kk):
    """The first pass (128 columns), a partial last pass, and n_neighbors == n, on random data."""
    n = kk if n == "kk" else n
    m, k = 200, 40
    rng = np.random.default_rng(n * 100 + kk)
    x = rng.standard_normal((m, k)).astype(np.float32)
    y = rng.standard_normal((n, k)).astype(np.float32)
    ref, _ = oracle.knn(x, y, kk, DT.L2Expanded)
    gd, gi = run_knn(x, y, kk, "sqeuclidean")
    check_knn_strict(gd, gi, x, y, kk, "sqeuclidean", ref)
    if n == kk:
        assert (np.sort(gi, axis=1) == np.arange(n)).all()


def test_argument_limits():
    """Feature dimension 320 is the limit (knn_fix_kernel keeps the query row in a 320-float buffer), 64 neighbours."""
    rng = np.random.default_rng(1)
    y = torch.from_numpy(rng.standard_normal((500, 321)).astype(np.float32)).cuda()
    x = torch.from_numpy(rng.standard_normal((20, 321)).astype(np.float32)).cuda()
    gd, gi = brute_force.knn(y[:, :320].contiguous(), x[:, :320].contiguous(), k=4)
    assert tuple(gi.shape) == (20, 4)
    with pytest.raises(LogicError):
        brute_force.knn(y, x, k=4)
    with pytest.raises(LogicError):
        brute_force.knn(y[:, :320].contiguous(), x[:, :320].contiguous(), k=65)
