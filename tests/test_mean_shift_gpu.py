"""mean_shift on the GPU against the fp64 model (tests/mean_shift_ref.py) and sklearn.cluster.MeanShift.

Accuracy bound of one step.  The new mean of a seed is sum_{j in N} x_j / |N| with the sum formed on the tensor cores:
  * split: every prepared x_j 2^E = hi + lo + r_j with |r_j| <= 2^-22 |x_j 2^E| + 2^-25 (fp16 rounding of hi, then of lo,
    and lo's subnormal floor; the matrix maximum M 2^E lies in [2^14, 2^15)), so r_j adds at most 2^-22 |x_j| + 2^-38 M;
  * fp32 accumulation: a chunk of at most 2048 data rows is 128 k-steps of 16 rows, each rounding the running sum once
    (relative 2^-23 at most, truncation included), so a chunk partial is off by <= 128 * 2^-23 sum |x_j| = 2^-16 sum |x_j|;
    adding the hi and lo halves rounds once more (2^-23 of it); the fp64 fold of the chunks adds nothing that matters;
  * the mean is rounded once to fp32 (2^-24 relative).
So per coordinate |got - ref| <= 2^-15 mean_{j in N} |x_j| + 2^-23 |ref| + 2^-37 M, with ref the fp64 mean over N.  When
every step of a fit sees the same neighbourhoods as the exact model, the final centres are one such step from the model's,
so the same bound holds for them; the fits below check that their data keep every decision (neighbourhood, stop rule,
suppression, label radius) at least 2^-14 max |x| away from its threshold."""
import numpy as np
import pytest

import mean_shift_ref as R

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


def step_bound(X, nb, ref):
    """the per-coordinate bound above for the means of the rows nb [s, n] of X"""
    ax = np.abs(X.astype(np.float64))
    mean_abs = (nb.astype(np.float64) @ ax) / np.maximum(nb.sum(1, keepdims=True), 1)
    return 2.0 ** -15 * mean_abs + 2.0 ** -23 * np.abs(ref) + 2.0 ** -37 * ax.max()


def grid(k, d, step):
    """k points on a grid of rows of three, step apart (first two coordinates)"""
    c = np.zeros((k, d))
    c[:, 0] = step * (np.arange(k) % 3)
    c[:, min(1, d - 1)] += step * (np.arange(k) // 3)
    return c


def blobs(n, d, k, h, seed, spread=0.1, sep=6.0):
    """k blobs on a grid sep * h apart, each of radius about 3.5 spread * h: every pair of a blob lies well within h,
    every other pair far beyond it.  The grid is offset from the bin lattice by 0.2 h, and rows within 0.02 h of their
    blob's mean are left out, so that no first step (from a row or a bin) moves a seed by about the stop threshold."""
    rng = np.random.default_rng(seed)
    c = grid(k, d, sep * h)
    c[:, : min(2, d)] += 0.2 * h
    lab = rng.integers(0, k, n)
    x = c[lab] + rng.normal(size=(n, d)) * (spread * h / np.sqrt(d))
    keep = np.ones(n, bool)
    for b in range(k):
        m = lab == b
        if m.any():
            keep[m] = np.linalg.norm(x[m] - x[m].mean(0), axis=1) > 0.02 * h
    return x[keep].astype(np.float32)


def pitched(x, extra=5):
    t = torch.zeros((x.shape[0], x.shape[1] + extra), dtype=torch.float32, device="cuda")
    t[:, : x.shape[1]] = torch.from_numpy(x)
    return t[:, : x.shape[1]]


def gpu(x, h, **kw):
    from raft_b200.cluster import mean_shift
    xt = x if isinstance(x, torch.Tensor) else torch.from_numpy(x).cuda()
    if kw.get("seeds") is not None and not isinstance(kw["seeds"], torch.Tensor):
        kw["seeds"] = torch.from_numpy(kw["seeds"]).cuda()
    c, lab, it = mean_shift(xt, bandwidth=h, **kw)
    return c.cpu().numpy(), lab.cpu().numpy(), it


def exact_model(x, h, **kw):
    """the model on exact distances, with the smallest distance of any decision to its threshold"""
    gaps = [np.inf]

    def within(P, Q):
        dist = np.sqrt(R.exact_d2(P, Q))
        gaps.append(np.abs(dist - h).min())
        return dist <= h

    trace = []
    out = R.mean_shift(x, h, within, R.exact_d2, h2=h * h, trace=trace, **kw)
    moved = np.asarray(trace)[np.asarray(trace) > 0]   # a shift of 0 repeats a step exactly, on the device too
    if len(moved):
        gaps.append(np.abs(moved - 1e-3 * h).min())
    return out, min(gaps)


def check_fit(x, h, x_gpu=None, **kw):
    (mc, ml, mi), gap = exact_model(x, h, **kw)
    assert gap > 2.0 ** -14 * np.abs(x).max(), "the data put a decision within %g of its threshold" % gap
    gc, gl, gi = gpu(x if x_gpu is None else x_gpu, h, **kw)
    assert gi == mi
    assert gc.shape == mc.shape
    bound = 2.0 ** -15 * np.abs(x).max() + 2.0 ** -23 * np.abs(mc)
    assert (np.abs(gc.astype(np.float64) - mc) <= bound).all()
    assert (gl == ml).all()
    return gc, gl, gi


# ---------------------------------------------------------------------------------------------------------- one step
@pytest.mark.parametrize("n,d", [(5000, 2), (3001, 17), (2500, 128), (777, 300)])
def test_single_step_against_engine_adjacency(n, d):
    """max_iter = 0 moves every seed once.  The seeds lie > 3h apart, so every mean survives as its own centre; they
    come back in (count, coordinates) order.  The counts are those of eps_neighbors_l2sq exactly: the order is by count,
    and a mean over another set would miss the reference by about |x| / |N|, far beyond the bound."""
    from raft_b200.neighbors.epsilon_neighborhood import eps_neighbors_l2sq
    h = 1.0
    rng = np.random.default_rng(n + d)
    centres = grid(12, d, 5.0 * h)
    x = (centres[rng.integers(0, 12, n)] + rng.normal(size=(n, d)) * (0.8 * h / np.sqrt(d))).astype(np.float32)
    seeds = (centres + rng.normal(size=centres.shape) * (0.1 * h / np.sqrt(d))).astype(np.float32)
    xd, sd = torch.from_numpy(x).cuda(), torch.from_numpy(seeds).cuda()
    adj, _ = eps_neighbors_l2sq(sd, xd, float(np.float32(h * h)))
    nb = torch.as_tensor(adj, device="cuda").cpu().numpy().astype(bool)
    cnt = nb.sum(1)
    assert (cnt > 0).all()
    ref = (nb.astype(np.float64) @ x.astype(np.float64)) / cnt[:, None]
    refk = ref.astype(np.float32)
    order = sorted(range(len(seeds)), key=lambda i: (cnt[i], tuple(R.ordered_bits(refk[i]))), reverse=True)
    gc, _, gi = gpu(x, h, seeds=seeds, max_iter=0)
    assert gi == 0
    assert gc.shape == seeds.shape
    bound = step_bound(x, nb, ref)
    err = np.abs(gc.astype(np.float64) - ref[order])
    assert (err <= bound[order]).all(), err.max()


# ----------------------------------------------------------------------------------------------------------- full fits
def test_full_fit_against_sklearn():
    from sklearn.cluster import MeanShift
    x = blobs(1500, 2, 5, 1.0, seed=3)
    h = 1.0
    sk = MeanShift(bandwidth=h).fit(x.astype(np.float64))
    _, gap = exact_model(x, h)
    assert gap > 2.0 ** -14 * np.abs(x).max()
    gc, gl, gi = gpu(x, h)
    assert gi == sk.n_iter_
    assert gc.shape == sk.cluster_centers_.shape
    assert (np.abs(gc - sk.cluster_centers_) <= 2.0 ** -15 * np.abs(x).max() + 1e-6).all()
    assert (gl == sk.labels_).all()


@pytest.mark.parametrize("d", [2, 3, 17, 128, 300])
def test_parameters(d):
    h = 1.0
    n = 2 * 2048 + 77 if d <= 17 else 1031   # n % 128 != 0; two chunks and a ragged third for the small d
    x = blobs(n, d, 6, h, seed=d)
    rng = np.random.default_rng(d)
    seeds = x[rng.choice(len(x), 40, replace=False)] + np.float32(0.01)
    check_fit(x, h, seeds=seeds, x_gpu=pitched(x))
    check_fit(x, h, bin_seeding=True, min_bin_freq=3)
    far = np.concatenate([x, np.full((9, d), 40.0 * h, np.float32)])   # rows far from every blob
    check_fit(far, h, seeds=seeds, cluster_all=False)


def test_every_row_a_seed():
    x = blobs(3000, 8, 4, 1.0, seed=5)
    check_fit(x, 1.0)


def test_no_neighbour_raises():
    x = blobs(500, 4, 3, 1.0, seed=6)
    with pytest.raises(ValueError, match="No point was within bandwidth"):
        gpu(x, 1.0, seeds=np.full((3, 4), 1e4, np.float32))


# -------------------------------------------------------------------------------------------------------- determinism
def test_deterministic():
    x = blobs(6000, 16, 5, 1.0, seed=7, spread=0.3)
    rng = np.random.default_rng(1)
    seeds = x[rng.choice(len(x), 700, replace=False)]
    a = gpu(x, 1.0, seeds=seeds)
    b = gpu(x, 1.0, seeds=seeds)
    ld = (len(x) + 15) // 16 * 16
    c = gpu(x, 1.0, seeds=seeds, max_mbytes_per_batch=128 * ld / 2 ** 20)          # 6 batches of 128 seeds
    perm = rng.permutation(len(seeds))
    e = gpu(x, 1.0, seeds=seeds[perm].copy(), max_mbytes_per_batch=384 * ld / 2 ** 20)
    for o in (b, c, e):
        assert o[2] == a[2]
        assert o[0].tobytes() == a[0].tobytes()
        assert (o[1] == a[1]).all()


def test_estimate_bandwidth():
    from sklearn.cluster import estimate_bandwidth as sk_eb
    from raft_b200.cluster import estimate_bandwidth
    for n, d, q in ((700, 3, 0.3), (2000, 17, 0.1), (50, 2, 0.01)):
        x = blobs(n, d, 3, 1.0, seed=n, spread=0.5)
        want = sk_eb(x.astype(np.float64), quantile=q)
        got = estimate_bandwidth(torch.from_numpy(x).cuda(), quantile=q)
        # the fp32 expanded distance: d^2 within about 2^-22 max |x|^2, so d within 2^-23 max |x|^2 / d
        mx = float(np.abs(x).max())
        assert abs(got - want) <= (2.0 ** -20 * mx * mx / want + 1e-6 * want if want > 0 else 2.0 ** -10 * mx)
    x = blobs(400, 5, 2, 1.0, seed=8, spread=0.5)
    from raft_b200.cluster import mean_shift
    c1, l1, _ = mean_shift(torch.from_numpy(x).cuda())
    c2, l2, _ = mean_shift(torch.from_numpy(x).cuda(), bandwidth=estimate_bandwidth(torch.from_numpy(x).cuda()))
    assert torch.equal(c1, c2) and torch.equal(l1, l2)
