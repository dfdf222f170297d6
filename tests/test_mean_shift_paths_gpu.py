"""mean_shift's neighbour sums (ms_sum_kernel, raft_b200/csrc/mean_shift.cuh) on every k-block group, chunk, seed tile
and batch edge against fp64, through b2d_debug_mean_shift_sums (the fit's data preparation and launcher on a caller's
adjacency) and through the fit; non-finite and scaled data rows; and, without a GPU, the debug entry's argument checks
and the power of the comparison to catch a slip of the kernel.

Bound of one chunk partial (the per-chunk form of the one-step bound in tests/test_mean_shift_gpu.py).  For seed i,
chunk c and column t let N_c be the rows j of the chunk with adj[i][j] = 1 and D the rows whose factor 2^(E - e_j)
rounds to 0 in fp16 (tests/mean_shift_ref.py prep_scales; they are left out of the sums, not of the counts).  With
S = sum_{j in N_c \\ D} x_j[t] and A = sum_{j in N_c \\ D} |x_j[t]| in fp64:
  * split: each prepared row is x_j 2^(e_j) = hi + lo + r_j with |r_j| <= 2^-22 |x_j 2^(e_j)| + 2^-25, and 2^-25
    2^(-e_j) <= 2^-39 M (M the data maximum): 2^-22 A + 2^-38 M |N_c| in all;
  * fp32 accumulation: the products (A is 0 / 1 or a power of two) are exact; a k-step of 16 rows that has a neighbour
    rounds the running sum at most twice (the MMA may add its k = 16 in two halves), 2^-23 relative to A 2^E each; a
    k-step without one adds zeros, exactly.  The lo columns' sums are 2^-11 A at most, counted by a factor 1 + 2^-10;
  * hi + lo are added once in fp32: 2^-23 |S|.
So |part[c][i][t] 2^-E - S| <= (2 k_c 2^-23 + 2^-22) (1 + 2^-10) A + 2^-23 |S| + 2^-38 M |N_c|, with k_c the k-steps of
chunk c holding a neighbour of seed i, and counts[c][i] = |N_c| exactly."""
import ctypes

import numpy as np
import pytest
import torch

import mean_shift_ref as R
from raft_b200 import _lib

CHUNK, KS, TILE = 2048, 16, 128
P = 1 << 12   # a non-null pointer that is never dereferenced (every call below fails before any work)
E_ARG, E_UNS = _lib.B2D_ERR_INVALID_ARG, _lib.B2D_ERR_UNSUPPORTED
# d -> (k-blocks per group, groups, k-blocks of the last group): every class of ms_sums and a column tail in each
SUM_D = [1, 31, 32, 33, 64, 65, 96, 97, 128, 129, 160, 193, 224, 256, 257, 288, 300, 320]


def plan(d):
    nkb = (d + 31) // 32
    g = nkb if nkb < 3 else 4
    ng = -(-nkb // g)
    return g, ng, nkb - (ng - 1) * g


def round16(v):
    return (v + 15) // 16 * 16


# ------------------------------------------------------------------------------------------------------- reference
def chunk_reference(adj, x):
    """fp64 sums of the data x [n, d] (torch fp32) per chunk over the adjacency adj [m, n] (torch uint8, 0 / 1), as the
    kernel forms them: non-finite rows and rows of D (module docstring) left out of the sums.  Returns (S, A, cnt, ks,
    E, M): S, A [nchunks, m, d], cnt and ks (k-steps with a neighbour) [nchunks, m]."""
    m, n = adj.shape
    E, M, svec, _ = R.prep_scales(x.cpu().numpy())
    keep = torch.from_numpy(svec >= 2.0 ** -24).to(x.device) & torch.isfinite(x).all(1)
    xd = torch.where(keep[:, None], x.double(), torch.zeros((), dtype=torch.float64, device=x.device))
    S, A, cnt, ks = [], [], [], []
    for c0 in range(0, n, CHUNK):
        a = adj[:, c0:c0 + CHUNK].double()
        S.append(a @ xd[c0:c0 + CHUNK])
        A.append(a @ xd[c0:c0 + CHUNK].abs())
        cnt.append(a.sum(1))
        pad = torch.nn.functional.pad(a, (0, (-a.shape[1]) % KS))
        ks.append(pad.view(m, -1, KS).amax(2).sum(1))
    return torch.stack(S), torch.stack(A), torch.stack(cnt), torch.stack(ks), E, M


def check_sums(part, counts, E, ref):
    """part [nchunks, m, d] (fp32, 2^E scaled) and counts [nchunks, m] against chunk_reference's ref, within the module
    docstring's bound; raises AssertionError"""
    S, A, cnt, ks, _, M = ref
    assert tuple(part.shape) == tuple(S.shape) and tuple(counts.shape) == tuple(cnt.shape)
    assert torch.equal(counts.double(), cnt), "counts differ from the adjacency's"
    got = part.double() * 2.0 ** -E
    assert bool(torch.isfinite(got).all()), "a partial is not finite"
    bound = ((2 * ks[..., None] * 2.0 ** -23 + 2.0 ** -22) * (1 + 2.0 ** -10) * A + 2.0 ** -23 * S.abs()
             + 2.0 ** -38 * M * cnt[..., None])
    err = (got - S).abs()
    bad = err > bound
    assert not bool(bad.any()), "%d partials beyond the bound, worst excess %g" % (
        int(bad.sum()), float((err - bound).max()))


# --------------------------------------------------------------------------------------------------------- data
def make_adj(m, n, density, rng, extra=0):
    """Bernoulli(density) bytes [m, n + extra]; with m >= 4 row 0 empty, row 1 full and rows 2, 3 with one neighbour (the
    last row and a random one).  The extra columns are 0xff: past n nothing may be read."""
    a = (rng.random((m, n)) < density).astype(np.uint8)
    if m >= 4:
        a[0], a[1], a[2:4] = 0, 1, 0
        a[2, n - 1] = 1
        a[3, rng.integers(n)] = 1
    return np.concatenate([a, np.full((m, extra), 0xFF, np.uint8)], axis=1)


def make_x(n, d, rng):
    """rows of varied scale and sign, fp32"""
    return (rng.normal(size=(n, d)) * rng.uniform(0.5, 2.0, d) + rng.normal(size=d)).astype(np.float32)


def on_device(a, pitch):
    """a [r, c] in a device matrix with row pitch `pitch` (elements), as a view of its first c columns"""
    t = torch.zeros((a.shape[0], pitch), dtype=torch.from_numpy(a).dtype, device="cuda")
    t[:, : a.shape[1]] = torch.from_numpy(a)
    return t[:, : a.shape[1]]


def debug_sums(adj, x):
    """b2d_debug_mean_shift_sums on the device views adj [m, n] (uint8, any row pitch) and x [n, d] (fp32): (part,
    counts, E, info)"""
    m, n, d = adj.shape[0], x.shape[0], x.shape[1]
    nch = -(-n // CHUNK)
    part = torch.full((nch, m, d), float("nan"), dtype=torch.float32, device="cuda")
    counts = torch.full((nch, m), 0xDEAD, dtype=torch.int32, device="cuda")
    e = torch.zeros(1, dtype=torch.int32, device="cuda")
    info = (ctypes.c_int64 * 6)()
    L = _lib.lib()
    ws = torch.empty(L.b2d_mean_shift_fit_workspace_bytes(n, d, m, 0), dtype=torch.uint8, device="cuda")
    ws.fill_(0xA5)   # stale bytes: nothing may depend on the workspace's contents
    stream = torch.cuda.current_stream().cuda_stream
    _lib.check(L.b2d_debug_mean_shift_sums(stream, adj.data_ptr(), adj.stride(0), m, x.data_ptr(), x.stride(0), n, d,
                                           part.data_ptr(), counts.data_ptr(), e.data_ptr(), info, ws.data_ptr(),
                                           ws.numel()))
    torch.cuda.synchronize()
    return part, counts, int(e.item()), list(info)


def run_case(m, n, d, density, seed, x=None, adj=None, extra=16, ldx_extra=3):
    """the sums of one case against the reference; returns (part, counts, info, ref)"""
    rng = np.random.default_rng(seed)
    x = make_x(n, d, rng) if x is None else x
    adj = make_adj(m, n, density, rng, extra) if adj is None else adj
    pitch = round16(adj.shape[1])
    ad, xd = on_device(adj, pitch), on_device(x, d + ldx_extra)
    part, counts, E, info = debug_sums(ad, xd)
    ref = chunk_reference(ad[:, :n], xd)
    assert E == ref[4]
    g, ng, _ = plan(d)
    nch = -(-n // CHUNK)
    items = -(-m // TILE) * nch * ng
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert info == [g, ng, nch, items, min(items, sms), int(R.prep_scales(x)[3].any())]
    check_sums(part, counts, E, ref)
    return part, counts, info, ref


# ----------------------------------------------------------------------------------------------- CPU: the contract
def test_sum_dims_reach_every_group_class():
    """the d of the GPU cases reach G = 1, 2 and 4, one to three groups, and a last group of 1, 2, 3 and 4 k-blocks"""
    classes = {plan(d) for d in SUM_D}
    assert {(g, gn) for g, _, gn in classes} == {(1, 1), (2, 2), (4, 1), (4, 2), (4, 3), (4, 4)}
    assert {ng for _, ng, _ in classes} == {1, 2, 3}
    assert {d % 32 for d in SUM_D} >= {0, 1, 31}


def debug_call(adj=P, ld=16, m=4, x=P, ldx=8, n=10, d=8, part=P, cnt=P, e=P, info=True, ws=P * 256, wsb=1 << 40):
    buf = (ctypes.c_int64 * 6)() if info else None
    rc = _lib.lib().b2d_debug_mean_shift_sums(None, adj, ld, m, x, ldx, n, d, part, cnt, e, buf, ws, wsb)
    return rc, _lib.lib().b2d_last_error().decode()


def test_debug_sums_argument_errors():
    for kw in ({"m": 0}, {"n": 0}, {"m": -1}):
        assert debug_call(**kw) == (E_ARG, "m and n must be positive")
    assert debug_call(m=2 ** 31) == (E_ARG, "mean_shift: m and n must be below 2^31")
    assert debug_call(d=0) == (E_ARG, "d must be positive")
    assert debug_call(d=321, ldx=321) == (E_UNS, "mean_shift supports d <= 320 (the whole distance at once)")
    for kw in ({"adj": None}, {"x": None}, {"part": None}, {"cnt": None}, {"e": None}, {"info": False}):
        assert debug_call(**kw) == (E_ARG, "null adj / x / part / counts / exponent / info")
    assert debug_call(ldx=7) == (E_ARG, "leading dimension smaller than d")
    msg = "adjacency pitch must be >= n and a multiple of 16, on a 16-byte boundary"
    for kw in ({"ld": 8}, {"ld": 24, "n": 20}, {"adj": P + 8}):
        assert debug_call(**kw) == (E_ARG, msg)
    assert debug_call(wsb=10)[0] == _lib.B2D_ERR_WORKSPACE
    assert debug_call(ws=None)[0] == _lib.B2D_ERR_WORKSPACE


# --------------------------------------------------------------------------------- CPU: the comparison's power
MUTATION_CASES = [(129, 4097, 97, 0.5), (64, 2049, 300, 0.3), (300, 2500, 40, 0.001)]


def mutants(adj, x):
    """the exact sums of each plausible kernel slip at (adj, x), as (name, part 2^-E, counts) in chunk_reference's form"""
    n, d = adj.shape[1], x.shape[1]
    S, _, cnt, _, E, _ = chunk_reference(adj, x)
    g, ng, _ = plan(d)
    nkb = (d + 31) // 32
    out = []
    sw = adj.clone()   # the two bytes of every pair (2h, 2h + 1) swapped
    sw[:, 0:n - n % 2:2], sw[:, 1:n - n % 2:2] = adj[:, 1:n - n % 2:2], adj[:, 0:n - n % 2:2]
    out.append(("adjacency pair swapped", chunk_reference(sw, x)[0], cnt))
    if nkb > 1:   # each k-block's columns from the k-block one group on (one k-block on with a single group)
        step = g if ng > 1 else 1
        pad = torch.nn.functional.pad(S, (0, nkb * 32 - d))
        src = [((c // 32 + step) % nkb) * 32 + c % 32 for c in range(d)]
        out.append(("k-block off by one group", pad[..., src], cnt))
    _, _, svec, _ = R.prep_scales(x.numpy())
    scale = 2.0 ** -np.log2(svec)   # 2^(e_j - E): the row's own power of two relative to E
    xs = x.numpy().astype(np.float64) * 2.0 ** E * scale[:, None]
    hi = xs.astype(np.float32).astype(np.float16).astype(np.float64) / (2.0 ** E * scale[:, None])
    out.append(("lo half dropped", chunk_reference(adj, torch.from_numpy(hi.astype(np.float32)))[0], cnt))
    dropped = S.clone()
    dropped[-1] = 0
    out.append(("last chunk's partial dropped", dropped, cnt))
    if cnt.shape[0] > 1:
        out.append(("counts of the next chunk", S, cnt.roll(1, 0)))
    return out, (S, cnt, E)


@pytest.mark.parametrize("m,n,d,density", MUTATION_CASES)
def test_bound_catches_kernel_slips(m, n, d, density):
    """every slip, applied exactly (no rounding error at all), falls outside the bound at the data of the GPU cases; the
    exact sums themselves pass"""
    rng = np.random.default_rng(m + n + d)
    x = torch.from_numpy(make_x(n, d, rng))
    adj = torch.from_numpy(make_adj(m, n, density, rng))
    ref = chunk_reference(adj, x)
    muts, (S, cnt, E) = mutants(adj, x)
    check_sums((S * 2.0 ** E).float(), cnt, E, ref)
    assert len(muts) >= 4
    for name, s_mut, c_mut in muts:
        with pytest.raises(AssertionError):
            check_sums((s_mut * 2.0 ** E).float(), c_mut, E, ref)
            pytest.fail("the bound accepts the slip: " + name)


# ---------------------------------------------------------------------------------------------- GPU: the sums
@pytest.mark.gpu
@pytest.mark.parametrize("d", SUM_D)
def test_sums_every_group_class(d):
    """two seed tiles (129 seeds), two chunks and a ragged third, a pitched x and adjacency with 0xff past n"""
    run_case(129, 2 * CHUNK + 77, d, 0.5, seed=d)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 127, 128, 2047, 2048, 2049, 4097, 40001])
def test_sums_chunk_edges(n):
    d = 33 if n % 2 else 129
    run_case(64, n, d, [0.5, 1e-3, 1.0][n % 3], seed=n)


@pytest.mark.gpu
@pytest.mark.parametrize("m", [1, 64, 127, 128, 129, 300])
def test_sums_tile_edges(m):
    run_case(m, CHUNK + 1, 97, 0.5, seed=m)


@pytest.mark.gpu
@pytest.mark.parametrize("density", [0.0, 1e-3, 0.5, 1.0])
def test_sums_densities(density):
    run_case(300, 2 * CHUNK + 1, 65, density, seed=int(density * 1000) + 1, extra=0, ldx_extra=0)


@pytest.mark.gpu
def test_sums_more_items_than_sms():
    _, _, info, _ = run_case(1000, 40000, 65, 0.05, seed=11)
    assert info[3] > info[4]   # every CTA takes several work items


@pytest.mark.gpu
def test_sums_refuse_adjacency_bytes_other_than_0_and_1():
    """a byte of 2 would enter A as fp16 2^15: the entry checks the bytes it reads (the 0xff past n are not read)"""
    rng = np.random.default_rng(1)
    adj = make_adj(8, 100, 0.5, rng, extra=12)
    adj[5, 99] = 2
    with pytest.raises(_lib.LogicError, match="adjacency bytes must be 0 or 1"):
        debug_sums(on_device(adj, 112), on_device(make_x(100, 8, rng), 8))


@pytest.mark.gpu
@pytest.mark.parametrize("d", [5, 70, 160])
def test_sums_scaled_rows(d):
    """a far outlier: the ordinary rows take their own exponent, with factors 2^(E - e_j) in (2^-24, 1)"""
    rng = np.random.default_rng(d)
    x = make_x(3000, d, rng)
    x[1234, d // 2] = 2.0 ** 17
    _, svec, own = R.prep_scales(x)[1:]
    assert own.sum() > 2900 and svec.min() > 2.0 ** -24
    _, _, info, _ = run_case(130, 3000, d, 0.3, seed=d, x=x)
    assert info[5] == 1


@pytest.mark.gpu
def test_sums_leave_out_rows_far_below_the_maximum():
    """Rows more than 2^24 below the data maximum: their factor 2^(E - e_j) is 0 in fp16, so the sums leave them out
    while the counts keep them.  A seed whose neighbours are all such rows gets sums of exactly 0 (a mean of 0); the
    others meet the bound against the sums without those rows."""
    rng = np.random.default_rng(5)
    n, d = 2500, 40
    x = make_x(n, d, rng)
    x[100:200] = (rng.normal(size=(100, d)) * 2.0 ** -20).astype(np.float32)   # the tiny cluster
    x[7] = 2.0 ** 10
    svec = R.prep_scales(x)[2]
    assert (svec[100:200] < 2.0 ** -24).all() and (svec[200:] >= 2.0 ** -24).all()
    adj = make_adj(64, n, 0.2, rng)
    adj[5] = 0
    adj[5, 100:200] = 1
    part, counts, _, _ = run_case(64, n, d, 0.0, seed=0, x=x, adj=adj)
    assert int(counts[0, 5]) == 100
    assert bool((part[:, 5] == 0).all())


@pytest.mark.gpu
def test_sums_skip_non_finite_rows():
    """NaN and +-inf elements in data rows of every chunk: the rows are cleared from the prepared data, so every other
    sum stays finite and equal to the sums without them (before, 0 * NaN put NaN into the column of every seed)"""
    rng = np.random.default_rng(9)
    n, d = 3 * CHUNK + 5, 70
    x = make_x(n, d, rng)
    bad = [3, 2047, 2048, 4500, n - 1]
    for r, (c, v) in zip(bad, [(0, np.nan), (33, np.inf), (69, -np.inf), (40, np.nan), (5, np.inf)]):
        x[r, c] = v
    adj = make_adj(200, n, 0.3, rng)
    adj[:, bad] = 0   # a non-finite row is adjacent to nothing (EPI_EPS)
    run_case(200, n, d, 0.0, seed=0, x=x, adj=adj)


# ----------------------------------------------------------------------------------------------- GPU: the fit
def abi_fit(x, h, seeds=None, max_iter=300, cluster_all=True, max_bytes=0):
    """b2d_mean_shift_fit on the device matrix x (the Python call refuses non-finite data): (centres, labels, n_iter)"""
    n, d = x.shape
    ns = 0 if seeds is None else seeds.shape[0]
    centers = torch.empty((max(ns, n), d), dtype=torch.float32, device="cuda")
    labels = torch.empty(n, dtype=torch.int32, device="cuda")
    out = torch.zeros(2, dtype=torch.int32, device="cuda")
    L = _lib.lib()
    ws = torch.empty(L.b2d_mean_shift_fit_workspace_bytes(n, d, ns, max_bytes), dtype=torch.uint8, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    _lib.check(L.b2d_mean_shift_fit(stream, x.data_ptr(), x.stride(0), n, d, h, None if seeds is None else
                                    seeds.data_ptr(), d, ns, 0, 1, int(cluster_all), max_iter, max_bytes,
                                    centers.data_ptr(), out.data_ptr(), labels.data_ptr(), out.data_ptr() + 4,
                                    ws.data_ptr(), ws.numel()))
    nc, it = (int(v) for v in out.cpu().tolist())
    return centers[:nc].cpu().numpy(), labels.cpu().numpy(), it


@pytest.mark.gpu
@pytest.mark.parametrize("d,n", [(2, 4800), (40, 4801), (96, 4816), (160, 4803)])
def test_single_step_many_seed_tiles_and_batches(d, n):
    """max_iter = 0 from 300 seeds 5h apart (two seed tiles and a ragged third; then two batches of 128 and a ragged
    one): every mean survives, in (count, coordinates) order, each within the one-step bound of the fp64 mean over
    eps_neighbors_l2sq's neighbourhood; every G class, with n % 16 == 0 (the adjacency's TMA store) and without"""
    from raft_b200.neighbors.epsilon_neighborhood import eps_neighbors_l2sq
    from test_mean_shift_gpu import gpu, grid, step_bound
    h, k = 1.0, 300
    rng = np.random.default_rng(d)
    centres = grid(k, d, 5.0 * h)
    x = (centres[rng.integers(0, k, n)] + rng.normal(size=(n, d)) * (0.8 * h / np.sqrt(d))).astype(np.float32)
    seeds = (centres + rng.normal(size=centres.shape) * (0.1 * h / np.sqrt(d))).astype(np.float32)
    adj, _ = eps_neighbors_l2sq(torch.from_numpy(seeds).cuda(), torch.from_numpy(x).cuda(), float(np.float32(h * h)))
    nb = torch.as_tensor(adj, device="cuda").cpu().numpy().astype(bool)
    cnt = nb.sum(1)
    assert (cnt > 0).all()
    ref = (nb.astype(np.float64) @ x.astype(np.float64)) / cnt[:, None]
    refk = ref.astype(np.float32)
    order = sorted(range(k), key=lambda i: (cnt[i], tuple(R.ordered_bits(refk[i]))), reverse=True)
    ld = round16(n)
    bound = step_bound(x, nb, ref)[order]
    for mb in (None, TILE * ld / 2 ** 20):   # all seeds in one batch (three tiles and a ragged one); batches of 128
        gc, _, gi = gpu(x, h, seeds=seeds, max_iter=0, max_mbytes_per_batch=mb)
        assert gi == 0 and gc.shape == seeds.shape
        err = np.abs(gc.astype(np.float64) - ref[order])
        assert (err <= bound).all(), err.max()


def suppression_data(pairs=130, h=1.0, d=3):
    """One big blob, then `pairs` triples of sub-blobs A, B, C on a line 0.9h apart (each of radius 0.03h), 5h from
    everything else.  Seeds at the centres of A and C see A + B and B + C; with |A| = 2, |C| = 1 and a heavy B their means
    lie within 0.4h of each other.  B's size falls with the triple, so the walk order is the blob, then A + B and B + C of
    each triple in turn: candidates 127 / 128 and 255 / 256 (the batch boundaries of 128) are a triple whose second is
    suppressed by its first, kept one batch earlier."""
    rng = np.random.default_rng(pairs)
    base = np.zeros((pairs + 1, d))
    base[:, 0] = 5.0 * h * (np.arange(pairs + 1) % 12)
    base[:, 1] = 5.0 * h * (np.arange(pairs + 1) // 12)
    rows, seeds = [], [base[0] + 0.1 * h]   # (off the blob's centre: its first shift is far from the stop threshold)
    rows.append(base[0] + ball(rng, 10 + 2 * pairs + 10, d, 0.03 * h))
    line = np.zeros(d)
    line[2 % d] = 0.9 * h
    for p in range(pairs):
        b = 4 + 2 * (pairs - p)
        o = base[p + 1]
        rows += [o + ball(rng, 2, d, 0.03 * h), o + line + ball(rng, b, d, 0.03 * h),
                 o + 2 * line + ball(rng, 1, d, 0.03 * h)]
        seeds += [o, o + 2 * line]
    x = np.concatenate(rows).astype(np.float32)
    return x, np.asarray(seeds, np.float32)


def ball(rng, k, d, r):
    v = rng.normal(size=(k, d))
    return v / np.linalg.norm(v, axis=1, keepdims=True) * r * rng.uniform(0, 1, (k, 1))


@pytest.mark.gpu
def test_fit_suppression_across_walk_batches():
    from test_mean_shift_gpu import check_fit
    x, seeds = suppression_data()
    assert len(seeds) > 2 * TILE
    ld = round16(len(x))
    gc, _, _ = check_fit(x, 1.0, seeds=seeds, max_iter=0, max_mbytes_per_batch=TILE * ld / 2 ** 20)
    assert len(gc) == 1 + 130   # one centre per triple: the B + C mean was suppressed in every one


@pytest.mark.gpu
@pytest.mark.parametrize("cluster_all", [True, False])
def test_fit_more_seeds_than_rows(cluster_all):
    """600 seeds on 150 rows: the adjacency pitch is the seeds' count, far past n"""
    from test_mean_shift_gpu import blobs, check_fit
    x = blobs(150, 4, 3, 1.0, seed=4)
    x = np.concatenate([x, np.full((3, 4), 30.0, np.float32)])   # rows far from every blob
    rng = np.random.default_rng(4)
    seeds = x[rng.integers(0, len(x) - 3, 600)] + np.float32(0.01)
    check_fit(x, 1.0, seeds=seeds, cluster_all=cluster_all)


@pytest.mark.gpu
def test_fit_non_finite_rows():
    """A row with a NaN or an infinity is within h of nothing: the fit on every row (those rows dropped as seeds) gives
    the model's result on the finite rows, with label -1 for the others; the Python call refuses such data"""
    from raft_b200.cluster import mean_shift
    from test_mean_shift_gpu import blobs, exact_model
    x = blobs(2 * CHUNK + 300, 6, 4, 1.0, seed=12)
    bad = np.array([0, 700, 2048, 3000, len(x) - 1])
    xb = x.copy()
    for r, v in zip(bad, [np.nan, np.inf, -np.inf, np.nan, np.inf]):
        xb[r, r % 6] = v
    good = np.setdiff1d(np.arange(len(x)), bad)
    (mc, ml, mi), gap = exact_model(x[good], 1.0)
    assert gap > 2.0 ** -14 * np.abs(x).max()
    gc, gl, gi = abi_fit(torch.from_numpy(xb).cuda(), 1.0)
    assert gi == mi and gc.shape == mc.shape
    assert (np.abs(gc.astype(np.float64) - mc) <= 2.0 ** -15 * np.abs(x).max() + 2.0 ** -23 * np.abs(mc)).all()
    assert (gl[good] == ml).all() and (gl[bad] == -1).all()
    with pytest.raises(ValueError, match="NaN or infinity"):
        mean_shift(torch.from_numpy(xb).cuda(), bandwidth=1.0)
