"""GPU tier: the fused 1-NN (b2d_fused_l2_nn / b2d_fused_distance_nn / b2d_fused_l2_nn_keys) on every search path,
against the fp64 arg-min over all n rows.

The call picks its arithmetic from the shape and from decisions taken on the device (nearest.cu: fused_nn_keys_chunk,
DESIGN.md section 2, K3b).  Every case below runs the C ABI with a workspace it owns, filled with 0xFF, reads the control
words of the screened search with b2d_debug_nn_stats afterwards and asserts the path it is named after before it looks
at the numbers:

    path          reached by                                            control words [overflow, go_screen, go_exact, redo]
    exact         k <= 64, n < 16384, nn_screen 0, 128 < k <= 320       not written (still 0xFFFFFFFF)
    screen        64 < k <= 128, n >= 16384, L2 or the cosine family    [0, 1, 0, 0]
    called_off    norms that dwarf the NN distances; nn_tau 0 + ties    [0, 0, 1, 0]
    overflow      nn_tau huge + a near-duplicate database               [!= 0, -, 1, -]
    redo          a row of y with its own exponent (L2)                 [-, 0, 1, 1]

A chunked call (n > 2^20) reports the words of its last screened chunk; when the remainder is shorter than 16384 rows it
takes the exact kernel, which writes none, so the words are those of the first chunk.

Checks, per row and with no count allowance (`check_bound`): for the returned (j, v) and the fp64 minimum at j*,
    d64(i, j) <= d64(i, j*) + eps(i, j) + eps(i, j*)      and      |v - d64(i, j)| <= eps(i, j),
eps as derived next to `eps_bound`.  Integer data, power-of-two copies and power-of-two scalings are exact in every
arithmetic of the search, so those cases compare bit for bit."""
import ctypes

import numpy as np
import pytest
import torch

import oracle
from oracle import DistanceType as DT
from raft_b200 import _lib

pytestmark = pytest.mark.gpu

L2, L2S, COS, CORR = DT.L2Expanded, DT.L2SqrtExpanded, DT.CosineExpanded, DT.CorrelationExpanded
FAM = (L2, COS, CORR)
CHUNK = 1 << 20
ULP = 2.0 ** -24
SENTINEL = (0x7FFFFFFF, np.finfo(np.float32).max)
UNWRITTEN = (0xFFFFFFFF,) * 7
NAME = {L2: "l2", L2S: "l2sqrt", COS: "cosine", CORR: "correlation"}
RATIO = {}            # path -> largest |v - d64(i, j)| / eps(i, j) seen


@pytest.fixture(scope="module", autouse=True)
def report_ratios():
    yield
    for path, r in sorted(RATIO.items()):
        print(f"\nmax |err| / eps on path {path}: {r:.3f}")


@pytest.fixture
def opts():
    """b2d_set_option for this test only: nn_tau = 6 and nn_screen = 1 are restored however the test ends."""
    L = _lib.lib()

    def set_(nn_tau=None, nn_screen=None):
        if nn_tau is not None:
            _lib.check(L.b2d_set_option(b"nn_tau", float(nn_tau)))
        if nn_screen is not None:
            _lib.check(L.b2d_set_option(b"nn_screen", float(nn_screen)))
    try:
        yield set_
    finally:
        L.b2d_set_option(b"nn_tau", 6.0)
        L.b2d_set_option(b"nn_screen", 1.0)


# ---------------------------------------------------------------------------------------------------------------------
# the call, its path, the oracle

def _ptr(t):
    return None if t is None else t.data_ptr()


def call(x, y, metric, *, xn=None, yn=None, out=None, init_out=1):
    """One fused 1-NN call on device fp32 operands (rows may be padded views: the pitch is the view's row stride).
    Returns (index, value, the 7 control words)."""
    L = _lib.lib()
    m, k = x.shape
    n = 0 if y is None else y.shape[0]
    nb = L.b2d_fused_l2_nn_workspace_bytes(m, n, k)
    ws = torch.full((nb,), 255, dtype=torch.uint8, device="cuda")
    if out is None:
        out = torch.empty((m, 2), dtype=torch.int32, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    ldx, ldy = x.stride(0), (k if y is None else y.stride(0))
    yp = None if y is None else y.data_ptr()
    if metric in (L2, L2S):
        rc = L.b2d_fused_l2_nn(s, out.data_ptr(), x.data_ptr(), ldx, yp, ldy, _ptr(xn), _ptr(yn), m, n, k,
                               int(metric == L2S), init_out, ws.data_ptr(), nb)
    else:
        rc = L.b2d_fused_distance_nn(s, out.data_ptr(), int(metric), x.data_ptr(), ldx, yp, ldy, None, None, m, n, k,
                                     init_out, ws.data_ptr(), nb)
    _lib.check(rc)
    st = (ctypes.c_uint * 7)()
    _lib.check(L.b2d_debug_nn_stats(s, ws.data_ptr(), m, n, k, st))
    torch.cuda.synchronize()
    return out[:, 0].cpu().numpy(), out[:, 1].contiguous().view(torch.float32).cpu().numpy(), tuple(st)


def assert_path(path, st):
    ovf, go_screen, go_exact, redo = st[1], st[2], st[3], st[4]
    if path == "exact":
        assert st == UNWRITTEN, f"expected the exact kernel alone, the screened search left {st}"
    elif path == "screen":
        assert (ovf, go_screen, go_exact, redo) == (0, 1, 0, 0), st
    elif path == "called_off":
        assert (ovf, go_screen, go_exact, redo) == (0, 0, 1, 0), st
    elif path == "overflow":
        assert ovf != 0 and go_exact == 1 and ovf != 0xFFFFFFFF, st
    elif path == "redo":
        assert (go_screen, go_exact, redo) == (0, 1, 1), st
    else:
        raise ValueError(path)


def d64(x, y, metric):
    """fp64 distance of row i of x to row i of y."""
    a, b = x.astype(np.float64), y.astype(np.float64)
    if metric in (L2, L2S):
        return ((a - b) ** 2).sum(1)
    if metric == CORR:
        a = a - a.mean(1, keepdims=True)
        b = b - b.mean(1, keepdims=True)
    with np.errstate(divide="ignore", invalid="ignore"):
        return 1.0 - (a * b).sum(1) / np.sqrt((a * a).sum(1) * (b * b).sum(1))


def ref_nn(x, y, metric, block=65536):
    """fp64 arg-min over all rows of y, ties -> smallest index (NaN distances never win), squared for the L2 family."""
    mt = L2 if metric in (L2, L2S) else metric
    m = x.shape[0]
    best_v, best_i = np.full(m, np.inf), np.zeros(m, np.int64)
    for j0 in range(0, y.shape[0], block):
        d = oracle.pairwise_distance(x, y[j0:j0 + block], mt)
        d[np.isnan(d)] = np.inf
        loc = d.argmin(1)
        v = d[np.arange(m), loc]
        upd = v < best_v
        best_v, best_i = np.where(upd, v, best_v), np.where(upd, loc + j0, best_i)
    return best_i, best_v


def eps_bound(x, yj, d, metric):
    """The error a path may make on d(i, j).
    L2: the expanded form d = |x|^2 + |y|^2 - 2 x.y (tensor cores, 3-term fp16 split with ~22 bits per operand, norms
    rounded once from fp64) errs by a few ulp of |x|^2 + |y|^2: 16 ulp.  Step E's direct sum (x - y)^2 rounds each
    difference and square (2 ulp) and each of k/32 + 5 partial sums of non-negative terms: (k/32 + 8) ulp of d.
    Cosine family: d = 1 - <x', y'> on unit rows, a few ulp of 1 for the tensor path, and E's fp64 value rounded once:
    16 ulp of 1 + |d|."""
    if metric in (L2, L2S):
        k = x.shape[1]
        nx, ny = (x.astype(np.float64) ** 2).sum(1), (yj.astype(np.float64) ** 2).sum(1)
        return 16 * ULP * (nx + ny) + (k / 32 + 8) * ULP * d
    return 16 * ULP * (1.0 + np.abs(d))


def check_bound(path, x, y, idx, val, metric, rows=None):
    """Every row (or `rows`): the returned neighbour is a true minimum up to eps, and its value is its distance up to
    eps."""
    rows = np.arange(x.shape[0]) if rows is None else rows
    x, idx, val = x[rows], idx[rows], val[rows]
    ri, rv = ref_nn(x, y, metric)
    assert np.all((idx >= 0) & (idx < y.shape[0])), idx
    dj = d64(x, y[idx], metric)
    ej, es = eps_bound(x, y[idx], dj, metric), eps_bound(x, y[ri], rv, metric)
    bad = np.nonzero(~(dj <= rv + ej + es))[0]
    assert len(bad) == 0, [(int(rows[i]), int(idx[i]), dj[i], int(ri[i]), rv[i]) for i in bad[:5]]
    err = np.abs(val.astype(np.float64) - dj)
    bad = np.nonzero(~(err <= ej))[0]
    assert len(bad) == 0, [(int(rows[i]), int(idx[i]), float(val[i]), dj[i], ej[i]) for i in bad[:5]]
    RATIO[path] = max(RATIO.get(path, 0.0), float((err / ej).max()))


def gpu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def packed_block(y):
    """The 256-row block of the norm-sorted chunk every row of y lands in on the screened L2 path: nn_sortkey_kernel's
    key (the top 24 bits of the fp32 squared norm; exact for integer data) and a stable sort."""
    key = (y.astype(np.float64) ** 2).sum(1).astype(np.float32).view(np.uint32) >> 8
    pos = np.empty(len(y), np.int64)
    pos[np.argsort(key, kind="stable")] = np.arange(len(y))
    return pos // 256


# ---------------------------------------------------------------------------------------------------------------------
# 1. every path against the fp64 bound

def data(kind, m, n, k, seed=0):
    rng = np.random.default_rng(100 + seed)
    if kind == "blobs":
        x, _, c = oracle.make_blobs(m, k, seed=77 + seed)
        y, _, _ = oracle.make_blobs(n, k, seed=99 + seed, centers=c)
        return x, y
    x = rng.standard_normal((m, k)).astype(np.float32) * 3
    y = (rng.standard_normal((n, k)) * 3 + 0.5).astype(np.float32)
    if kind == "offset":        # norms of ~1e3 * sqrt(k) against NN distances of ~sqrt(k): no screen margin is tight
        x += 1000.0
        y += 1000.0
    elif kind == "twins":       # every row of y twice: each incumbent of the trial has an equidistant twin
        y[1::2] = y[0::2]
    elif kind == "neardup":     # 20000 rows within 1e-4 of each other: every column is a candidate
        y = (1.0 + rng.standard_normal((n, k)) * 1e-4).astype(np.float32)
    elif kind == "y_outlier":   # a row of y with its own exponent
        y[n // 2] *= 1.0e9
    elif kind == "x_outlier":   # rows of x with their own exponents, y uniform: the screen scales those rows (xsc)
        x[3] *= 1.0e9
        x[4] *= 1.0e-6
        x[200] *= 1.0e-6
    return x, y


PATH_CASES = [
    # name                    m     n      k    data          metrics     path          options
    ("exact-resident-k64",    300, 20000,  64, "gauss",      FAM,        "exact",      {}),
    ("screen-k65",            300, 20000,  65, "blobs",      FAM,        "screen",     {}),
    ("screen-k96-gauss",      500, 40000,  96, "gauss",      FAM,        "screen",     {}),
    ("screen-k128",           300, 20000, 128, "blobs",      FAM,        "screen",     {}),
    ("exact-streaming-k129",  300, 20000, 129, "gauss",      FAM,        "exact",      {}),
    ("exact-streaming-k320",  200,  5000, 320, "gauss",      FAM,        "exact",      {}),
    ("exact-n16383",          300, 16383,  96, "gauss",      FAM,        "exact",      {}),
    ("screen-n16384",         300, 16384,  96, "gauss",      FAM,        "screen",     {}),
    ("exact-screen-off",      300, 20000,  96, "gauss",      FAM,        "exact",      {"nn_screen": 0}),
    ("called-off-offset",     300, 20000,  96, "offset",     (L2, COS),  "called_off", {}),
    ("called-off-tau0-ties",  300, 20000,  96, "twins",      FAM,        "called_off", {"nn_tau": 0}),
    ("overflow-neardup",      300, 20000,  96, "neardup",    (L2, COS),  "overflow",   {"nn_tau": 1e9}),
    ("redo-y-outlier",        300, 20000,  96, "y_outlier",  (L2,),      "redo",       {}),
    ("screen-x-outliers",     300, 20000,  96, "x_outlier",  (L2,),      "screen",     {}),
]


@pytest.mark.parametrize("case", PATH_CASES, ids=[c[0] for c in PATH_CASES])
def test_path_against_fp64(case, opts):
    name, m, n, k, kind, metrics, path, o = case
    opts(**o)
    x, y = data(kind, m, n, k, seed=len(name))
    xd, yd = gpu(x), gpu(y)
    for metric in metrics:
        idx, val, st = call(xd, yd, metric)
        assert_path(path, st)
        check_bound(path, x, y, idx, val, metric)
        if metric == L2:    # the sqrt output is sqrtf of the squared one, bit for bit, on the same path
            idx2, val2, st2 = call(xd, yd, L2S)
            assert_path(path, st2)
            assert np.array_equal(idx2, idx)
            if path == "overflow":
                # which finalists reach the list depends on the order of the screen's atomics, and a winner measured
                # by both E and X keeps the smaller of the two values: the last bit may differ from call to call
                check_bound(path, x, y, idx2, val2.astype(np.float64) ** 2, L2)
            else:
                assert np.array_equal(val2.view(np.uint32), np.sqrt(val).view(np.uint32))


@pytest.mark.parametrize("n", [CHUNK, CHUNK + 1, CHUNK + 5000, CHUNK + 20000])
@pytest.mark.parametrize("metric", [L2, COS], ids=NAME.get)
def test_chunked_database(n, metric):
    """n > 2^20: chunks of 2^20 rows, later chunks start from the keys (A skipped); a remainder below 16384 rows takes
    the exact kernel.  Neighbours planted on both sides of the chunk boundary must come back with global indices."""
    m, k = 64, 96
    g = torch.Generator(device="cuda").manual_seed(n)
    yd = torch.randn(n, k, device="cuda", generator=g) * 2 + 0.3
    targets = [5, CHUNK - 1, min(CHUNK, n - 1), n - 1, 700000]
    xd = torch.randn(m, k, device="cuda", generator=g) * 2 + 0.3
    xd[: len(targets)] = yd[targets] + 0.01 * torch.randn(len(targets), k, device="cuda", generator=g)
    idx, val, st = call(xd, yd, metric)
    assert_path("screen", st)
    x, y = xd.cpu().numpy(), yd.cpu().numpy()
    assert idx[: len(targets)].tolist() == targets
    check_bound("chunked", x, y, idx, val, metric)


def test_continued_keys_equal_single_call(opts):
    """b2d_fused_l2_nn_keys as the shards call it: the second shard continues from the first one's keys
    (init_keys = 0, idx_offset > 0, step A skipped); the finalised result is the single call's, bit for bit."""
    L = _lib.lib()
    x, y = data("gauss", 500, 40000, 96, seed=3)
    xd, yd = gpu(x), gpu(y)
    m, k = x.shape
    i1, v1, st1 = call(xd, yd, L2)
    assert_path("screen", st1)
    s = torch.cuda.current_stream().cuda_stream
    for cut in (16384, 20000):
        keys = torch.empty(m, dtype=torch.int64, device="cuda")
        kvp = torch.empty((m, 2), dtype=torch.int32, device="cuda")
        for lo, hi in ((0, cut), (cut, y.shape[0])):
            nb = L.b2d_fused_l2_nn_workspace_bytes(m, hi - lo, k)
            ws = torch.full((nb,), 255, dtype=torch.uint8, device="cuda")
            _lib.check(L.b2d_fused_l2_nn_keys(s, keys.data_ptr(), xd.data_ptr(), k, yd[lo:hi].data_ptr(), k, None, None,
                                              m, hi - lo, k, lo, 1 if lo == 0 else 0, ws.data_ptr(), nb))
            st = (ctypes.c_uint * 7)()
            _lib.check(L.b2d_debug_nn_stats(s, ws.data_ptr(), m, hi - lo, k, st))
            assert_path("screen", tuple(st))
        _lib.check(L.b2d_fused_l2_nn_finalize(s, kvp.data_ptr(), keys.data_ptr(), m, 0, ws.data_ptr(), nb))
        torch.cuda.synchronize()
        assert np.array_equal(kvp[:, 0].cpu().numpy(), i1)
        assert np.array_equal(kvp[:, 1].cpu().numpy().view(np.uint32), v1.view(np.uint32))


# ---------------------------------------------------------------------------------------------------------------------
# 2. exact arithmetic: bit for bit

def int_tie_data(n, k, seed):
    """Integers in [-3, 3] (k * 6^2 < 2^24: every path computes exact distances), and queries with planted ties:
    - `sparse`: q of norm <= 12 (packed block 0, a sampled block), rows q + s e_c and q - s e_c (s = sign q_c) at
      distance 1; the larger norm sits at the SMALLER source index, so the packed order is the reverse of the source order
    - `dense`: the same with an ordinary q (a block in the middle of the packed order: unsampled)
    - `copies`: a row written 200 times (consecutive in the packed order, across a block boundary), the query at
      distance 1 of it
    - `near`: a row plus e_c, distance 1 to one row."""
    rng = np.random.default_rng(seed)
    y = rng.integers(-3, 4, (n, k)).astype(np.float32)
    free = iter(rng.permutation(n).tolist())
    xs, expect, kinds = [], [], []

    def twin(q):
        c = int(np.flatnonzero(q)[rng.integers(0, np.count_nonzero(q))])
        e = np.zeros(k, np.float32)
        e[c] = np.sign(q[c])
        p1, p2 = sorted((next(free), next(free)))
        y[p1], y[p2] = q + e, q - e       # |q + e|^2 = |q - e|^2 + 4 |q_c|
        return p1

    for _ in range(12):
        q = np.zeros(k, np.float32)
        q[rng.choice(k, 3, replace=False)] = rng.choice([-2, -1, 1, 2], 3)
        expect.append(twin(q)); xs.append(q); kinds.append("sparse")
    for _ in range(12):
        q = rng.integers(-3, 4, k).astype(np.float32)
        q[0] = rng.choice([-2, -1, 1, 2])
        expect.append(twin(q)); xs.append(q); kinds.append("dense")
    for _ in range(3):
        pos = sorted(next(free) for _ in range(200))
        y[pos] = y[pos[-1]]
        q = y[pos[0]].copy()
        q[rng.integers(0, k)] += 0.5     # distance 0.25 (exact): no other row comes near
        expect.append(pos[0]); xs.append(q); kinds.append("copies")
    for _ in range(13):
        t = next(free)
        q = y[t].copy()
        q[rng.integers(0, k)] += 1.0
        expect.append(t); xs.append(q); kinds.append("near")
    return np.stack(xs), y, np.array(expect), np.array(kinds)


INT_RUNS = [  # name, k, options, path
    ("screen", 96, {}, "screen"),
    ("exact-screen-off", 96, {"nn_screen": 0}, "exact"),
    ("called-off-tau0", 96, {"nn_tau": 0}, "called_off"),
    ("exact-streaming-k129", 129, {}, "exact"),
]


@pytest.mark.parametrize("run", INT_RUNS, ids=[r[0] for r in INT_RUNS])
def test_integer_data_exact_with_ties(run, opts):
    name, k, o, path = run
    x, y, expect, kinds = int_tie_data(20000, k, seed=k)
    ri, rv = ref_nn(x, y, L2)
    assert np.array_equal(ri, expect)    # the planted ties are the true minima
    blk = packed_block(y)
    tw = np.array([e for e, kd in zip(expect, kinds) if kd in ("sparse", "dense")])
    assert (blk[tw] % 32 == 0).any() and (blk[tw] % 32 != 0).any()   # ties in sampled and in unsampled blocks
    opts(**o)
    xd, yd = gpu(x), gpu(y)
    idx, val, st = call(xd, yd, L2)
    assert_path(path, st)
    assert np.array_equal(idx, ri)
    assert np.array_equal(val.astype(np.float64), rv)
    idx2, val2, _ = call(xd, yd, L2S)
    assert np.array_equal(idx2, ri)
    assert np.array_equal(val2.view(np.uint32), np.sqrt(rv.astype(np.float32)).view(np.uint32))


def test_integer_data_exact_across_chunk_boundary():
    """2^20 + 20000 integer rows: equidistant rows with different norms on both sides of the boundary (the smaller
    index in the first chunk), copies of a row at 2^20 - 1, 2^20 and n - 1, planted neighbours in the second chunk."""
    n, k, m = CHUNK + 20000, 96, 24
    g = torch.Generator(device="cuda").manual_seed(7)
    yd = torch.randint(-3, 4, (n, k), device="cuda", generator=g).float()
    xd = torch.randint(-3, 4, (m, k), device="cuda", generator=g).float()
    e = torch.zeros(k, device="cuda")
    e[0] = 1.0
    xd[0, 0] = 2.0
    yd[CHUNK - 3], yd[CHUNK + 7] = xd[0] + e, xd[0] - e          # |x+e|^2 > |x-e|^2: larger norm, smaller index
    xd[1, 0] = -1.0
    yd[CHUNK + 9], yd[CHUNK - 2] = xd[1] + e, xd[1] - e          # the same the other way round
    yd[[CHUNK - 1, CHUNK, n - 1]] = yd[CHUNK + 100].clone()
    xd[2] = yd[CHUNK + 100]
    xd[2, 5] += 0.5
    for i, t in enumerate((CHUNK + 11, CHUNK + 300, n - 2, 17, CHUNK - 5), start=3):
        xd[i] = yd[t]
        xd[i, i] += 1.0
    idx, val, st = call(xd, yd, L2)
    assert_path("screen", st)
    x, y = xd.cpu().numpy(), yd.cpu().numpy()
    ri, rv = ref_nn(x, y, L2)
    assert ri[:8].tolist() == [CHUNK - 3, CHUNK - 2, CHUNK - 1, CHUNK + 11, CHUNK + 300, n - 2, 17, CHUNK - 5]
    assert np.array_equal(idx, ri)
    assert np.array_equal(val.astype(np.float64), rv)


@pytest.mark.parametrize("metric", [COS, CORR], ids=NAME.get)
@pytest.mark.parametrize("path", ["screen", "exact"])
def test_power_of_two_copies_tie_to_smallest_index(metric, path, opts):
    """2^p y_r (p = -3..3) has exactly the distance of y_r in every arithmetic of the cosine family: copies spread over
    sampled (block % 32 == 0) and unsampled 256-row blocks; the smallest index must win."""
    opts(nn_screen=1 if path == "screen" else 0)
    rng = np.random.default_rng(17)
    n, k, m = 20000, 96, 64
    y = (rng.standard_normal((n, k)) + 0.3).astype(np.float32)
    x = (rng.standard_normal((m, k)) + 0.3).astype(np.float32)
    in_sampled = [3, 8200, 8300, 16400, 200, 120, 16390, 8195]     # blocks 0, 32 and 64
    free = iter(rng.permutation(np.setdiff1d(np.arange(300, n), in_sampled)).tolist())
    sampled = iter(in_sampled)
    expect = {}
    for i in range(8):
        # 7 places per row of copies, one in a sampled block for every other row; the original row is the last
        pos = [next(sampled) if (i % 2 == 0 and p == i % 7) else next(free) for p in range(7)]
        base = y[pos[-1]].copy()
        for p, j in zip(range(-3, 4), pos):
            y[j] = base * np.float32(2.0 ** p)
        x[i] = base + 0.05 * rng.standard_normal(k).astype(np.float32)
        expect[i] = min(pos)
    ri, _ = ref_nn(x, y, metric)
    assert all(ri[i] == e for i, e in expect.items())
    idx, val, st = call(gpu(x), gpu(y), metric)
    assert_path(path, st)
    assert all(idx[i] == e for i, e in expect.items()), (idx[:8], expect)
    check_bound(path, x, y, idx, val, metric)


# ---------------------------------------------------------------------------------------------------------------------
# 3. scaling law: bit for bit, every path

@pytest.mark.parametrize("path", ["screen", "exact"])
def test_l2_scaling_law(path, opts):
    """Scaling x and y by the same 2^s scales every distance by 2^2s exactly (no fast math, everything stays normal):
    the indices must not move and every value must be the unscaled one times 2^2s (2^s with sqrt)."""
    opts(nn_screen=1 if path == "screen" else 0)
    x, y = data("gauss", 300, 20000, 96, seed=8)
    xd, yd = gpu(x), gpu(y)
    i0, v0, st = call(xd, yd, L2)
    assert_path(path, st)
    check_bound(path, x, y, i0, v0, L2)
    for s in (-50, -20, 20, 50):
        f = 2.0 ** s
        i1, v1, st1 = call(xd * f, yd * f, L2)
        assert_path(path, st1)
        assert np.array_equal(i1, i0), s
        assert np.array_equal(v1.view(np.uint32), (v0 * np.float32(f * f)).view(np.uint32)), s
        i2, v2, _ = call(xd * f, yd * f, L2S)
        assert np.array_equal(i2, i0), s
        assert np.array_equal(v2.view(np.uint32), (np.sqrt(v0) * np.float32(f)).view(np.uint32)), s


@pytest.mark.parametrize("metric", [COS, CORR], ids=NAME.get)
@pytest.mark.parametrize("path", ["screen", "exact"])
def test_cosine_family_scaling_law(metric, path, opts):
    """The cosine family does not depend on the scale of either operand: x * 2^s against y * 2^t, s and t independently
    in {-60, -30, 0, 30, 60}, must give the unscaled output bit for bit."""
    opts(nn_screen=1 if path == "screen" else 0)
    rng = np.random.default_rng(23)
    x = (rng.standard_normal((300, 96)) + 0.3).astype(np.float32)
    y = (rng.standard_normal((20000, 96)) + 0.3).astype(np.float32)
    xd, yd = gpu(x), gpu(y)
    i0, v0, st = call(xd, yd, metric)
    assert_path(path, st)
    check_bound(path, x, y, i0, v0, metric)
    for s in (-60, -30, 0, 30, 60):
        for t in (-60, -30, 0, 30, 60):
            i1, v1, st1 = call(xd * 2.0 ** s, yd * 2.0 ** t, metric)
            assert_path(path, st1)
            bad = np.nonzero((i1 != i0) | (v1.view(np.uint32) != v0.view(np.uint32)))[0]
            assert len(bad) == 0, (s, t, len(bad), [(int(i0[r]), float(v0[r]), int(i1[r]), float(v1[r])) for r in bad[:3]])


# ---------------------------------------------------------------------------------------------------------------------
# 4. ABI details, on the screened path and on an exact one

ABI_PATHS = ["screen", "exact"]


def _abi_data(path, opts, seed=31):
    opts(nn_screen=1 if path == "screen" else 0)
    return data("gauss", 300, 20000, 97, seed=seed)


def padded(a, ld, off):
    """a on the device with row pitch ld and its first element `off` floats behind an allocation boundary (off = 1:
    only 4-byte aligned); the padding holds a finite junk value."""
    r, c = a.shape
    buf = torch.full((off + r * ld,), 777.0, device="cuda")
    v = buf[off:].view(r, ld)[:, :c]
    v.copy_(torch.from_numpy(a))
    return v


@pytest.mark.parametrize("path", ABI_PATHS)
@pytest.mark.parametrize("metric", [L2, COS], ids=NAME.get)
def test_padded_pitch_and_unaligned_base(path, metric, opts):
    x, y = _abi_data(path, opts)
    i0, v0, st0 = call(gpu(x), gpu(y), metric)
    i1, v1, st1 = call(padded(x, 101, 0), padded(y, 101, 1), metric)
    assert_path(path, st0)
    assert_path(path, st1)
    assert np.array_equal(i1, i0) and np.array_equal(v1.view(np.uint32), v0.view(np.uint32))


@pytest.mark.parametrize("path", ABI_PATHS)
def test_precomputed_norms_bit_identical(path, opts):
    """b2d_row_norm sums the squares in fp64 in the order prep does and rounds once, so caller norms change no bit."""
    L = _lib.lib()
    x, y = _abi_data(path, opts)
    xd, yd = gpu(x), gpu(y)
    xn, yn = torch.empty(x.shape[0], device="cuda"), torch.empty(y.shape[0], device="cuda")
    for t, nrm in ((xd, xn), (yd, yn)):
        _lib.check(L.b2d_row_norm(None, nrm.data_ptr(), t.data_ptr(), t.shape[1], t.shape[0], t.shape[1], 2, 0))
    i0, v0, st0 = call(xd, yd, L2)
    i1, v1, st1 = call(xd, yd, L2, xn=xn, yn=yn)
    assert_path(path, st0)
    assert_path(path, st1)
    assert np.array_equal(i1, i0) and np.array_equal(v1.view(np.uint32), v0.view(np.uint32))


@pytest.mark.parametrize("path", ABI_PATHS)
@pytest.mark.parametrize("metric", [L2, COS], ids=NAME.get)
def test_init_out_false_merges_by_argmin_op(path, metric, opts):
    """init_out = 0 reduces into the caller's values: smaller value kept; equal value -> smaller index."""
    x, y = _abi_data(path, opts)
    xd, yd = gpu(x), gpu(y)
    i0, v0, _ = call(xd, yd, metric)
    m = len(i0)
    r = np.arange(m) % 4
    ei = np.where(r == 1, i0 - 1, i0 + 1).astype(np.int32)
    ei[(r == 1) & (i0 == 0)] = 0
    ev = np.where(r == 0, v0 * np.float32(0.5), np.where(r == 3, v0 * np.float32(2) + np.float32(1), v0)).astype(np.float32)
    out = torch.from_numpy(np.stack([ei, ev.view(np.int32)], 1)).cuda()
    i1, v1, st = call(xd, yd, metric, out=out, init_out=0)
    assert_path(path, st)
    keep = (ev < v0) | ((ev == v0) & (ei < i0))
    assert keep[r == 0].all() and not keep[r >= 2].any()
    assert np.array_equal(i1, np.where(keep, ei, i0))
    assert np.array_equal(v1.view(np.uint32), np.where(keep, ev, v0).view(np.uint32))


@pytest.mark.parametrize("k", [64, 96, 200])
@pytest.mark.parametrize("metric", [L2, L2S, COS, CORR], ids=NAME.get)
def test_empty_database_gives_sentinel(k, metric):
    i, v, st = call(torch.randn(37, k, device="cuda"), None, metric)
    assert st == UNWRITTEN
    assert (i == SENTINEL[0]).all() and (v == SENTINEL[1]).all()


@pytest.mark.parametrize("metric", [L2, COS, CORR], ids=["l2", "cosine", "correlation"])
def test_degenerate_rows_same_on_every_path(metric, opts):
    """A NaN query row, a zero row (cosine: 0/0) and a constant row (correlation: zero after centring) have only NaN
    distances: no candidate ever passes the arg-min's comparison, so every path returns the empty-row sentinel.  The
    other rows get exactly what they get without them.  A NaN row of y, planted where it would otherwise be the
    nearest, never wins."""
    x, y = data("gauss", 300, 20000, 96, seed=41)
    j0 = 1234
    x[0] = y[j0] + 0.01
    y_nan = y.copy()
    y_nan[j0] = np.nan
    y_far = y.copy()
    y_far[j0] = -1000.0 * x[0]     # what the oracle sees instead of the NaN row: far from every query in every metric
    rows = [5, 6, 7]
    xb = x.copy()
    xb[5] = np.nan
    xb[6] = 0.0
    xb[7] = 2.5
    nan_rows = {L2: [5], COS: [5, 6], CORR: [5, 6, 7]}[metric]    # the rows whose every distance is NaN
    ok = np.setdiff1d(np.arange(len(x)), rows)
    for path in ("screen", "exact"):
        opts(nn_screen=1 if path == "screen" else 0)
        ib, vb, st = call(gpu(xb), gpu(y_nan), metric)
        assert_path(path, st)
        assert (ib[nan_rows] == SENTINEL[0]).all() and (vb[nan_rows] == SENTINEL[1]).all(), (path, ib[rows], vb[rows])
        ic, vc, _ = call(gpu(x[ok]), gpu(y_nan), metric)
        assert np.array_equal(ib[ok], ic) and np.array_equal(vb[ok].view(np.uint32), vc.view(np.uint32)), path
        assert ib[0] != j0 and np.isfinite(vb[0])
        check_bound(path, x[ok], y_far, ic, vc, metric)
        real = np.setdiff1d(rows, nan_rows)    # ordinary rows under this metric
        if len(real):
            check_bound(path, xb[real], y_far, ib[real], vb[real], metric)
