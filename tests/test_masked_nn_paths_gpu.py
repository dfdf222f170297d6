"""GPU tier: masked_l2_nn (b2d_masked_l2_nn, the fused L2 1-NN under a row x group adjacency mask) on every tile class,
kernel variant and operand edge, against the fp64 masked arg-min (masked_nn_ref.py).

Every call goes through the C ABI with a workspace it owns, filled with 0xFF (`call`).  The masked path is always the
exact tensor kernel (DESIGN.md section 2, K3m): resident for k <= 128, streaming for 128 < k <= 320, and streaming with
more k-blocks per half than the ring has stages beyond that.

Checks, per row and with no count allowance (`check`): a row without an adjacent candidate gets exactly
{0x7fffffff, FLT_MAX}; otherwise, for the returned (j, v) and the reference's arg-min j* over the adjacent columns,
    j is adjacent to i,   d64(i, j) is finite,   d64(i, j) <= d64(i, j*) + hi(i, j*) + lo(i, j),
    -lo(i, j) <= v - d64(i, j) <= hi(i, j),
with S = |x_i|^2 + |y_j|^2 and, in ulp (2^-24) of S,
    hi = 16 + k/8, lo = 16     where x_i.y_j >= 0,       hi = 16, lo = 16 + k/8     where x_i.y_j < 0.
16 ulp is the expanded form |x|^2 + |y|^2 - 2 x.y (3-term fp16 split, norms rounded once from fp64).  The k term is the
hi.hi accumulator, which holds x.y (up to S/2) and loses the bits of every product below its exponent: the tensor core
aligns and truncates toward zero (DESIGN.md section 3, "Accumulator behaviour"), so |x.y| comes out too small and v errs
toward the sign of x.y, never the other way by more than the 16 ulp.  On blobs, whose x.y is close to S/2, that term
measures about k/12 ulp of S, so 16 ulp alone fails from k ~ 190 on.  The sqrt output is sqrtf of the squared one, bit
for bit.

Bit-exact laws, no tolerance: a mask of ALL tiles is exact fusedL2NN; masked(A | B) is masked(A) merged with masked(B)
through init_out = 0; integer data is the reference, tie order included; 2^s x, 2^s y scale every value by 2^2s; caller
norms from b2d_row_norm change no bit."""
import numpy as np
import pytest
import torch

import oracle
from masked_nn_ref import FLT_MAX, NO_CANDIDATE, column_groups, masked_l2_nn as ref_masked_l2_nn, tile_classes
from raft_b200 import _lib
from raft_b200.distance import masked_l2_nn

pytestmark = pytest.mark.gpu

ULP = 2.0 ** -24
FLT_MAX_BITS = 0x7F7FFFFF
POISON = (0x7FFFFFFF, 0x7FFFFFFF)       # {key, value bits} of every row after an invalid group_idxs: {0x7fffffff, NaN}
RATIO = {}                               # kernel variant (and side) -> largest |v - d64(i, j)| / its bound seen

# resident (k <= 128), streaming (128 < k <= 320), streaming past the ring (k > 320)
KS = [1, 2, 31, 32, 33, 64, 127, 128, 129, 192, 193, 320, 321, 784]
KS_REGIMES = [32, 128, 200, 784]
# m: below 32, 33, m % 128 in {1, 63, 64, 65, 127};  n: 1, below 128, n % 256 in {1, 127, 128, 129, 255}.  The last
# shape has 16 x tiles and 18 y blocks: 288 work items, more than one per CTA
SHAPES = [(17, 1), (33, 100), (129, 257), (191, 383), (192, 384), (193, 385), (255, 511), (1985, 4353)]
PATTERNS = ["all", "none", "0.1", "0.5", "cc", "slab"]


@pytest.fixture(scope="module", autouse=True)
def report_ratio():
    yield
    for variant, r in sorted(RATIO.items()):
        print(f"\nmasked_l2_nn {variant}: max |err| / bound = {r:.3f}")


@pytest.fixture
def exact_fused():
    """nn_screen = 0 (fused_l2_nn on the exact kernel) for this test only, restored however it ends."""
    L = _lib.lib()
    _lib.check(L.b2d_set_option(b"nn_screen", 0.0))
    try:
        yield
    finally:
        L.b2d_set_option(b"nn_screen", 1.0)


# ---------------------------------------------------------------------------------------------------------------------
# the call, the data, the check

def _ptr(t):
    return None if t is None else t.data_ptr()


def call(x, y, adj, gidx, *, G=None, ldx=None, ldy=None, ld_adj=None, xn=None, yn=None, sqrt=False, out=None,
         init_out=1, ws=None):
    """One b2d_masked_l2_nn call on device operands: x [m, k] and y [n, k] fp32 (views; the pitches default to their row
    strides), adj uint8 [m, >= G] (the pitch defaults to its row stride), gidx int32 [G].  The workspace is a fresh one
    filled with 0xFF unless `ws` is given.  Returns out, the [m, 2] int32 {key, value bits} tensor."""
    L = _lib.lib()
    m, k = x.shape
    n = 0 if y is None else y.shape[0]
    G = (0 if gidx is None else gidx.numel()) if G is None else G
    ldx = x.stride(0) if ldx is None else ldx
    ldy = (k if y is None else y.stride(0)) if ldy is None else ldy
    ld_adj = (G if adj is None else adj.stride(0)) if ld_adj is None else ld_adj
    nb = L.b2d_masked_l2_nn_workspace_bytes(m, n, k, G)
    if ws is None:
        ws = torch.full((nb,), 255, dtype=torch.uint8, device="cuda")
    if out is None:
        out = torch.empty((m, 2), dtype=torch.int32, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    _lib.check(L.b2d_masked_l2_nn(s, out.data_ptr(), x.data_ptr(), ldx, _ptr(y), ldy, _ptr(xn), _ptr(yn), _ptr(adj),
                                  ld_adj, _ptr(gidx), G, m, n, k, int(sqrt), init_out, ws.data_ptr(), nb))
    return out


def host(out):
    """(index int32 [m], value fp32 [m]) of an out tensor."""
    torch.cuda.synchronize()
    o = out.cpu().numpy()
    return o[:, 0].copy(), o[:, 1].copy().view(np.float32)


def gpu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def data(kind, m, n, k, seed=0):
    """The blobs and gauss data of the fused 1-NN suite."""
    if kind == "blobs":
        x, _, c = oracle.make_blobs(m, k, seed=77 + seed)
        y, _, _ = oracle.make_blobs(n, k, seed=99 + seed, centers=c)
        return x, y
    rng = np.random.default_rng(100 + seed)
    x = rng.standard_normal((m, k)).astype(np.float32) * 3
    y = (rng.standard_normal((n, k)) * 3 + 0.5).astype(np.float32)
    return x, y


def groups(n, rng, tail=True):
    """group_idxs with every kind of edge: group_idxs[0] = 0 and consecutive empty groups, single-row groups, groups
    ending anywhere inside a 128-row half or a 256-row block, and (tail) rows of y after the last end."""
    limit = n - int(rng.integers(1, max(2, n // 8 + 1))) if tail and n > 1 else n
    ends = [0, 0]
    while ends[-1] < limit:
        size = int(rng.choice([0, 0, 1, 1, int(rng.integers(2, 64)), int(rng.integers(64, 300))]))
        ends.append(min(ends[-1] + size, limit))
    ends += [limit, limit]
    return np.array(ends, dtype=np.int32)


def adjacency(kind, m, G, rng):
    """[m, G] bool: all, none, random with p, connect_components (every group but the row's own colour) or sparse slabs
    (every 64-row slab of x adjacent to the same few groups: whole NONE and ALL tiles)."""
    if kind == "all":
        return np.ones((m, G), bool)
    if kind == "none":
        return np.zeros((m, G), bool)
    if kind == "cc":
        a = np.ones((m, G), bool)
        a[np.arange(m), rng.integers(0, G, size=m)] = False
        return a
    if kind == "slab":
        a = np.zeros((m, G), bool)
        for s in range(0, m, 64):
            a[s:s + 64, rng.random(G) < 0.25] = True
        return a
    return rng.random((m, G)) < float(kind)


def device_adj(adj, rng, pad=5):
    """adj as the bytes a caller may pass: every adjacent entry one of 1, 2, 0x80, 0xFF, and a pitch of G + pad whose
    padding holds 1s (beyond num_groups: never read)."""
    m, G = adj.shape
    b = np.ones((m, G + pad), np.uint8)
    b[:, :G] = np.where(adj, rng.choice(np.array([1, 2, 0x80, 0xFF], np.uint8), size=adj.shape), 0)
    return gpu(b)


def d64(x, y):
    """fp64 squared distance of row i of x to row i of y."""
    return ((x.astype(np.float64) - y.astype(np.float64)) ** 2).sum(1)


def bounds(x, y, dnorm=0.0):
    """(lo, hi): how far below and above d(i, j) the masked kernel's value may lie, per row i of x and y (module
    docstring).  dnorm: the error of caller norms, |xn_i - |x_i|^2| + |yn_j - |y_j|^2|, enters both sides."""
    a, b = x.astype(np.float64), y.astype(np.float64)
    s = ULP * ((a * a).sum(1) + (b * b).sum(1))
    acc = (16 + x.shape[1] / 8) * s
    pos = (a * b).sum(1) >= 0
    return np.where(pos, 16 * s, acc) + dnorm, np.where(pos, acc, 16 * s) + dnorm


def variant(k):
    return "resident" if k <= 128 else "streaming" if k <= 320 else "streaming k > 320"


def check(x, y, adj, gidx, idx, val, rows=None, xn=None, yn=None):
    """Every row (or `rows`) of a squared call against the fp64 masked arg-min, as in the module docstring.  xn / yn:
    the squared norms the caller passed (fp32), whose error widens the bounds."""
    rows = np.arange(x.shape[0]) if rows is None else np.asarray(rows)
    x, adj, idx, val = x[rows], (np.asarray(adj) != 0)[rows], idx[rows], val[rows]
    dxn = np.zeros(len(rows)) if xn is None else np.abs(np.float64(1) * xn[rows] - (x.astype(np.float64) ** 2).sum(1))
    dyn = np.zeros(len(y)) if yn is None else np.abs(np.float64(1) * yn - (y.astype(np.float64) ** 2).sum(1))
    ri, _ = ref_masked_l2_nn(x, y, adj, gidx)
    none = ri == NO_CANDIDATE
    bad = np.nonzero(none & ((idx != NO_CANDIDATE) | (val.view(np.uint32) != FLT_MAX_BITS)))[0]
    assert len(bad) == 0, [(int(rows[i]), int(idx[i]), float(val[i])) for i in bad[:5]]
    live = np.nonzero(~none)[0]
    if len(live) == 0:
        return
    j, js = idx[live].astype(np.int64), ri[live].astype(np.int64)
    assert np.all((j >= 0) & (j < y.shape[0])), [(int(rows[i]), int(idx[i])) for i in live[(j < 0) | (j >= len(y))][:5]]
    grp = column_groups(gidx, y.shape[0])
    ok = (grp[j] >= 0) & adj[live, np.maximum(grp[j], 0)]
    assert ok.all(), [(int(rows[live[i]]), int(j[i]), int(grp[j[i]])) for i in np.nonzero(~ok)[0][:5]]
    xl = x[live]
    dj, ds = d64(xl, y[j]), d64(xl, y[js])
    bad = np.nonzero(~np.isfinite(dj))[0]                  # an Inf row of y: the bounds below would read inf <= inf
    assert len(bad) == 0, [(int(rows[live[i]]), int(j[i]), float(val[live[i]])) for i in bad[:5]]
    lo_j, hi_j = bounds(xl, y[j], dxn[live] + dyn[j])
    _, hi_s = bounds(xl, y[js], dxn[live] + dyn[js])
    bad = np.nonzero(~(dj <= ds + hi_s + lo_j))[0]
    assert len(bad) == 0, [(int(rows[live[i]]), int(j[i]), dj[i], int(js[i]), ds[i]) for i in bad[:5]]
    err = val[live].astype(np.float64) - dj
    bad = np.nonzero(~((-lo_j <= err) & (err <= hi_j)))[0]
    assert len(bad) == 0, [(int(rows[live[i]]), int(j[i]), float(val[live[i]]), dj[i], -lo_j[i], hi_j[i])
                           for i in bad[:5]]
    side = np.where(err >= 0, hi_j, lo_j)
    ratio = np.abs(err) / np.where(side > 0, side, np.inf)
    with_sign = (err >= 0) == ((xl.astype(np.float64) * y[j].astype(np.float64)).sum(1) >= 0)
    v = variant(x.shape[1])
    for key, r in ((v, ratio[with_sign]), (v + ", against the sign of x.y (bound 16 ulp)", ratio[~with_sign])):
        RATIO[key] = max(RATIO.get(key, 0.0), float(r.max(initial=0.0)))


def assert_sqrt_law(idx, val, idx2, val2):
    """The sqrt call: the same indices, values sqrtf of the squared ones bit for bit (FLT_MAX on rows without one)."""
    assert np.array_equal(idx2, idx)
    want = np.where(idx == NO_CANDIDATE, np.float32(FLT_MAX), np.sqrt(val))
    assert np.array_equal(val2.view(np.uint32), want.view(np.uint32))


def assert_same(a, b, what=""):
    ia, va = a
    ib, vb = b
    bad = np.nonzero((ia != ib) | (va.view(np.uint32) != vb.view(np.uint32)))[0]
    assert len(bad) == 0, (what, len(bad), [(int(r), int(ia[r]), float(va[r]), int(ib[r]), float(vb[r])) for r in bad[:5]])


def run_checked(x, y, adj, gidx, rng, xd=None, yd=None):
    """The squared and the sqrt call with caller-style adjacency bytes, both checked.  Returns (idx, val)."""
    xd = gpu(x) if xd is None else xd
    yd = gpu(y) if yd is None else yd
    ad, gd = device_adj(adj, rng), gpu(gidx)
    idx, val = host(call(xd, yd, ad, gd))
    check(x, y, adj, gidx, idx, val)
    assert_sqrt_law(idx, val, *host(call(xd, yd, ad, gd, sqrt=True)))
    return idx, val


# ---------------------------------------------------------------------------------------------------------------------
# 1. every k regime, shape edge, group layout and adjacency pattern against the fp64 bound

@pytest.mark.parametrize("shape", SHAPES, ids=[f"m{m}-n{n}" for m, n in SHAPES])
@pytest.mark.parametrize("k", KS)
def test_against_fp64(k, shape):
    m, n = shape
    rng = np.random.default_rng(k * 1000 + m + n)
    for kind in ("blobs", "gauss"):
        x, y = data(kind, m, n, k, seed=k + m)
        xd, yd = gpu(x), gpu(y)
        gidx = groups(n, rng, tail=(kind == "gauss"))
        for pat in PATTERNS:
            run_checked(x, y, adjacency(pat, m, len(gidx), rng), gidx, rng, xd, yd)


def test_tile_classes_are_reached():
    """The cases above reach NONE, ALL and PARTIAL tiles at the larger shape."""
    m, n = SHAPES[-1]
    rng = np.random.default_rng(3)
    seen = set()
    gidx = groups(n, rng)
    for pat in PATTERNS:
        seen |= set(np.unique(tile_classes(adjacency(pat, m, len(gidx), rng), gidx, m, n)).tolist())
    assert seen == {0, 1, 2}


@pytest.mark.parametrize("k", KS_REGIMES + [33])
def test_special_rows(k):
    """Outlier rows of x (x 1e9, x 1e-6) and of y (x 1e9), NaN and zero rows of x, NaN and Inf rows of y, under masks
    where each is adjacent to some rows and not to others; an Inf or NaN row never wins, a NaN row of x has no
    candidate, and a NaN row of y does not hide the minimum of its block."""
    rng = np.random.default_rng(k)
    m, n = 300, 1100
    x, y = data("gauss", m, n, k, seed=k)
    gidx = groups(n, rng)
    x[3] *= 1.0e9
    x[4] *= 1.0e-6
    x[200] *= 1.0e-6
    x[5] = np.nan
    x[250] = np.nan
    x[6] = 0.0
    y[[10, 700]] *= 1.0e9
    y[[11, 300, 301, 800]] = np.nan
    y[[12, 500]] = np.inf
    y[600] = 0.0
    x[20:40] = y[302] + 0.01                   # the nearest row is the one after two NaN rows
    x[40:50] = y[801] + 0.01
    for pat in ("0.5", "all", "slab"):
        adj = adjacency(pat, m, len(gidx), rng)
        if pat != "slab":                       # (slab: the rows keep whatever their slab has)
            adj[20:50, :] = True
        idx, val = run_checked(x, y, adj, gidx, rng)
        assert (idx[[5, 250]] == NO_CANDIDATE).all()
        assert not np.isin(idx, [11, 300, 301, 800, 12, 500]).any()
        if pat != "slab":
            assert (idx[20:40] == 302).all() and (idx[40:50] == 801).all()


def test_large_group_count():
    """G = 1500 (masked_validate_kernel takes two passes over group_idxs) with small random groups."""
    rng = np.random.default_rng(15)
    m, n, k = 400, 3100, 48
    x, y = data("blobs", m, n, k, seed=15)
    gidx = np.minimum(np.cumsum(rng.integers(0, 6, size=1500)), n - 3).astype(np.int32)
    assert len(gidx) == 1500 and gidx[-1] == n - 3
    for pat in ("0.1", "0.5", "cc"):
        run_checked(x, y, adjacency(pat, m, 1500, rng), gidx, rng)


@pytest.mark.parametrize("k", [33, 200, 784])
@pytest.mark.parametrize("end", ["n", "before_n", "mid_block"])
def test_single_group(k, end):
    """G = 1: one group ending at n, 37 rows before n, or inside the first y block; each row of x adjacent to it or not
    (random), so the tiles are ALL, NONE and PARTIAL."""
    rng = np.random.default_rng(k + len(end))
    m, n = 333, 1300
    x, y = data("blobs", m, n, k, seed=k + 3)
    gidx = np.array([{"n": n, "before_n": n - 37, "mid_block": 100}[end]], np.int32)
    for pat in ("all", "none", "0.5", "slab"):
        idx, _ = run_checked(x, y, adjacency(pat, m, 1, rng), gidx, rng)
        assert (idx[idx != NO_CANDIDATE] < gidx[0]).all()


@pytest.mark.parametrize("k", [64, 200, 784])
def test_none_runs_for_one_slab_followed_by_live_tiles(k, exact_fused):
    """The one-slab NONE runs of the K3m skip protocol (the even slab of x tile t adjacent to group 0 only unless
    t % 4 == 3, the odd slab to every group), at 16384 x 16384 so that the work items hold runs of x tiles.  Sampled rows
    of both slabs against the fp64 bound, and the whole result through the union law: the result merged with the
    complement mask's (init_out = 0) is the exact fusedL2NN, bit for bit."""
    m = n = 16384
    x, _, c = oracle.make_blobs(m, k, seed=31)
    y, _, _ = oracle.make_blobs(n, k, seed=32, centers=c)
    G = n // 1024
    gidx = np.arange(1024, n + 1, 1024, dtype=np.int32)
    adj = np.ones((m, G), bool)
    for t in range(m // 128):
        if t % 4 != 3:
            adj[128 * t:128 * t + 64, 1:] = False
    xd, yd, gd = gpu(x), gpu(y), gpu(gidx)
    out = call(xd, yd, gpu(adj.astype(np.uint8)), gd)
    idx, val = host(out)
    rows = np.concatenate([np.arange(0, m, 37), np.arange(384, 512)])
    check(x, y, adj, gidx, idx, val, rows=rows)
    call(xd, yd, gpu((~adj).astype(np.uint8)), gd, out=out, init_out=0)
    union = host(out)
    fused = fused_exact(xd, yd)
    assert (fused[1] > 0).all()
    assert_same(union, fused, k)


# ---------------------------------------------------------------------------------------------------------------------
# 2. operands, adjacency bytes, group edges

@pytest.mark.parametrize("k,pitch", [(37, 40), (37, 48), (200, 203)])
def test_padded_unaligned_and_aliased_operands(k, pitch):
    """Padded pitches, a base one float behind an allocation boundary, y the same pointer as x (connect_components) and
    y a row window of x give the contiguous call's result, bit for bit."""
    rng = np.random.default_rng(k + pitch)
    m, n = 333, 900
    x, y = data("blobs", m, n, k, seed=4)
    gidx = groups(n, rng)
    adj = adjacency("0.5", m, len(gidx), rng)
    ad, gd = device_adj(adj, rng), gpu(gidx)
    base = run_checked(x, y, adj, gidx, rng)

    def padded(a, ld, off):
        buf = torch.full((off + a.shape[0] * ld,), 777.0, device="cuda")
        v = buf[off:].view(a.shape[0], ld)[:, :a.shape[1]]
        v.copy_(torch.from_numpy(a))
        return v

    for offx, offy in ((0, 0), (1, 0), (0, 1), (1, 1)):
        assert_same(host(call(padded(x, pitch, offx), padded(y, pitch, offy), ad, gd)), base, (offx, offy))
    # y is x (the same pointer; connect_components: every group but the row's own), and y a window of rows of x
    xx = padded(np.concatenate([x, y]), pitch, 1)
    gx = groups(m, rng)
    own = column_groups(gx, m)
    adjx = np.ones((m, len(gx)), bool)
    adjx[np.nonzero(own >= 0)[0], own[own >= 0]] = False
    idx, val = host(call(xx[:m], xx[:m], device_adj(adjx, rng), gpu(gx)))
    check(x, x, adjx, gx, idx, val)
    assert_same(host(call(xx[:m], xx[m:], ad, gd)), base, "window")


def test_adjacency_bytes_and_wrapper():
    """Bytes 2, 0x80 and 0xFF are adjacent like 1; the padding of a pitch ld_adj > G is never read; bool and uint8
    through the Python wrapper give the ABI's result."""
    rng = np.random.default_rng(8)
    m, n, k = 300, 1000, 40
    x, y = data("gauss", m, n, k, seed=8)
    xd, yd = gpu(x), gpu(y)
    gidx = groups(n, rng)
    G = len(gidx)
    adj = adjacency("0.5", m, G, rng)
    gd = gpu(gidx)
    base = host(call(xd, yd, gpu(adj.astype(np.uint8)), gd))
    check(x, y, adj, gidx, *base)
    for v in (2, 0x80, 0xFF):
        b = np.full((m, G + 9), 1, np.uint8)
        b[:, :G] = np.where(adj, v, 0)
        assert_same(host(call(xd, yd, gpu(b), gd, G=G)), base, v)
    # the padding full of 1s where the mask says nothing is adjacent: still no candidate anywhere
    b = np.ones((m, G + 3), np.uint8)
    b[:, :G] = 0
    i0, v0 = host(call(xd, yd, gpu(b), gd, G=G))
    assert (i0 == NO_CANDIDATE).all() and (v0.view(np.uint32) == FLT_MAX_BITS).all()
    for a in (torch.from_numpy(adj).cuda(), torch.from_numpy(adj.astype(np.uint8) * 0x80).cuda()):
        wi, wv = masked_l2_nn(xd, yd, a, gd)
        assert_same((wi.cpu().numpy(), wv.cpu().numpy()), base, a.dtype)


def test_empty_groups_and_database_give_sentinel():
    """G = 0 (no adjacency, no group_idxs), n = 0, every group empty, and every row of y after the last end: every row
    is {0x7fffffff, FLT_MAX}; with init_out = 0 the caller's values stay."""
    m, k = 70, 33
    x, y = data("gauss", m, 500, k)
    xd, yd = gpu(x), gpu(y)
    ones = torch.ones((m, 4), dtype=torch.uint8, device="cuda")
    cases = [
        (yd, None, None, 0),                                                    # G = 0
        (None, ones, torch.zeros(4, dtype=torch.int32, device="cuda"), 4),      # n = 0
        (yd, ones, torch.zeros(4, dtype=torch.int32, device="cuda"), 4),        # all groups empty
        (yd[:1], ones, torch.zeros(4, dtype=torch.int32, device="cuda"), 4),    # n = 1, after the last end
    ]
    for y_, a, g, G in cases:
        i, v = host(call(xd, y_, a, g, G=G))
        assert (i == NO_CANDIDATE).all() and (v.view(np.uint32) == FLT_MAX_BITS).all(), G
        mine = torch.stack([torch.arange(m, dtype=torch.int32, device="cuda"),
                            torch.full((m,), 3.5, device="cuda").view(torch.int32)], 1)
        i, v = host(call(xd, y_, a, g, G=G, out=mine.clone(), init_out=0))
        assert np.array_equal(i, np.arange(m)) and (v == 3.5).all()


# ---------------------------------------------------------------------------------------------------------------------
# 3. bit-exact laws

def fused_exact(xd, yd):
    """fusedL2NN through the ABI (the caller holds nn_screen = 0: the exact kernel)."""
    L = _lib.lib()
    m, k = xd.shape
    n = yd.shape[0]
    nb = L.b2d_fused_l2_nn_workspace_bytes(m, n, k)
    ws = torch.full((nb,), 255, dtype=torch.uint8, device="cuda")
    out = torch.empty((m, 2), dtype=torch.int32, device="cuda")
    _lib.check(L.b2d_fused_l2_nn(torch.cuda.current_stream().cuda_stream, out.data_ptr(), xd.data_ptr(), xd.stride(0),
                                 yd.data_ptr(), yd.stride(0), None, None, m, n, k, 0, 1, ws.data_ptr(), nb))
    return host(out)


@pytest.mark.parametrize("k", KS)
def test_all_tiles_equal_exact_fused_l2_nn(k, exact_fused):
    """Every group adjacent and the last one ending at n: every tile is ALL, and the result is fusedL2NN's exact kernel
    bit for bit -- also with NaN rows of x and y, Inf rows of y, outliers and zero rows."""
    rng = np.random.default_rng(k + 5)
    m, n = 1985, 4353
    for kind in ("gauss", "special"):
        x, y = data("gauss", m, n, k, seed=k)
        if kind == "special":
            x[3] *= 1.0e9
            x[4] *= 1.0e-6
            x[[5, 1000]] = np.nan
            x[6] = 0.0
            y[[10, 2000]] *= 1.0e9
            y[[11, 300, 4352]] = np.nan
            y[[12, 3000]] = np.inf
            y[600] = 0.0
        xd, yd = gpu(x), gpu(y)
        gidx = groups(n, rng, tail=False)
        adj = np.ones((m, len(gidx)), bool)
        assert (tile_classes(adj, gidx, m, n) == 1).all()
        got = host(call(xd, yd, device_adj(adj, rng), gpu(gidx)))
        assert_same(got, fused_exact(xd, yd), kind)
        if kind == "special":
            assert (got[0][[5, 1000]] == NO_CANDIDATE).all()


@pytest.mark.parametrize("k", [2, 64, 129, 320, 784])
def test_union_law(k):
    """masked(A | B) == masked(A) merged with masked(B) through init_out = 0, bit for bit: a pair's value does not depend
    on the mask.  (Data without duplicates: no value clamps to 0, where two different raw values would both read 0.)"""
    rng = np.random.default_rng(k + 9)
    m, n = 700, 2100
    x, y = data("gauss", m, n, k, seed=k + 1)
    xd, yd = gpu(x), gpu(y)
    gidx = groups(n, rng)
    gd = gpu(gidx)
    G = len(gidx)
    for pa, pb in (("0.1", "slab"), ("cc", "0.5"), ("none", "slab"), ("slab", "slab")):
        a, b = adjacency(pa, m, G, rng), adjacency(pb, m, G, rng)
        whole = host(call(xd, yd, device_adj(a | b, rng), gd))
        out = call(xd, yd, device_adj(a, rng), gd)
        call(xd, yd, device_adj(b, rng), gd, out=out, init_out=0)
        merged = host(out)
        assert (whole[1] > 0).all()
        assert_same(merged, whole, (pa, pb))
        check(x, y, a | b, gidx, *whole)


def int_tie_case(k, seed):
    """Small integers (every step of the kernel exact), groups of 64 rows (two per 128-column half; rows 1984.. in no
    group), and for the query rows 0..39 of slab 0 duplicates of the nearest row (distance 1) planted at a smaller index
    in a group that is not adjacent, in an ALL tile and in a PARTIAL tile of the same row, in another y block, and after
    the last group end.  Returns x, y, adj, gidx and the expected index of the query rows."""
    rng = np.random.default_rng(seed)
    m, n = 256, 2048
    x = rng.integers(-3, 4, (m, k)).astype(np.float32)
    y = rng.integers(-3, 4, (n, k)).astype(np.float32)
    gidx = np.arange(64, n - 63, 64, dtype=np.int32)           # group g: rows [64 g, 64 g + 64), g < 31
    G = len(gidx)
    adj = rng.random((m, G)) < 0.3
    adj[:64] = False
    adj[:64, [2, 3, 4, 12, 13, 20]] = True
    adj[:64:2, 20] = False                                      # group 20: the odd rows of slab 0 only
    cls = tile_classes(adj, gidx, m, n)
    # slab 0: half 0 (groups 0, 1) NONE, half 1 (2, 3) ALL, half 2 (4, 5) PARTIAL, half 6 (12, 13) ALL, half 10 PARTIAL
    assert cls[0, 0] == 0 and cls[0, 1] == 1 and cls[0, 2] == 2 and cls[0, 6] == 1 and cls[0, 10] == 2
    free = {lo: iter((lo + rng.permutation(size)).tolist()) for lo, size in
            ((0, 64), (128, 64), (256, 64), (768, 128), (1280, 64), (1984, 64))}
    e = np.zeros(k, np.float32)
    e[0] = 1.0
    expect = []
    for r in range(40):
        if r % 4 == 0:     # a PARTIAL tile (group 4); the same point at a smaller index in group 0, not adjacent
            pos = [next(free[0]), next(free[256])]
        elif r % 4 == 1:   # an ALL tile (group 2) and a PARTIAL tile (group 20, adjacent to the odd rows)
            pos = [next(free[128]), next(free[1280])]
        elif r % 4 == 2:   # a PARTIAL tile, an ALL tile of another y block (groups 12, 13) and after the last end
            pos = [next(free[256]), next(free[768]), next(free[1984])]
        else:              # an ALL tile of another y block and after the last end
            pos = [next(free[768]), next(free[1984])]
        for j in pos:
            y[j] = x[r] + e
        expect.append(pos[1] if r % 4 == 0 else pos[0])
    return x, y, adj, gidx, np.array(expect)


@pytest.mark.parametrize("k", [16, 96, 200, 784])
def test_integer_data_bit_exact_with_ties(k):
    """Integer data against the reference bit for bit, tie order included, with the planted duplicates of int_tie_case;
    the other rows have random masks and their own ties."""
    x, y, adj, gidx, expect = int_tie_case(k, seed=k)
    assert k * 2 * max(np.abs(x).max(), np.abs(y).max()) ** 2 < 2 ** 24
    ri, rv = ref_masked_l2_nn(x, y, adj, gidx)
    assert np.array_equal(ri[:40], expect) and (rv[:40] == 1.0).all()
    rng = np.random.default_rng(k)
    xd, yd, ad, gd = gpu(x), gpu(y), device_adj(adj, rng), gpu(gidx)
    idx, val = host(call(xd, yd, ad, gd))
    assert np.array_equal(idx, ri)
    assert np.array_equal(val.astype(np.float64), np.where(ri == NO_CANDIDATE, np.float32(FLT_MAX), rv))
    assert_sqrt_law(idx, val, *host(call(xd, yd, ad, gd, sqrt=True)))


@pytest.mark.parametrize("k", [64, 200, 784])
def test_scaling_law(k):
    """x, y -> 2^s x, 2^s y (s = +-20, +-50) multiplies every value by 2^2s exactly and moves no index."""
    rng = np.random.default_rng(k + 2)
    m, n = 500, 1500
    x, y = data("blobs", m, n, k, seed=k + 2)
    xd, yd = gpu(x), gpu(y)
    gidx = groups(n, rng)
    adj = adjacency("0.5", m, len(gidx), rng)
    ad, gd = device_adj(adj, rng), gpu(gidx)
    i0, v0 = run_checked(x, y, adj, gidx, rng, xd, yd)
    live = i0 != NO_CANDIDATE
    for s in (-50, -20, 20, 50):
        f = 2.0 ** s
        i1, v1 = host(call(xd * f, yd * f, ad, gd))
        assert np.array_equal(i1, i0), s
        assert np.array_equal(v1[live].view(np.uint32), (v0[live] * np.float32(f * f)).view(np.uint32)), s
        assert (v1[~live].view(np.uint32) == FLT_MAX_BITS).all()
        i2, v2 = host(call(xd * f, yd * f, ad, gd, sqrt=True))
        assert np.array_equal(i2, i0), s
        assert np.array_equal(v2[live].view(np.uint32), (np.sqrt(v0[live]) * np.float32(f)).view(np.uint32)), s


@pytest.mark.parametrize("k", [33, 200, 784])
def test_caller_norms_change_no_bit(k):
    """xn / yn from b2d_row_norm (L2Norm, no sqrt: fp64 sums rounded once, as the operand preparation does)."""
    L = _lib.lib()
    rng = np.random.default_rng(k + 4)
    m, n = 400, 1300
    x, y = data("gauss", m, n, k, seed=k + 4)
    xd, yd = gpu(x), gpu(y)
    gidx = groups(n, rng)
    ad, gd = device_adj(adjacency("cc", m, len(gidx), rng), rng), gpu(gidx)
    xn, yn = torch.empty(m, device="cuda"), torch.empty(n, device="cuda")
    for t, nrm in ((xd, xn), (yd, yn)):
        _lib.check(L.b2d_row_norm(None, nrm.data_ptr(), t.data_ptr(), k, t.shape[0], k, 2, 0))
    assert_same(host(call(xd, yd, ad, gd, xn=xn, yn=yn)), host(call(xd, yd, ad, gd)))


# ---------------------------------------------------------------------------------------------------------------------
# 4. protocol: init_out = 0, invalid group_idxs, determinism, stale workspace, graph capture

def test_init_out_false_merges_by_argmin_op():
    """The caller's smaller value stays; its equal value with a smaller key stays, with a larger key it is replaced; a
    larger value is replaced; on rows without a candidate the caller's value stays."""
    rng = np.random.default_rng(12)
    m, n, k = 400, 1200, 64
    x, y = data("blobs", m, n, k, seed=12)
    xd, yd = gpu(x), gpu(y)
    gidx = groups(n, rng)
    adj = adjacency("0.5", m, len(gidx), rng)
    adj[300:] = False
    ad, gd = device_adj(adj, rng), gpu(gidx)
    i0, v0 = host(call(xd, yd, ad, gd))
    assert (i0[300:] == NO_CANDIDATE).all() and (i0[:300] != NO_CANDIDATE).all() and (v0[:300] > 0).all()
    r = np.arange(m) % 4
    ei = np.where(r == 1, i0 - 1, i0 + 1).astype(np.int32)
    ei[(r == 1) & (i0 == 0)] = 0
    ev = v0.copy()
    ev[r == 0] *= np.float32(0.5)
    ev[(r == 3) & (i0 != NO_CANDIDATE)] = v0[(r == 3) & (i0 != NO_CANDIDATE)] * np.float32(2) + np.float32(1)
    ei[300:] = np.arange(300, m)
    ev[300:] = np.float32(1e30)
    out = gpu(np.stack([ei, ev.view(np.int32)], 1))
    i1, v1 = host(call(xd, yd, ad, gd, out=out, init_out=0))
    keep = (ev < v0) | ((ev == v0) & (ei < i0))
    live = np.arange(m) < 300
    assert keep[live & (r == 0)].all() and keep[live & (r == 1) & (i0 > 0)].all() and not keep[live & (r >= 2)].any()
    assert keep[~live].all()
    assert np.array_equal(i1, np.where(keep, ei, i0))
    assert np.array_equal(v1.view(np.uint32), np.where(keep, ev, v0).view(np.uint32))


@pytest.mark.parametrize("init_out", [1, 0])
def test_invalid_group_idxs_poison_every_row(init_out):
    """A group_idxs that decreases or leaves [0, n] (also past the first 1024 entries) gives every row
    {0x7fffffff, NaN}, whatever out held."""
    m, n, k = 150, 600, 24
    x, y = data("gauss", m, n, k)
    xd, yd = gpu(x), gpu(y)
    bad = [np.array([100, 50, 300], np.int32), np.array([100, 200, n + 1], np.int32), np.array([-1, 10, 20], np.int32)]
    big = np.minimum(np.arange(1500) // 3, n).astype(np.int32)
    big[1300] = big[1299] - 1
    bad.append(big)
    big2 = big.copy()
    big2[1300] = big2[1299]
    big2[-1] = n + 5
    bad.append(big2)
    for g in bad:
        G = len(g)
        a = torch.ones((m, G), dtype=torch.uint8, device="cuda")
        out = torch.zeros((m, 2), dtype=torch.int32, device="cuda")
        i, v = host(call(xd, yd, a, gpu(g), out=out, init_out=init_out))
        assert (i == POISON[0]).all() and (v.view(np.uint32) == POISON[1]).all(), g[:4]


def test_determinism_stale_workspace_and_graph_capture():
    """Two calls give identical bytes; a workspace left over from a call with another mask and other data changes
    nothing; a CUDA graph captured on a side stream and replayed once gives the eager result."""
    rng = np.random.default_rng(77)
    L = _lib.lib()
    m, n, k = 1000, 3000, 200
    x, y = data("blobs", m, n, k, seed=77)
    xd, yd = gpu(x), gpu(y)
    gidx = groups(n, rng)
    G = len(gidx)
    adj = adjacency("0.5", m, G, rng)
    ad, gd = device_adj(adj, rng), gpu(gidx)
    first = host(call(xd, yd, ad, gd))
    check(x, y, adj, gidx, *first)
    assert_same(host(call(xd, yd, ad, gd)), first, "second call")
    nb = L.b2d_masked_l2_nn_workspace_bytes(m, n, k, G)
    ws = torch.full((nb,), 255, dtype=torch.uint8, device="cuda")
    call(xd.flip(0).contiguous(), yd * 2, device_adj(adjacency("slab", m, G, rng), rng), gd, ws=ws, sqrt=True)
    assert_same(host(call(xd, yd, ad, gd, ws=ws)), first, "stale workspace")
    out = torch.full((m, 2), -1, dtype=torch.int32, device="cuda")
    ws.fill_(255)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            call(xd, yd, ad, gd, out=out, ws=ws)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph.replay()
    assert_same(host(out), first, "graph replay")
