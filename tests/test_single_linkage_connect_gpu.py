"""GPU tier: single_linkage's connect_components (b2d_single_linkage step 4, DESIGN.md K13) on every chunk, sort block,
round and tie edge, against the exact reference (single_linkage_ref.py).

Integer data first.  Small integers are exact in every arithmetic of the path (the fp16 hi/lo split, the tensor
accumulation, the fp64 norms, the fused kNN and the masked arg-min) while every |x|^2 < 2^22, so the device must equal
the reference bit for bit, ties included.  The rows form islands: each island holds between n_nb and 2 n_nb - 1 rows
(or any number of rows of a unit grid when n_nb >= 7, so that every row's kNN holds its grid neighbours), and the gaps
between islands are wider than any island, so the kNN graph's components are exactly the islands and their count is
known in advance.  The rows are shuffled, so every island is spread over the chunks and sort blocks.  Every case
asserts the plan it is named after (b2d_debug_single_linkage_plan) for its first connect round, then that the device
kNN is the exact kNN bit for bit (ties by index included), then children, sizes, labels, n_connected_components and
the deltas bytes against single_linkage_from_knn.

Float data second: blobs, where no value is bit-exact.  The sorted deltas are the sorted kNN-forest weights of the
device's own kNN, bit for bit, followed by the sorted weights of the exact inter-component minimum spanning tree, each
within the masked arg-min's error bound (test_masked_nn_paths_gpu.py, `bounds`)."""
import ctypes

import numpy as np
import pytest

import single_linkage_ref as ref

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

METRIC = {"sqeuclidean": 0, "euclidean": 1}   # B2D_L2Expanded, B2D_L2SqrtExpanded
ULP = 2.0 ** -24


# ---------------------------------------------------------------------------------------------------------------------
# the call, the plan, the exact kNN

def plan(m, comps):
    """b2d_debug_single_linkage_plan: (chunk rows, chunks, sort block rows, sort blocks) of a connect round."""
    from raft_b200 import _lib
    out = (ctypes.c_int64 * 4)()
    _lib.check(_lib.lib().b2d_debug_single_linkage_plan(m, comps, ctypes.addressof(out)))
    return tuple(out)


def c_arg(m, n_nb):
    """The c argument that gives n_nb neighbours on m rows."""
    c = n_nb - int(np.floor(np.log2(m)))
    assert ref.n_neighbors(m, c) == n_nb
    return c


def sl_call(xd, m, d, c, nc, metric, ldx=None, ws=None):
    """One b2d_single_linkage call on the device buffer xd (rows of pitch ldx), with a workspace filled with 0xFF
    unless `ws` is given.  Returns (children, deltas, sizes, labels, n_components) on the host."""
    from raft_b200 import _lib
    L = _lib.lib()
    need = L.b2d_single_linkage_workspace_bytes(m, d, c)
    if ws is None:
        ws = torch.full((need,), 255, dtype=torch.uint8, device="cuda")
    ch = torch.empty((m - 1, 2), dtype=torch.int32, device="cuda")
    de = torch.empty(m - 1, dtype=torch.float32, device="cuda")
    sz = torch.empty(m - 1, dtype=torch.int32, device="cuda")
    lab = torch.empty(m, dtype=torch.int32, device="cuda")
    ncomp = np.zeros(1, np.int32)
    s = torch.cuda.current_stream().cuda_stream
    _lib.check(L.b2d_single_linkage(s, METRIC[metric], xd.data_ptr(), d if ldx is None else ldx, m, d, c, nc,
                                    ch.data_ptr(), de.data_ptr(), sz.data_ptr(), lab.data_ptr(), ncomp.ctypes.data,
                                    ws.data_ptr(), need))
    torch.cuda.synchronize()
    return ch.cpu().numpy(), de.cpu().numpy(), sz.cpu().numpy(), lab.cpu().numpy(), int(ncomp[0])


def device_knn(x, k):
    from raft_b200.neighbors import brute_force
    xd = torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()
    dist, idx = brute_force.knn(xd, xd, k, metric="sqeuclidean")
    return idx.cpu().numpy(), dist.cpu().numpy()


def knn_exact_int(x, k):
    """The exact kNN of integer rows against themselves in (squared distance, index) order, in row blocks."""
    x = np.asarray(x, np.float64)
    m = len(x)
    nx = (x * x).sum(1)
    idx = np.zeros((m, k), np.int64)
    dist = np.zeros((m, k), np.float64)
    for r0 in range(0, m, 512):
        d2 = nx[r0:r0 + 512, None] + nx[None, :] - 2 * x[r0:r0 + 512] @ x.T   # integers below 2^53: exact
        key = d2.astype(np.int64) * m + np.arange(m)[None, :]
        part = np.argpartition(key, k - 1, axis=1)[:, :k]
        part = np.take_along_axis(part, np.argsort(np.take_along_axis(key, part, 1), axis=1), 1)
        idx[r0:r0 + 512] = part
        dist[r0:r0 + 512] = np.take_along_axis(d2, part, 1)
    return idx, dist.astype(np.float32)


def labels_after(children, m, nc):
    """The labels of scipy's convention from a dendrogram: clusters after the first m - nc merges, numbered in order
    of their smallest row."""
    p = np.arange(2 * m - 1)
    for t in range(m - nc):
        p[children[t, 0]] = p[children[t, 1]] = m + t
    top = np.arange(m)
    for _ in range(m):   # follow every row up to its cluster after m - nc merges
        nxt = p[top]
        if (nxt == top).all():
            break
        top = nxt
    return ref.canonical_labels(top)


def check_exact(x, n_nb, comps, metric, want_plan):
    """The whole comparison of one integer case (module docstring), for n_clusters in {1, 2, comps, comps + 1, m}."""
    m, d = x.shape
    assert (x.astype(np.float64) ** 2).sum(1).max() < 2 ** 22 and (x == np.round(x)).all()
    assert plan(m, comps) == want_plan
    idx, dist = knn_exact_int(x, n_nb)
    didx, ddist = device_knn(x, n_nb)
    assert (didx == idx).all() and ddist.tobytes() == dist.tobytes()
    sq = metric == "euclidean"
    rch, rde, rsz, rlab, rncomp = ref.single_linkage_from_knn(x, idx, dist, 1, sqrt=sq)
    assert rncomp == comps
    c = c_arg(m, n_nb)
    xd = torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()
    for nc in sorted({1, 2, comps, min(comps + 1, m), m}):
        ch, de, sz, lab, ncomp = sl_call(xd, m, d, c, nc, metric)
        assert ncomp == comps
        assert (ch == rch).all(), nc
        assert (sz == rsz).all(), nc
        assert de.tobytes() == rde.astype(np.float32).tobytes(), nc
        assert (lab == labels_after(rch, m, nc)).all(), nc
    assert (labels_after(rch, m, 1) == rlab).all()


# ---------------------------------------------------------------------------------------------------------------------
# integer islands

def island_sizes(m, comps, n_nb, dl):
    """comps island sizes summing to m, each of one kNN component (module docstring)."""
    sizes = np.full(comps, m // comps)
    sizes[:m % comps] += 1
    assert sizes.min() >= n_nb and (sizes.max() <= 2 * n_nb - 1 or n_nb >= 2 * dl + 1), (sizes.max(), n_nb)
    return sizes


def grid_prefix(s, dl):
    """The first s points of a k^dl unit grid in lexicographic order (a connected set), and k."""
    k = int(np.ceil(s ** (1.0 / dl) - 1e-9))
    while k ** dl < s:
        k += 1
    g = np.stack(np.meshgrid(*[np.arange(k)] * dl, indexing="ij"), -1).reshape(-1, dl)
    return g[:s], k


def lattice_islands(m, comps, n_nb, d, seed, spread=8):
    """Islands on a regular super-lattice of the first min(d, 3) coordinates (many equidistant islands and rows);
    the other coordinates, when d > 3, a small random integer per island.  Rows shuffled."""
    rng = np.random.default_rng(seed)
    dl = min(d, 3)
    sizes = island_sizes(m, comps, n_nb, dl)
    _, k = grid_prefix(int(sizes.max()), dl)
    G = 3 * k   # island diameter <= sqrt(3) (k - 1): every gap is wider
    side = int(np.ceil(comps ** (1.0 / dl) - 1e-9))
    while side ** dl < comps:
        side += 1
    sites = np.stack(np.meshgrid(*[np.arange(side)] * dl, indexing="ij"), -1).reshape(-1, dl)[:comps] * G
    sites -= (side - 1) * G // 2
    rows = []
    for g, s in enumerate(sizes):
        pts = np.zeros((s, d))
        pts[:, :dl] = sites[g] + grid_prefix(int(s), dl)[0]
        if d > dl:
            pts[:, dl:] = rng.integers(-spread, spread + 1, d - dl)
        rows.append(pts)
    return rng.permutation(np.concatenate(rows)).astype(np.float32)


def line_islands(gaps, s, d, seed):
    """len(gaps) + 1 islands of s rows at unit spacing on the first coordinate, gaps[i] between islands i and i + 1
    (end to start); the other coordinates 0.  Centred, rows shuffled."""
    starts = np.concatenate([[0], np.cumsum(np.asarray(gaps) + s - 1)])
    pos = (starts[:, None] + np.arange(s)[None, :]).reshape(-1)
    pos -= (pos.max() + pos.min()) // 2
    x = np.zeros((len(pos), d))
    x[:, 0] = pos
    return np.random.default_rng(seed).permutation(x).astype(np.float32)


def ruler(n):
    """1, 2, 1, 4, 1, 2, 1, 8, ...: 2^(trailing zeros of i) for i = 1 .. n."""
    i = np.arange(1, n + 1)
    return i & -i


# (name, m, d, islands, n_nb, metric, plan of the first connect round)
LATTICE = [
    ("one chunk, two islands", 5000, 8, 2, 20, "sqeuclidean", (5120, 1, 2048, 3)),
    ("last single chunk", 5000, 3, 125, 40, "euclidean", (5120, 1, 2048, 3)),
    ("first two chunks", 5000, 3, 126, 39, "sqeuclidean", (4992, 2, 2048, 3)),
    ("two chunks at 128 islands", 5000, 2, 128, 39, "euclidean", (4992, 2, 2048, 3)),
    ("three chunks", 5000, 2, 257, 19, "sqeuclidean", (2432, 3, 2048, 3)),
    ("eight chunks", 5000, 8, 1000, 5, "euclidean", (640, 8, 2048, 3)),
    ("two-row islands, 256-row chunks", 5000, 3, 2500, 2, "sqeuclidean", (256, 20, 2048, 3)),
    ("sort: one block short of 2048", 2047, 33, 300, 6, "euclidean", (768, 3, 2048, 1)),
    ("sort: one full block", 2048, 2, 64, 32, "sqeuclidean", (2048, 1, 2048, 1)),
    ("sort: one row past a block", 2049, 129, 100, 20, "euclidean", (2176, 1, 2048, 2)),
    ("sort: four blocks, streaming operands", 6145, 320, 500, 12, "sqeuclidean", (1536, 5, 2048, 4)),
    ("ties: 2-D lattice", 3001, 2, 300, 10, "euclidean", (1280, 3, 2048, 2)),
    ("ties: 3-D lattice", 3001, 3, 343, 8, "sqeuclidean", (1024, 3, 2048, 2)),
]


@pytest.mark.parametrize("name,m,d,comps,n_nb,metric,want_plan", LATTICE, ids=[c[0] for c in LATTICE])
def test_lattice_islands(name, m, d, comps, n_nb, metric, want_plan):
    x = lattice_islands(m, comps, n_nb, d, seed=m + d + comps)
    check_exact(x, n_nb, comps, metric, want_plan)


# (name, gaps, rows per island, d, metric, plan)
LINES = [
    ("rounds: ruler gaps, 128 islands", 3 * ruler(127), 3, 1, "sqeuclidean", (384, 1, 2048, 1)),
    ("rounds: ruler gaps, 256 islands, d = 8", 2 * ruler(255), 2, 8, "euclidean", (256, 2, 2048, 1)),
    ("rounds: distinct random gaps", 3 + np.random.default_rng(5).permutation(59), 3, 1, "euclidean",
     (256, 1, 2048, 1)),
]


def reference_rounds(x, idx, dist):
    """The number of connect rounds of single_linkage_from_knn."""
    src, dst, w = ref.knn_edges(idx, dist)
    _, colour = ref.kruskal(src, dst, w, len(x))
    rounds = 0
    while len(np.unique(colour)) > 1:
        cs, cd, cw = ref.connect_edges(x, colour)
        src, dst, w = np.concatenate([src, cs]), np.concatenate([dst, cd]), np.concatenate([w, cw.astype(w.dtype)])
        _, colour = ref.kruskal(src, dst, w, len(x))
        rounds += 1
    return rounds


@pytest.mark.parametrize("name,gaps,s,d,metric,want_plan", LINES, ids=[c[0] for c in LINES])
def test_line_islands_force_rounds(name, gaps, s, d, metric, want_plan):
    comps = len(gaps) + 1
    x = line_islands(gaps, s, d, seed=comps)
    check_exact(x, s, comps, metric, want_plan)
    if "ruler" in name:   # every round only halves the components
        assert reference_rounds(x, *knn_exact_int(x, s)) == int(np.ceil(np.log2(comps)))


def test_pitched_offset_x_equals_contiguous():
    """x at an element offset inside a larger buffer, with a row pitch ldx > d, through the C ABI: the same bytes as
    the contiguous call."""
    m, d, comps, n_nb = 3001, 5, 300, 10
    x = lattice_islands(m, comps, n_nb, d, seed=3)
    assert plan(m, comps) == (1280, 3, 2048, 2)
    c = c_arg(m, n_nb)
    want = sl_call(torch.from_numpy(x).cuda(), m, d, c, comps, "euclidean")
    for ldx, off in ((7, 3), (64, 1), (133, 0)):
        buf = torch.full((m * ldx + off + 5,), float("nan"), dtype=torch.float32, device="cuda")
        view = buf[off:off + m * ldx].view(m, ldx)
        view[:, :d] = torch.from_numpy(x).cuda()
        view[:, d:] = 1e30   # the pitch padding is never read
        got = sl_call(buf[off:], m, d, c, comps, "euclidean", ldx=ldx)
        for a, b in zip(got[:4], want[:4]):
            assert a.tobytes() == b.tobytes(), (ldx, off)
        assert got[4] == want[4] == comps


def test_repeats_are_identical():
    """Repeated calls, with a fresh or a reused (stale) workspace, give identical bytes."""
    from raft_b200 import _lib
    m, d, comps, n_nb = 5000, 8, 1000, 5
    x = lattice_islands(m, comps, n_nb, d, seed=9)
    c = c_arg(m, n_nb)
    xd = torch.from_numpy(x).cuda()
    ws = torch.full((_lib.lib().b2d_single_linkage_workspace_bytes(m, d, c),), 255, dtype=torch.uint8, device="cuda")
    runs = [sl_call(xd, m, d, c, 7, "euclidean")] + [sl_call(xd, m, d, c, 7, "euclidean", ws=ws) for _ in range(3)]
    for r in runs[1:]:
        for a, b in zip(r[:4], runs[0][:4]):
            assert a.tobytes() == b.tobytes()
        assert r[4] == comps


# ---------------------------------------------------------------------------------------------------------------------
# float blobs

def component_distances(x, colour):
    """The exact (fp64) smallest squared distance between every two components, c x c (inf on the diagonal)."""
    x = np.asarray(x, np.float64)
    comp = np.unique(colour, return_inverse=True)[1]
    order = np.argsort(comp, kind="stable")
    xs, cs = x[order], comp[order]
    starts = np.flatnonzero(np.r_[True, cs[1:] != cs[:-1]])
    c = len(starts)
    nx = (xs * xs).sum(1)
    D = np.full((c, c), np.inf)
    for r0 in range(0, len(xs), 1024):
        d2 = np.maximum(nx[r0:r0 + 1024, None] + nx[None, :] - 2 * xs[r0:r0 + 1024] @ xs.T, 0)
        per = np.minimum.reduceat(d2, starts, axis=1)                # rows x components
        rc = cs[r0:r0 + 1024]
        np.minimum.at(D, rc, per)
    np.fill_diagonal(D, np.inf)
    return D


@pytest.mark.parametrize("m,d,n_blobs,sep,metric", [
    (4000, 8, 10, 60.0, "sqeuclidean"), (9000, 33, 60, 80.0, "euclidean"), (20000, 16, 300, 200.0, "sqeuclidean"),
    (12000, 130, 120, 100.0, "euclidean"),
])
def test_blobs_against_exact_component_tree(m, d, n_blobs, sep, metric):
    from scipy.sparse.csgraph import minimum_spanning_tree
    rng = np.random.default_rng(m + n_blobs)
    centres = rng.uniform(-sep, sep, (n_blobs, d))
    x = (centres[rng.integers(0, n_blobs, m)] + rng.standard_normal((m, d))).astype(np.float32)
    n_nb = ref.n_neighbors(m)
    idx, dist = device_knn(x, n_nb)
    chosen, colour = ref.kruskal(*ref.knn_edges(idx, dist), m)
    comps = len(np.unique(colour))
    assert 10 <= comps <= 400
    assert plan(m, comps)[1] >= 1
    ch, de, sz, lab, ncomp = sl_call(torch.from_numpy(x).cuda(), m, d, 15, comps, metric)
    assert ncomp == comps
    forest = np.sort(dist.reshape(-1)[chosen])                      # the kNN forest's squared weights, fp32
    D = component_distances(x, colour)
    T = minimum_spanning_tree(np.where(np.isinf(D), 0, D)).tocoo()
    inter = np.sort(T.data)
    assert len(inter) == comps - 1 and forest.max() < inter.min() / 2
    # the masked arg-min's bound (bounds() of test_masked_nn_paths_gpu.py) at the largest norms: each connecting edge
    # is a nearest pair up to hi + lo, and its weight is off by at most hi or lo
    big = np.sort((x.astype(np.float64) ** 2).sum(1))[-2:].sum()
    tol = 3 * (32 + d / 8) * ULP * big
    sq = metric == "euclidean"
    got = np.sort(de)
    k = m - comps
    want_forest = np.sqrt(forest) if sq else forest
    assert got[:k].tobytes() == want_forest.astype(np.float32).tobytes()
    g = got[k:].astype(np.float64) ** (2 if sq else 1)
    bad = np.nonzero(np.abs(g - inter) > tol + 2 * ULP * inter)[0]
    assert len(bad) == 0, [(int(i), g[i], inter[i], tol) for i in bad[:5]]
    # n_clusters = comps: the kNN graph's components
    assert (lab == ref.canonical_labels(colour)).all()
    assert sz[-1] == m and sorted(np.unique(ch).tolist()) == list(range(2 * m - 2))


def test_histogram_cap_duplicate_pairs():
    """135000 distinct integer sites of the plane, each held by two identical rows: with n_nb = 2 every pair is one
    component, and 135000 components x 132 sort blocks pass the 2^24 histogram words, so the sort widens its blocks.
    The arithmetic is exact, so the sorted deltas are m - c zeros followed by the sorted squared weights of the sites'
    exact Euclidean minimum spanning tree (over their Delaunay edges), bit for bit."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import minimum_spanning_tree
    from scipy.spatial import Delaunay
    comps = 135000
    m = 2 * comps
    assert plan(m, comps) == (256, 1055, 4096, 66)
    rng = np.random.default_rng(13)
    side = 1024
    sites = rng.choice(side * side, comps, replace=False)
    sites = np.stack([sites % side, sites // side], 1) - side // 2
    owner = rng.permutation(np.repeat(np.arange(comps), 2))   # the site of every row
    x = sites[owner].astype(np.float32)
    assert (x.astype(np.float64) ** 2).sum(1).max() < 2 ** 22
    # the exact kNN: every row and its twin, at distance 0, in index order
    order = np.lexsort((np.arange(m), owner))
    pair = order.reshape(comps, 2)
    want_idx = np.zeros((m, 2), np.int64)
    want_idx[pair[:, 0]] = pair
    want_idx[pair[:, 1]] = pair
    idx, dist = device_knn(x, 2)
    assert (idx == want_idx).all() and not dist.any()
    tri = Delaunay(sites.astype(np.float64)).simplices
    e = np.unique(np.sort(np.concatenate([tri[:, [0, 1]], tri[:, [1, 2]], tri[:, [0, 2]]]), 1), axis=0)   # (no sums)
    w = ((sites[e[:, 0]] - sites[e[:, 1]]) ** 2).sum(1).astype(np.float64)
    T = minimum_spanning_tree(coo_matrix((w, (e[:, 0], e[:, 1])), shape=(comps, comps)).tocsr()).tocoo()
    inter = np.sort(T.data)
    assert len(inter) == comps - 1
    ch, de, sz, lab, ncomp = sl_call(torch.from_numpy(x).cuda(), m, 2, c_arg(m, 2), comps, "sqeuclidean")
    assert ncomp == comps
    want = np.concatenate([np.zeros(m - comps), inter]).astype(np.float32)
    assert np.sort(de).tobytes() == want.tobytes()
    assert (lab == ref.canonical_labels(owner)).all()
    assert (sz[:m - comps] == 2).all() and sz[-1] == m and sorted(np.unique(ch).tolist()) == list(range(2 * m - 2))
