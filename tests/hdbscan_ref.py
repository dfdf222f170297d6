"""The oracle of HDBSCAN on the ball cover (include/raft_b200.h, b2d_hdbscan_rbc_fit; DESIGN.md K22), in numpy fp64 on
the float32 pair values s of tests/ball_cover_ref.dist (term by term, each operation rounded on its own):
  core distances   core[i] = the min_samples-th smallest s(i, j) over every j, i itself (s = 0) included;
  the MR tree      Prim's algorithm under the strict edge order (w, min row, max row), w(i, j) = max(core_i, core_j,
                   s(i, j)), so the tree is the unique one the contract names; its m - 1 edges in that order;
  the tree stages  sklearn.cluster.HDBSCAN's condensed tree, stability, EOM / leaf selection with allow_single_cluster
                   and cluster_selection_epsilon, labels and probabilities (cluster/_hdbscan/_tree.pyx), on the tree's
                   weights in the metric (s, or its correctly rounded float32 root).  Clusters are numbered in order of
                   their smallest row.
tests/test_hdbscan_rbc.py checks the whole against sklearn.cluster.HDBSCAN(metric="precomputed")."""
import math

import numpy as np


def pair_row(x, i):
    """float32 s(i, j) for every j (x float32 [m, d])"""
    s = None
    for c in range(x.shape[1]):
        t = x[i, c] - x[:, c]
        t = t * t
        s = t if s is None else s + t
    return s


def pair_matrix(x):
    return np.stack([pair_row(x, i) for i in range(len(x))])


def core_distances(x, min_samples):
    """float32 [m]: the min_samples-th smallest s of every row, the row itself included"""
    m = len(x)
    out = np.empty(m, np.float32)
    chunk = max(1, (1 << 24) // max(m, 1))
    for a in range(0, m, chunk):
        rows = np.stack([pair_row(x, i) for i in range(a, min(m, a + chunk))])
        out[a:a + len(rows)] = np.partition(rows, min_samples - 1, axis=1)[:, min_samples - 1]
    return out


def mr_tree(x, min_samples, metric="sqeuclidean"):
    """(src, dst, w, core): the MR tree's m - 1 edges in (w, min row, max row) order, src < dst (int32), w float32 (s
    domain, or its root for "euclidean"), and the core distances (s domain)"""
    x = np.ascontiguousarray(x, np.float32)
    m = len(x)
    core = core_distances(x, min_samples)
    rows = np.arange(m)
    bw = np.full(m, np.inf)
    ba = np.full(m, m, np.int64)
    bb = np.full(m, m, np.int64)
    done = np.zeros(m, bool)
    ea, eb, ew = [], [], []
    v = 0
    for it in range(m):
        done[v] = True
        bw[v] = np.inf
        if it == m - 1:
            break
        w = np.maximum(np.maximum(core, core[v]), pair_row(x, v)).astype(np.float64)
        a, b = np.minimum(rows, v), np.maximum(rows, v)
        better = ~done & ((w < bw) | ((w == bw) & ((a < ba) | ((a == ba) & (b < bb)))))
        bw[better], ba[better], bb[better] = w[better], a[better], b[better]
        c = np.flatnonzero(bw == bw.min())
        c = c[ba[c] == ba[c].min()]
        v = int(c[np.argmin(bb[c])])
        ea.append(ba[v])
        eb.append(bb[v])
        ew.append(bw[v])
    ea, eb, ew = np.array(ea, np.int64), np.array(eb, np.int64), np.array(ew, np.float32)
    o = np.lexsort((eb, ea, ew))
    w = ew[o]
    if metric == "euclidean":
        w = np.sqrt(w, dtype=np.float32)
    return ea[o].astype(np.int32), eb[o].astype(np.int32), w.astype(np.float32), core


def merges(m, src, dst):
    """children [m - 1, 2] (smaller id first) and sizes of the merges of the edges taken in order"""
    uf, cid, sz = list(range(m)), list(range(m)), [1] * m

    def find(v):
        while uf[v] != v:
            uf[v] = uf[uf[v]]
            v = uf[v]
        return v

    ch, size = np.zeros((max(m - 1, 0), 2), np.int64), np.zeros(max(m - 1, 0), np.int64)
    for t in range(m - 1):
        a, b = find(int(src[t])), find(int(dst[t]))
        assert a != b
        ch[t] = sorted((cid[a], cid[b]))
        size[t] = sz[a] + sz[b]
        uf[b] = a
        sz[a] = size[t]
        cid[a] = m + t
    return ch, size


def condense(ch, size, w, m, mcs):
    """the condensed tree as rows (parent, child, lambda, size), clusters m (the root), m + 1, ... numbered as a breadth
    first pass from the root meets them"""
    def count(v):
        return 1 if v < m else int(size[v - m])

    def leaves_bfs(v):
        out, q = [], [v]
        while q:
            nq = []
            for u in q:
                if u < m:
                    out.append(u)
                else:
                    nq += [int(ch[u - m, 0]), int(ch[u - m, 1])]
            q = nq
        return out

    rows = []
    relabel = {2 * m - 2: m}
    nxt = m + 1
    queue = [2 * m - 2]
    while queue:
        nq = []
        for v in queue:
            left, right = int(ch[v - m, 0]), int(ch[v - m, 1])
            d = float(w[v - m])
            lam = 1.0 / d if d > 0 else math.inf
            lc, rc = count(left), count(right)
            pv = relabel[v]
            if lc >= mcs and rc >= mcs:
                for c, cnt in ((left, lc), (right, rc)):
                    relabel[c] = nxt
                    rows.append((pv, nxt, lam, cnt))
                    nxt += 1
                nq += [left, right]
            else:
                for c, cnt in ((left, lc), (right, rc)):
                    if cnt < mcs:
                        rows += [(pv, u, lam, 1) for u in leaves_bfs(c)]
                    else:
                        relabel[c] = pv
                        nq.append(c)
        queue = nq
    return rows


def tree_labels(src, dst, w, m, min_cluster_size, method="eom", allow_single_cluster=False, epsilon=0.0):
    """(labels int32, probabilities float64, n_clusters) of the tree stages on the edges in order; n_clusters counts the
    clusters that hold a row"""
    if m == 1:
        return np.array([-1], np.int32), np.zeros(1), 0
    ch, size = merges(m, src, dst)
    rows = condense(ch, size, w, m, min_cluster_size)
    root = m
    birth, parent, kids, stab = {root: 0.0}, {}, {}, {}
    for p, c, lam, s in rows:
        if c >= m:
            birth[c], parent[c] = lam, p
            kids.setdefault(p, []).append(c)
    for p, c, lam, s in rows:
        stab[p] = stab.get(p, 0.0) + (lam - birth[p]) * s
    death = {}
    k = 0
    while k < len(rows):   # the largest lambda of the last run of rows of each parent
        e, mx = k + 1, rows[k][2]
        while e < len(rows) and rows[e][0] == rows[k][0]:
            mx = max(mx, rows[e][2])
            e += 1
        death[rows[k][0]] = mx
        k = e
    clusters = sorted(birth)
    cand = [c for c in clusters if allow_single_cluster or c != root]

    def below(c):
        out, q = [], list(kids.get(c, []))
        while q:
            u = q.pop()
            out.append(u)
            q += kids.get(u, [])
        return out

    def eps_search(leaves):
        chosen, done = set(), set()
        for c in sorted(leaves):
            if 1.0 / birth[c] < epsilon:
                if c in done:
                    continue
                e = c
                while True:
                    p = parent[e]
                    if p == root:
                        if allow_single_cluster:
                            e = root
                        break
                    e = p
                    if 1.0 / birth[p] > epsilon:
                        break
                chosen.add(e)
                done.update(below(e))
            else:
                chosen.add(c)
        return chosen

    is_cl = {c: True for c in cand}
    if method == "eom":
        for c in sorted(cand, reverse=True):
            sub = sum(stab[k] for k in kids[c]) if c in kids else 0.0
            if sub > stab[c]:
                is_cl[c] = False
                stab[c] = sub
            else:
                for u in below(c):
                    is_cl[u] = False
        if epsilon != 0.0 and len(clusters) > 1:
            eom = [c for c in sorted(cand) if is_cl[c]]
            if not (len(eom) == 1 and eom[0] == root):
                sel = eps_search(eom)
                is_cl = {c: c in sel for c in cand}
    else:
        leaves = [c for c in clusters if c != root and c not in kids] if len(clusters) > 1 else []
        sel = eps_search(leaves) if epsilon != 0.0 else set(leaves)
        is_cl = {c: c in sel for c in cand}
    chosen = {c for c in cand if is_cl[c]}

    def owner(c):
        while c != root and c not in chosen:
            c = parent[c]
        return c

    single = len(chosen) == 1 and allow_single_cluster and root in chosen
    if single:
        thr = 1.0 / epsilon if epsilon != 0.0 else max(r[2] for r in rows if r[0] == root)
    cl = np.full(m, -1, np.int64)
    lam_of = np.zeros(m)
    for p, c, lam, s in rows:
        if c < m:
            o = owner(p)
            lam_of[c] = lam
            if o != root or (single and lam >= thr):
                cl[c] = o
    labels = np.full(m, -1, np.int32)
    prob = np.zeros(m)
    canon = {}
    for i in range(m):
        c = int(cl[i])
        if c < 0:
            continue
        labels[i] = canon.setdefault(c, len(canon))
        md = death[c]
        prob[i] = 1.0 if md == 0.0 or math.isinf(lam_of[i]) else min(lam_of[i], md) / md
    return labels, prob, len(canon)


def hdbscan(x, min_cluster_size=5, min_samples=None, cluster_selection_epsilon=0.0, cluster_selection_method="eom",
            allow_single_cluster=False, metric="euclidean"):
    """(labels, probabilities fp64, n_clusters, (src, dst, w)) of the whole fit"""
    ms = min_cluster_size if min_samples is None else min_samples
    src, dst, w, _ = mr_tree(x, ms, metric)
    lab, prob, n = tree_labels(src, dst, w, len(x), min_cluster_size, cluster_selection_method, allow_single_cluster,
                               cluster_selection_epsilon)
    return lab, prob, n, (src, dst, w)


def canonical(labels):
    """labels renumbered in order of each cluster's smallest row, noise (negative) as -1"""
    out = np.full(len(labels), -1, np.int32)
    seen = {}
    for i, l in enumerate(labels):
        if l >= 0:
            out[i] = seen.setdefault(int(l), len(seen))
    return out
