"""The oracle of HDBSCAN's approximate_predict on the ball cover (include/raft_b200.h,
b2d_hdbscan_rbc_approximate_predict; DESIGN.md K23), in numpy fp64 on the float32 pair values s of the fit's oracle
(tests/hdbscan_ref.py, term by term, each operation rounded on its own):
  the model     hdbscan_ref's MR tree, merges and condensed tree; from them each row's parent cluster and lambda, and
                each cluster's parent, birth, death, owner (nearest selected ancestor) and label, by the selection and
                label rule of hdbscan_ref.tree_labels (restated here, and checked against it);
  a query       core_q = the min_samples-th smallest s to the fitted rows; the neighbour j* = the first row in the order
                (w, s, row), w = max(core_q, core_j, s); W its metric value; lambda = min(1 / W, lambda_j*); the parent
                walk up while birth > lambda; the fit's label rule and probability there.
Cluster ids are 0 (the root), 1, ... in the condensing pass's order, as hdbscan_tree numbers them."""
import math

import numpy as np

import hdbscan_ref as H


def export(src, dst, w, m, mcs, method="eom", single=False, eps=0.0):
    """the fitted tree as a dict: row_parent, row_lambda [m]; parent, birth, death, owner, label [nc]; single_root, thr;
    and the fit's labels and probabilities (fp64) by the rule restated on these arrays"""
    if m == 1:
        return dict(row_parent=np.zeros(1, np.int64), row_lambda=np.zeros(1), parent=np.array([-1]), birth=np.zeros(1),
                    death=np.zeros(1), owner=np.zeros(1, np.int64), label=np.array([-1]), single_root=False, thr=0.0,
                    labels=np.array([-1], np.int32), prob=np.zeros(1))
    ch, size = H.merges(m, src, dst)
    rows = [(p - m, c, lam, s) for p, c, lam, s in H.condense(ch, size, w, m, mcs)]   # parents as cluster ids
    nc = 1 + sum(1 for _, c, _, _ in rows if c >= m)
    parent, birth, death, stab = np.full(nc, -1), np.zeros(nc), np.zeros(nc), np.zeros(nc)
    kids = [[] for _ in range(nc)]
    row_parent, row_lambda = np.zeros(m, np.int64), np.zeros(m)
    for p, c, lam, s in rows:
        if c >= m:
            parent[c - m], birth[c - m] = p, lam
            kids[p].append(c - m)
        else:
            row_parent[c], row_lambda[c] = p, lam
    for p, c, lam, s in rows:
        stab[p] += (lam - birth[p]) * s
    k = 0
    while k < len(rows):   # death: the largest lambda of the last run of rows of each parent
        e, mx = k + 1, rows[k][2]
        while e < len(rows) and rows[e][0] == rows[k][0]:
            mx = max(mx, rows[e][2])
            e += 1
        death[rows[k][0]] = mx
        k = e
    first = 0 if single else 1

    def below(c):
        out, q = [], list(kids[c])
        while q:
            u = q.pop()
            out.append(u)
            q += kids[u]
        return out

    def eps_search(leaves):
        chosen, done = set(), set()
        for c in sorted(leaves):
            if 1.0 / birth[c] < eps:
                if c in done:
                    continue
                e = c
                while True:
                    p = parent[e]
                    if p == 0:
                        if single:
                            e = 0
                        break
                    e = p
                    if 1.0 / birth[p] > eps:
                        break
                chosen.add(e)
                done.update(below(e))
            else:
                chosen.add(c)
        return chosen

    sel = np.zeros(nc, bool)
    if method == "eom":
        is_cl = {c: True for c in range(first, nc)}
        for c in range(nc - 1, first - 1, -1):
            sub = sum(stab[u] for u in kids[c]) if kids[c] else 0.0
            if sub > stab[c]:
                is_cl[c] = False
                stab[c] = sub
            else:
                for u in below(c):
                    is_cl[u] = False
        chosen = [c for c in range(first, nc) if is_cl[c]]
        if eps != 0.0 and nc > 1 and chosen != [0]:
            chosen = sorted(eps_search(chosen))
        sel[chosen] = True
    elif nc > 1:
        leaves = [c for c in range(1, nc) if not kids[c]]
        for c in (eps_search(leaves) if eps != 0.0 else leaves):
            if c >= first:
                sel[c] = True
    owner = np.zeros(nc, np.int64)
    for c in range(nc):
        owner[c] = c if c == 0 or sel[c] else owner[parent[c]]
    single_root = bool(sel.sum() == 1 and single and sel[0])
    thr = 0.0
    if single_root:
        thr = 1.0 / eps if eps != 0.0 else max(lam for p, c, lam, s in rows if p == 0)
    label, n_labels = np.full(nc, -1), 0
    labels, prob = np.full(m, -1, np.int32), np.zeros(m)
    for i in range(m):   # clusters numbered in order of their smallest row
        o = owner[row_parent[i]]
        if o == 0 and not (single_root and row_lambda[i] >= thr):
            continue
        if label[o] < 0:
            label[o], n_labels = n_labels, n_labels + 1
        labels[i] = label[o]
        prob[i] = _prob(row_lambda[i], death[o])
    return dict(row_parent=row_parent, row_lambda=row_lambda, parent=parent, birth=birth, death=death, owner=owner,
                label=label, single_root=single_root, thr=thr, labels=labels, prob=prob)


def _prob(lam, md):
    return 1.0 if md == 0.0 or math.isinf(lam) else min(lam, md) / md


def fit(x, min_cluster_size, min_samples, method="eom", single=False, eps=0.0, metric="euclidean", tree=None):
    """the model of the fit of x (float32 [m, d]): export()'s dict plus core (s domain, by row) and the tree.  tree: the
    s-domain H.mr_tree(x, min_samples), when the caller has it"""
    x = np.ascontiguousarray(x, np.float32)
    src, dst, w, core = H.mr_tree(x, min_samples) if tree is None else tree
    if metric == "euclidean":
        w = np.sqrt(w, dtype=np.float32)
    model = export(src, dst, w, len(x), min_cluster_size, method, single, eps)
    model.update(x=x, core=core, min_samples=min_samples, metric=metric, tree=(src, dst, w))
    return model


def neighbour(model, q):
    """(j*, W) of one finite query q: the first row in the order (w, s, row), W = w's metric value (float32)"""
    x = model["x"]
    s = None
    for c in range(x.shape[1]):
        t = np.float32(q[c]) - x[:, c]
        t = t * t
        s = t if s is None else s + t
    cq = np.partition(s, model["min_samples"] - 1)[model["min_samples"] - 1]
    w = np.maximum(np.maximum(cq, model["core"]), s)
    j = int(np.lexsort((np.arange(len(x)), s, w))[0])
    W = w[j] if model["metric"] == "sqeuclidean" else np.sqrt(w[j], dtype=np.float32)
    return j, np.float32(W)


def place(model, j, W):
    """(label, probability fp64) of a query whose neighbour is j at metric weight W"""
    lam = 1.0 / float(W) if W > 0 else math.inf
    lam = min(lam, model["row_lambda"][j])
    p = int(model["row_parent"][j])
    while p != 0 and model["birth"][p] > lam:
        p = int(model["parent"][p])
    o = int(model["owner"][p])
    lab = int(model["label"][o])
    if o == 0 and not (model["single_root"] and lam >= model["thr"]):
        lab = -1
    return lab, (_prob(lam, model["death"][o]) if lab >= 0 else 0.0)


def predict(model, q):
    """(labels int32, probabilities float32, neighbours int32, weights float32) of the queries q [n, d]"""
    q = np.asarray(q, np.float32)
    n = len(q)
    lab, prob = np.full(n, -1, np.int32), np.zeros(n, np.float32)
    nn, ww = np.full(n, -1, np.int32), np.full(n, np.inf, np.float32)
    for i in range(n):
        if not np.isfinite(q[i]).all():
            continue
        j, W = neighbour(model, q[i])
        l, p = place(model, j, W)
        lab[i], prob[i], nn[i], ww[i] = l, np.float32(p), j, W
    return lab, prob, nn, ww
