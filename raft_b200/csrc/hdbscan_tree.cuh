// Host-only tree stages of the linkage calls (no device code, so a C++ test can compile this header on its own): the
// dendrogram merges single linkage and HDBSCAN share, and HDBSCAN's condensed tree, stability, cluster selection, labels
// and probabilities (DESIGN.md K22).  The semantics are sklearn.cluster.HDBSCAN's (cluster/_hdbscan/_tree.pyx), applied
// to the mutual-reachability tree given as its m - 1 edges in order.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <vector>

namespace b2d {

inline int uf_find(std::vector<int>& p, int v)
{
  while (p[v] != v) v = p[v] = p[p[v]];
  return v;
}

// The merges of the m - 1 tree edges (src[t], dst[t]) taken in order: merge t joins the clusters of its two ends into
// cluster m + t, children[2 t], children[2 t + 1] (smaller id first), sizes[t] rows.  With labels, labels[i] = a row id
// naming row i's cluster after the first cut merges (cut in [0, m - 1]).  False: the edges hold a cycle.
inline bool sl_merges(int64_t m, const int* src, const int* dst, int* children, int* sizes, int64_t cut, int* labels)
{
  std::vector<int> uf(m), cid(m), sz(m, 1);
  for (int64_t i = 0; i < m; ++i) uf[i] = cid[i] = static_cast<int>(i);
  for (int64_t t = 0; t < m - 1; ++t) {
    if (labels && t == cut)
      for (int64_t i = 0; i < m; ++i) labels[i] = uf_find(uf, static_cast<int>(i));
    const int a = uf_find(uf, src[t]), b = uf_find(uf, dst[t]);
    if (a == b) return false;
    children[2 * t]     = std::min(cid[a], cid[b]);
    children[2 * t + 1] = std::max(cid[a], cid[b]);
    sizes[t]            = sz[a] + sz[b];
    uf[b]               = a;
    sz[a]               = sizes[t];
    cid[a]              = static_cast<int>(m + t);
  }
  if (labels && cut == m - 1)
    for (int64_t i = 0; i < m; ++i) labels[i] = uf_find(uf, static_cast<int>(i));
  return true;
}

// What approximate_predict looks up, besides the ball cover: where every row left the condensed tree, and the clusters
// (ids 0 = the root, 1, 2, ... as the condensing pass numbers them, so a parent's id is below its child's).
struct HdbTreeExport {
  std::vector<int> row_parent;      // [m] the cluster a row leaves
  std::vector<double> row_lambda;   // [m] the lambda at which it leaves it
  std::vector<int> parent;          // [nc] the parent cluster (-1: the root)
  std::vector<int> owner;           // [nc] the nearest selected ancestor, the cluster itself included (0: the root)
  std::vector<int> label;           // [nc] a selected cluster's label, or -1 (not selected, or no row took it)
  std::vector<double> birth;        // [nc] the lambda of the cluster's birth (0 for the root)
  std::vector<double> death;        // [nc] sklearn's max_lambdas of the cluster
  bool single_root = false;         // the root is the one selected cluster ...
  double thr       = 0.0;           // ... and a row that leaves it at a lambda >= thr takes its label
};

struct HdbTreeParams {
  int min_cluster_size;   // >= 2
  double epsilon;         // cluster_selection_epsilon >= 0
  bool leaf;              // cluster_selection_method "leaf" (else "eom")
  bool allow_single_cluster;
};

// HDBSCAN's tree stages on the mutual-reachability tree: its m - 1 edges (src[t], dst[t]) in order, at distance w[t] (the
// metric's, not necessarily distinct).  labels [m] (int32, -1 noise, clusters numbered in order of their smallest row)
// and probabilities [m].  Returns the number of clusters that hold a row, or -1 when the edges hold a cycle.
//
// Clusters are numbered as the condensing pass meets them (breadth first from the root, smaller child first), so that
// the row order of the condensed tree, which sums the stabilities and bounds the probabilities, is sklearn's.  A
// cluster's "death" is the largest lambda of the last run of consecutive condensed rows it parents, as sklearn's
// max_lambdas computes it.  The epsilon search visits the selected leaves in ascending cluster id.  With ex, the tree
// as HdbTreeExport describes it (one row: the root alone, which labels nothing).
inline int hdbscan_tree(int64_t m64, const int* src, const int* dst, const float* w, const HdbTreeParams& p, int* labels,
                        float* prob, HdbTreeExport* ex = nullptr)
{
  const int m = static_cast<int>(m64);
  if (m == 1) {
    labels[0] = -1;
    prob[0]   = 0.f;
    if (ex) *ex = HdbTreeExport{{0}, {0.0}, {-1}, {0}, {-1}, {0.0}, {0.0}};
    return 0;
  }
  std::vector<int> ch(2 * static_cast<size_t>(m - 1)), sz(m - 1);
  if (!sl_merges(m, src, dst, ch.data(), sz.data(), -1, nullptr)) return -1;
  const int mcs = p.min_cluster_size;
  auto count    = [&](int v) { return v < m ? 1 : sz[v - m]; };

  // 1. condensed tree: rows (parent cluster, child row or cluster, lambda, size); clusters are m, m + 1, ...
  std::vector<int> cpar, cchild, csize;
  std::vector<double> clam;
  auto row = [&](int par, int c, double l, int s) {
    cpar.push_back(par);
    cchild.push_back(c);
    clam.push_back(l);
    csize.push_back(s);
  };
  const int root_node = 2 * m - 2;
  std::vector<int> relabel(2 * static_cast<size_t>(m) - 1), queue{root_node}, sub;
  relabel[root_node] = m;
  int next           = m + 1;
  auto fall = [&](int from, int par, double l) {   // every row under `from` leaves cluster par at l, breadth first
    sub.assign(1, from);
    for (size_t h = 0; h < sub.size(); ++h) {
      const int v = sub[h];
      if (v < m) row(par, v, l, 1);
      else {
        sub.push_back(ch[2 * (v - m)]);
        sub.push_back(ch[2 * (v - m) + 1]);
      }
    }
  };
  for (size_t h = 0; h < queue.size(); ++h) {
    const int v = queue[h], t = v - m;
    const int left = ch[2 * t], right = ch[2 * t + 1], pv = relabel[v];
    const double d = w[t];
    const double l = d > 0.0 ? 1.0 / d : INFINITY;
    const int lc = count(left), rc = count(right);
    if (lc >= mcs && rc >= mcs) {
      relabel[left] = next++;
      row(pv, relabel[left], l, lc);
      relabel[right] = next++;
      row(pv, relabel[right], l, rc);
      queue.push_back(left);
      queue.push_back(right);
    } else if (lc < mcs && rc < mcs) {
      fall(left, pv, l);
      fall(right, pv, l);
    } else if (lc < mcs) {
      relabel[right] = pv;
      fall(left, pv, l);
      queue.push_back(right);
    } else {
      relabel[left] = pv;
      fall(right, pv, l);
      queue.push_back(left);
    }
  }
  const int nc = next - m;   // clusters, the root (index 0) included
  const size_t nr = cpar.size();

  // 2. stability: sum over a cluster's rows of (lambda - its birth) * size, in row order
  std::vector<double> birth(nc, 0.0), stab(nc, 0.0), death(nc, 0.0);
  std::vector<int> parent(nc, -1), kid0(nc, -1), kid1(nc, -1);
  for (size_t r = 0; r < nr; ++r)
    if (cchild[r] >= m) {
      const int c = cchild[r] - m, pc = cpar[r] - m;
      birth[c]  = clam[r];
      parent[c] = pc;
      (kid0[pc] < 0 ? kid0[pc] : kid1[pc]) = c;
    }
  for (size_t r = 0; r < nr; ++r) stab[cpar[r] - m] += (clam[r] - birth[cpar[r] - m]) * csize[r];
  for (size_t r = 0; r < nr;) {   // death: max lambda of the last run of rows of each parent
    size_t e = r;
    double mx = clam[r];
    while (++e < nr && cpar[e] == cpar[r]) mx = std::max(mx, clam[e]);
    death[cpar[r] - m] = mx;
    r = e;
  }

  // 3. selection.  The candidates are the clusters other than the root, and the root too with allow_single_cluster;
  // a child's id is above its parent's, so descending ids visit children first.
  const int first = p.allow_single_cluster ? 0 : 1;
  std::vector<char> sel(nc, 0);
  const bool has_tree = nc > 1;   // the condensed tree has a cluster row
  auto epsilon_search = [&](const std::vector<int>& leaves) {
    std::vector<char> out(nc, 0), done(nc, 0);
    std::vector<int> stack;
    for (int c : leaves) {
      if (1.0 / birth[c] < p.epsilon) {
        if (done[c]) continue;
        int e = c;
        for (;;) {   // sklearn's traverse_upwards
          const int par = parent[e];
          if (par == 0) {
            if (p.allow_single_cluster) e = 0;
            break;
          }
          e = par;
          if (1.0 / birth[par] > p.epsilon) break;
        }
        out[e] = 1;
        stack.assign(1, e);
        while (!stack.empty()) {
          const int v = stack.back();
          stack.pop_back();
          if (v != e) done[v] = 1;
          if (kid0[v] >= 0) stack.push_back(kid0[v]);
          if (kid1[v] >= 0) stack.push_back(kid1[v]);
        }
      } else
        out[c] = 1;
    }
    return out;
  };
  if (!p.leaf) {
    std::vector<char> chose(nc, 0);
    for (int c = nc - 1; c >= first; --c) {
      const double st = kid0[c] >= 0 ? stab[kid0[c]] + stab[kid1[c]] : 0.0;
      if (st > stab[c]) stab[c] = st;
      else chose[c] = 1;
    }
    std::vector<char> blocked(nc, 0);   // an ancestor chose itself
    for (int c = first; c < nc; ++c) {
      if (c > 0) blocked[c] = blocked[parent[c]] || (parent[c] >= first && chose[parent[c]]);
      sel[c] = chose[c] && !blocked[c];
    }
    if (p.epsilon != 0.0 && has_tree) {
      std::vector<int> eom;
      for (int c = first; c < nc; ++c)
        if (sel[c]) eom.push_back(c);
      if (eom.size() == 1 && eom[0] == 0) {
        // the root alone (allow_single_cluster) stays selected
      } else {
        const std::vector<char> e = epsilon_search(eom);
        for (int c = first; c < nc; ++c) sel[c] = e[c];
      }
    }
  } else if (has_tree) {
    std::vector<int> leaves;
    for (int c = 1; c < nc; ++c)
      if (kid0[c] < 0) leaves.push_back(c);
    if (p.epsilon != 0.0) {
      const std::vector<char> e = epsilon_search(leaves);
      for (int c = first; c < nc; ++c) sel[c] = e[c];
    } else
      for (int c : leaves) sel[c] = 1;
  }

  // 4. labels: a row belongs to its nearest selected ancestor cluster; rows that reach the root are noise, unless the
  // root is the one selected cluster and the row left it at a lambda no smaller than the threshold
  int n_sel = 0;
  std::vector<int> owner(nc);
  for (int c = 0; c < nc; ++c) {
    owner[c] = (c == 0 || sel[c]) ? c : owner[parent[c]];
    n_sel += sel[c];
  }
  double thr = 0.0;
  const bool single_root = n_sel == 1 && p.allow_single_cluster && sel[0];
  if (single_root) {
    if (p.epsilon != 0.0) thr = 1.0 / p.epsilon;
    else {
      thr = -INFINITY;
      for (size_t r = 0; r < nr; ++r)
        if (cpar[r] == m) thr = std::max(thr, clam[r]);
    }
  }
  std::vector<int> canon(nc, -1);   // selected cluster -> label in order of its smallest row
  std::vector<int> lab(m, -1), cl(m, -1);
  std::vector<double> lam(m, 0.0);
  for (size_t r = 0; r < nr; ++r)
    if (cchild[r] < m) {
      const int i = cchild[r], o = owner[cpar[r] - m];
      lam[i]      = clam[r];
      if (o != 0 || (single_root && clam[r] >= thr)) cl[i] = o;
    }
  int next_label = 0;
  for (int i = 0; i < m; ++i) {
    const int c = cl[i];
    if (c < 0) {
      labels[i] = -1;
      prob[i]   = 0.f;
      continue;
    }
    if (canon[c] < 0) canon[c] = next_label++;
    labels[i]       = canon[c];
    const double md = death[c];
    prob[i] = static_cast<float>(md == 0.0 || std::isinf(lam[i]) ? 1.0 : std::min(lam[i], md) / md);
  }
  if (ex) {
    ex->row_parent.assign(m, 0);
    for (size_t r = 0; r < nr; ++r)
      if (cchild[r] < m) ex->row_parent[cchild[r]] = cpar[r] - m;
    ex->row_lambda = lam;
    ex->parent     = parent;
    ex->owner      = owner;
    ex->label      = canon;
    ex->birth      = birth;
    ex->death      = death;
    ex->single_root = single_root;
    ex->thr         = thr;
  }
  return next_label;
}

}  // namespace b2d
