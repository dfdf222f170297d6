// Minimum spanning forest and single-linkage clustering (single_linkage.cuh).
#include <cuda_runtime.h>
#include <algorithm>
#include <string>
#include <vector>
#include <cub/device/device_radix_sort.cuh>

#include "hdbscan_rbc.cuh"
#include "hdbscan_tree.cuh"
#include "host.cuh"
#include "single_linkage.cuh"
#include "single_linkage_rbc.cuh"

using namespace b2d;

// ------------------------------------------------------------------------------------------
// Minimum spanning forest and single-linkage clustering (single_linkage.cuh): edge-list Borůvka under the key order
// key_pack(w, e); single_linkage runs it on the kNN graph, connects the components the graph leaves apart with the
// masked arg-min, and builds the dendrogram on the host.
namespace {
constexpr int64_t kSlMaxRows  = 1ll << 30;
constexpr int64_t kSlMaxEdges = 0xFFFFFFFFll;   // positions are the low 32 bits of a key (2^32 - 1 only in KEY_EMPTY)

struct MstLayout {
  SlCtrl* ctrl;
  int* colour;        // [n] component of every vertex (the id of a vertex of it)
  int* parent;        // [n] hook forest of the components of a round; at the end the smallest vertex of each tree
  long long* best;    // [n] minimum key of every component in a round
  long long* keys;    // [n] keys of the forest edges in the order they were chosen (KEY_EMPTY behind them)
  long long* alt;     // [n] the other buffer of the radix sort
  void* sort_tmp;
  size_t sort_bytes;
  size_t bytes;
};

static MstLayout mst_regions(Carve& c, int64_t n)
{
  MstLayout L{};
  L.ctrl       = c.take<SlCtrl>(1);
  L.colour     = c.take<int>(n);
  L.parent     = c.take<int>(n);
  L.best       = c.take<long long>(n);
  L.keys       = c.take<long long>(n);
  L.alt        = c.take<long long>(n);
  L.sort_bytes = kSortTmpBytes + static_cast<size_t>(n) * 4;   // (checked at run time)
  L.sort_tmp   = c.take<char>(L.sort_bytes);
  L.bytes      = c.bytes;
  return L;
}

static MstLayout mst_layout(void* base, int64_t n)
{
  Carve c(base, 1024);
  return mst_regions(c, n);
}

static int ceil_log2(int64_t n)
{
  int r = 0;
  while ((1ll << r) < n) ++r;
  return r;
}

// Borůvka rounds over the edges [e0, e1) of a graph on n vertices with at most `comps` components, every other edge
// already inside a component.  Only enqueues: the non-isolated components at least halve in every round, so
// ceil(log2 comps) rounds finish, and every kernel after a round that appended nothing returns at once.
static int mst_rounds(cudaStream_t s, const MstLayout& L, const int* src, const int* dst, const float* w, int64_t n,
                      int64_t e0, int64_t e1, int64_t comps)
{
  const int rounds = ceil_log2(comps) + 1;
  const int jumps  = std::min(kSlMaxJumps, ceil_log2(comps) + 1);   // hook chains are shorter than comps
  const unsigned ge = static_cast<unsigned>(std::max<int64_t>(1, std::min<int64_t>((e1 - e0 + 255) / 256, 1 << 16)));
  for (int r = 0; r < rounds; ++r) {
    sl_round_begin_kernel<<<sl_grid(std::max<int64_t>(n, kSlMaxJumps)), 256, 0, s>>>(L.ctrl, L.best, n);
    sl_edge_kernel<<<ge, 256, 0, s>>>(L.ctrl, src, dst, w, e0, e1, n, L.colour, L.best);
    sl_hook_kernel<<<sl_grid(n), 256, 0, s>>>(L.ctrl, src, dst, L.colour, L.best, L.parent, L.keys, n);
    for (int j = 0; j < jumps; ++j) sl_jump_kernel<<<sl_grid(n), 256, 0, s>>>(L.ctrl, L.colour, L.parent, n, j);
    sl_relabel_kernel<<<sl_grid(n), 256, 0, s>>>(L.ctrl, L.colour, L.parent, n);
    sl_round_end_kernel<<<1, 1, 0, s>>>(L.ctrl);
    B2D_CUDA(cudaGetLastError());
  }
  return B2D_OK;
}

// the forest edges in key order: endpoints, weights (their square roots with do_sqrt) and the count
static int mst_emit(cudaStream_t s, const MstLayout& L, const int* src, const int* dst, const float* w, int64_t n,
                    int do_sqrt, int* out_src, int* out_dst, float* out_w, int* out_count)
{
  cub::DoubleBuffer<long long> db(L.keys, L.alt);
  size_t need = 0;
  B2D_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, need, db, static_cast<int>(n), 0, 64, s));
  if (need > L.sort_bytes) return fail(B2D_ERR_WORKSPACE, "internal: radix sort scratch " + std::to_string(need) + " bytes");
  B2D_CUDA(cub::DeviceRadixSort::SortKeys(L.sort_tmp, need, db, static_cast<int>(n), 0, 64, s));
  sl_emit_kernel<<<sl_grid(n), 256, 0, s>>>(L.ctrl, db.Current(), src, dst, w, std::max<int64_t>(n - 1, 0), do_sqrt,
                                            out_src, out_dst, out_w, out_count);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

// kNN neighbours of single_linkage: min(m, max(2, floor(log2 m) + c))
static int64_t sl_neighbors(int64_t m, int64_t c)
{
  if (m < 1) return 0;
  const int64_t fl = 63 - __builtin_clzll(static_cast<unsigned long long>(m));
  return std::min<int64_t>(m, std::max<int64_t>(2, fl + c));
}

// Rows of x per masked arg-min launch of connect_components: the m x c adjacency bytes (and its m c / 8 bytes of bits)
// stay below 128 m, and the tile classes below 64 MiB; a multiple of TC_BM, at least TC_BM (c <= m).
static int64_t sl_max_chunk(int64_t m)
{
  const int64_t mm = std::max<int64_t>(m, 1);
  const int64_t cap = std::max<int64_t>(TC_BM, ((1ll << 40) / mm) / TC_BM * TC_BM);
  return std::min<int64_t>((mm + TC_BM - 1) / TC_BM * TC_BM, cap);
}

static int64_t sl_chunk_rows(int64_t m, int64_t c)
{
  const int64_t r = std::max<int64_t>(TC_BM, (128 * m / std::max<int64_t>(c, 1)) / TC_BM * TC_BM);
  return std::min(r, sl_max_chunk(m));
}

// Persistent regions first (the forest, the edge list, the host copies), then one scratch region used by the kNN phase
// and, afterwards, by connect_components.  Sized for any number of components up to m, so the workspace depends on
// (m, d, n_nb) only.
struct SlLayout {
  MstLayout mst;            // over the m rows
  int *src, *dst;           // [m n_nb + m] edge list: the kNN graph (position i n_nb + s), then the connecting edges
  float* w;                 //              squared L2 weights
  int *hsrc, *hdst;         // [m] forest edges in key order, for the host
  void* knn_ws;             // kNN phase: b2d_knn's workspace, then its outputs
  size_t knn_bytes;
  int64_t* idx;             // [m n_nb]
  float* dist;              // [m n_nb]
  TcWorkspace tc;           // connect phase: the colour-sorted rows as both operands
  float* xs;                // [m, d] the colour-sorted rows
  long long *keys, *cbest;  // [m] masked arg-min of every sorted row, [c] best row of every component
  unsigned* bad;            // [8] masked_classify's flag: 0 (the component ends are valid by construction)
  int *grp, *lab, *ends;    // [m]
  unsigned* ids;            // [m] root flags, scanned into dense component ids
  KmSort sort;              // the rows sorted by component, for up to m components
  unsigned* bits;           // [5 m] adjacency bits of one chunk
  uint8_t* cls;             // tile classes of one chunk
  uint8_t* adj;             // [128 m] adjacency of one chunk
  size_t bytes;
};

static SlLayout sl_layout(void* base, int64_t m, int64_t d, int64_t n_nb)
{
  Carve c(base, 1024);
  SlLayout L{};
  L.mst  = mst_regions(c, m);
  const size_t ne = static_cast<size_t>(m) * n_nb + m;
  L.src  = c.take<int>(ne);
  L.dst  = c.take<int>(ne);
  L.w    = c.take<float>(ne);
  L.hsrc = c.take<int>(m);
  L.hdst = c.take<int>(m);
  char* scratch = base ? static_cast<char*>(base) + c.bytes : nullptr;
  // kNN phase
  const KnnLayout K = knn_layout(nullptr, m, m, d, n_nb);
  Carve a(scratch, 1024);
  L.knn_ws    = a.take<char>(K.bytes);
  L.knn_bytes = K.bytes;
  L.idx       = a.take<int64_t>(static_cast<size_t>(m) * n_nb);
  L.dist      = a.take<float>(static_cast<size_t>(m) * n_nb);
  // connect phase
  Carve b(scratch, 1024);
  L.tc    = tc_layout(b, m, m, d, false);
  L.xs    = b.take<float>(static_cast<size_t>(m) * d);
  L.keys  = b.take<long long>(m);
  L.cbest = b.take<long long>(m);
  L.bad   = b.take<unsigned>(8);
  L.grp   = b.take<int>(m);
  L.lab   = b.take<int>(m);
  L.ends  = b.take<int>(m);
  L.ids   = b.take<unsigned>(m);
  L.sort  = km_sort_regions(b, m, m, true);
  const int64_t mm = std::max<int64_t>(m, 1);
  L.bits  = b.take<unsigned>(static_cast<size_t>(5) * mm);
  L.cls   = b.take<uint8_t>(static_cast<size_t>(sl_max_chunk(m) / TC_BM) * ((mm + TC_BN - 1) / TC_BN));
  L.adj   = b.take<uint8_t>(static_cast<size_t>(128) * mm);
  L.bytes = c.bytes + std::max(a.bytes, b.bytes);
  return L;
}

// One round of connect_components for c > 1 components: dense component ids in order of each component's smallest row,
// the rows sorted by component (stable), the masked arg-min of every sorted row against the rows of other components in
// row chunks, and for every component the edge from its row of smallest (distance, row) to that row's nearest row:
// edges [e0, e0 + c).  The arg-min takes the smallest sorted position among equidistant rows, so the nearest row's
// ties go to the first in (smallest row of its component, row) order.
static int sl_connect(cudaStream_t s, const SlLayout& L, const float* x, int64_t ldx, int64_t m, int64_t d, int64_t c,
                      int64_t e0)
{
  const MstLayout& T = L.mst;
  const KmSort& S = L.sort;
  int* minv = L.ends;   // [m] the smallest row of every component, by root (ends is written after the sort)
  sl_tree_min_init_kernel<<<sl_grid(m), 256, 0, s>>>(T.colour, minv, m);
  sl_min_vertex_kernel<<<sl_grid(m), 256, 0, s>>>(T.colour, minv, m);
  sl_root_flags_kernel<<<sl_grid(m), 256, 0, s>>>(T.colour, minv, L.ids, m);
  int rc = km_scan(s, nullptr, L.ids, m, S.tiles, S.ctrl);
  if (rc) return rc;
  sl_dense_label_kernel<<<sl_grid(m), 256, 0, s>>>(T.colour, minv, L.ids, L.lab, m);
  B2D_CUDA(cudaGetLastError());
  const KmSortPlan P = km_sort_plan(m, c);
  rc = km_sort_count(s, S, P, L.lab, m, c);
  if (rc) return rc;
  rc = km_sort_scatter(s, nullptr, S, P, L.lab, m, c);
  if (rc) return rc;
  sl_ends_kernel<<<sl_grid(c), 256, 0, s>>>(S.hist, P.nblk, c, L.ends);
  km_gather_rows(s, static_cast<unsigned>(m), x, ldx, static_cast<int>(d), S.perm, static_cast<int>(m), L.xs);
  B2D_CUDA(cudaGetLastError());
  // y (and x) prepared once per round; every chunk takes a window of the x side
  rc = launch_prep<float>(s, L.tc, L.xs, d, 1, m, L.xs, d, 1, m, d, nullptr, nullptr, TC_L2);
  if (rc) return rc;
  masked_group_map(s, sl_grid(m), L.grp, L.ends, c, m);
  B2D_CUDA(cudaMemsetAsync(L.bad, 0, 32, s));
  minloc_init(s, sl_grid(m), L.keys, m);
  minloc_init(s, sl_grid(c), L.cbest, c);
  B2D_CUDA(cudaGetLastError());
  const int64_t mc = sl_chunk_rows(m, c);
  for (int64_t r0 = 0; r0 < m; r0 += mc) {
    const int64_t rows = std::min(mc, m - r0);
    sl_adj_kernel<<<km_grid(rows * c), 256, 0, s>>>(S.slab, r0, rows, c, L.adj);
    B2D_CUDA(cudaGetLastError());
    rc = masked_keys(s, tc_rows(L.tc, 0, r0, d), L.keys + r0, L.grp, L.bits, L.cls, L.bad, L.adj, c, L.ends, c, rows, m, d);
    if (rc) return rc;
  }
  sl_comp_best_kernel<<<sl_grid(m), 256, 0, s>>>(L.keys, S.slab, m, L.cbest);
  sl_connect_kernel<<<sl_grid(c), 256, 0, s>>>(L.cbest, L.keys, S.perm, S.slab, c, e0, L.src, L.dst, L.w, T.ctrl);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

static int sl_read_ctrl(cudaStream_t s, const SlCtrl* d, SlCtrl* h)
{
  B2D_CUDA(cudaMemcpyAsync(h, d, sizeof(SlCtrl), cudaMemcpyDeviceToHost, s));
  B2D_CUDA(cudaStreamSynchronize(s));
  return B2D_OK;
}

// Step 5 of single_linkage: the m - 1 tree edges (hs[t], hd[t]) in key order merged on the host into children, sizes and
// labels (device pointers; children and sizes unused for m = 1).  Synchronises the stream.
static int sl_dendrogram(cudaStream_t s, int64_t m, int64_t n_clusters, const std::vector<int>& hs,
                         const std::vector<int>& hd, int32_t* children, int32_t* sizes, int32_t* labels)
{
  std::vector<int> hch(2 * (m - 1)), hsz(m - 1), hlab(m);
  // labels: the components after the first m - n_clusters merges
  if (!sl_merges(m, hs.data(), hd.data(), hch.data(), hsz.data(), m - n_clusters, hlab.data()))
    return fail(B2D_ERR_CUDA, "internal: the spanning tree has a cycle");
  std::vector<int> num(m, -1);   // numbered in order of each cluster's smallest row
  int next_label = 0;
  for (int64_t i = 0; i < m; ++i) {
    int& l = num[hlab[i]];
    if (l < 0) l = next_label++;
    hlab[i] = l;
  }
  if (m > 1) {
    B2D_CUDA(cudaMemcpyAsync(children, hch.data(), hch.size() * sizeof(int), cudaMemcpyHostToDevice, s));
    B2D_CUDA(cudaMemcpyAsync(sizes, hsz.data(), hsz.size() * sizeof(int), cudaMemcpyHostToDevice, s));
  }
  B2D_CUDA(cudaMemcpyAsync(labels, hlab.data(), m * sizeof(int), cudaMemcpyHostToDevice, s));
  B2D_CUDA(cudaStreamSynchronize(s));
  return B2D_OK;
}

// ------------------------------------------------------------------------------------------
// The exact EMST of 2-D and 3-D points (single_linkage_rbc.cuh): the ball-cover index of x, then Borůvka rounds whose
// edges come from a cross-component 1-NN walk over it.  Only enqueues work.

// The index, then the build's scratch, which is dead once the index is built: the rounds' arrays overlap it.
struct EmstLayout {
  BcIndex ix;
  BcBuildLayout build;
  SlCtrl* ctrl;
  int* colour;        // [m] component of every position (the position of its root)
  int* parent;        // [m] hook forest of a round
  int* pos;           // [m] the position of every caller row
  int* bcol;          // [nl] the single colour of every ball, or -1
  long long* best1;   // [m] per component: min of (s, min row)
  int* best2;         // [m] per component: min of the max row at best1
  long long* cand1;   // [m] per position: its row's candidate (s, min row) ... (the sort's second key buffer after the rounds)
  int* cand2;         // [m] ... and max row (the sort's second value buffer)
  long long* mst1;    // [m] the tree edges as appended: (s, min row) ...
  int* mst2;          // [m] ... and max row
  int *hsrc, *hdst;   // [m] single_linkage_rbc: the edges in order, for the host
  float* core;        // [m] HDBSCAN: the core distance of every position ...
  float* cmin;        // [nl] ... and the smallest of every ball
  void* sort_tmp;
  size_t sort_bytes;
  size_t bytes;
};

static EmstLayout emst_layout(void* base, int64_t m, int64_t d, int64_t nl, bool host_edges, bool mr = false)
{
  BcOverlay o(base, m, d, nl);
  Carve& c = o.rest;
  EmstLayout L{};
  L.ix     = o.ix;
  L.build  = o.build;
  L.ctrl   = c.take<SlCtrl>(1);
  L.colour = c.take<int>(m);
  L.parent = c.take<int>(m);
  L.pos    = c.take<int>(m);
  L.bcol   = c.take<int>(nl);
  L.best1  = c.take<long long>(m);
  L.best2  = c.take<int>(m);
  L.cand1  = c.take<long long>(m);
  L.cand2  = c.take<int>(m);
  L.mst1   = c.take<long long>(m);
  L.mst2   = c.take<int>(m);
  if (host_edges) {
    L.hsrc = c.take<int>(m);
    L.hdst = c.take<int>(m);
  }
  if (mr) {
    L.core = c.take<float>(m);
    L.cmin = c.take<float>(nl);
  }
  L.sort_bytes = bc_sort_bytes(m);
  L.sort_tmp   = c.take<char>(L.sort_bytes);
  L.bytes      = o.bytes();
  return L;
}

// the checks b2d_emst_rbc and b2d_single_linkage_rbc share
static int emst_args(const char* fn, int metric, const float* x, int64_t ldx, int64_t m, int64_t d, int64_t nl)
{
  if (metric != B2D_L2Unexpanded && metric != B2D_L2SqrtUnexpanded)
    return fail(B2D_ERR_UNSUPPORTED, std::string(fn) + " supports the L2Unexpanded and L2SqrtUnexpanded metrics, got metric " +
                                         std::to_string(metric));
  if (m < 1 || nl < 0) return fail(B2D_ERR_INVALID_ARG, "m must be positive and n_landmarks non-negative");
  if (d != 2 && d != 3) return fail(B2D_ERR_UNSUPPORTED, std::string(fn) + " supports d = 2 and d = 3, got d = " + std::to_string(d));
  if (m >= kSlMaxRows) return fail(B2D_ERR_UNSUPPORTED, std::string(fn) + ": m must be below 2^30");
  if (nl > m) return fail(B2D_ERR_INVALID_ARG, "n_landmarks must be in [0, m] (0: ceil(sqrt(m)))");
  if (!x) return fail(B2D_ERR_INVALID_ARG, "null x");
  if (ldx < d) return fail(B2D_ERR_INVALID_ARG, "leading dimension smaller than d");
  return B2D_OK;
}

static bool emst_extents_ok(int64_t m, int64_t d, int64_t nl)
{
  return m >= 1 && m < kSlMaxRows && (d == 2 || d == 3) && nl >= 0 && nl <= m;
}

// The index, the rounds, and the m - 1 tree edges sorted into (s, min row, max row) order as (out_src, out_dst, out_w).
// min_samples > 0 (HDBSCAN): the core distances first, and the rounds weigh pairs by mutual reachability, (s, ...)
// reading (w, ...).
template <int D>
static int emst_run(cudaStream_t s, const EmstLayout& L, int root, const float* x, int64_t ldx, int n, int nl,
                    uint64_t seed, int* out_src, int* out_dst, float* out_w, int min_samples = 0)
{
  int rc = bc_build<D>(s, L.ix, L.build, x, ldx, n, nl, seed);
  if (rc) return rc;
  // (after the build: its scratch lies under these arrays)
  sl_mst_init_kernel<<<sl_grid(n), 256, 0, s>>>(L.ctrl, L.colour, L.mst1, n);
  slr_pos_kernel<<<sl_grid(n), 256, 0, s>>>(L.ix.ids, n, L.pos);
  B2D_CUDA(cudaGetLastError());
  if (n < 2) return B2D_OK;
  const unsigned bg = static_cast<unsigned>((nl + kBcWarps - 1) / kBcWarps);
  if (min_samples > 0) {
    rc = bc_walk_launch(s, hdb_core_kernel<D>, n, nl, D, L.ix, n, nl, min_samples, L.core);
    if (rc) return rc;
    hdb_cmin_kernel<<<bg, kBcWarps * 32, 0, s>>>(L.ix.off, L.core, nl, L.cmin);
    B2D_CUDA(cudaGetLastError());
  }
  const int rounds  = ceil_log2(n) + 1;   // the components at least halve in every round
  const int jumps   = std::min(kSlMaxJumps, ceil_log2(n) + 1);
  for (int r = 0; r < rounds; ++r) {
    sl_round_begin_kernel<<<sl_grid(std::max<int64_t>(n, kSlMaxJumps)), 256, 0, s>>>(L.ctrl, L.best1, n);
    slr_ball_kernel<<<bg, kBcWarps * 32, 0, s>>>(L.ctrl, L.ix.off, L.colour, nl, L.bcol);
    if (min_samples > 0)
      rc = bc_walk_launch(s, hdb_walk_kernel<D>, n, nl, D, L.ctrl, L.ix, n, nl, L.colour, L.bcol, L.core, L.cmin,
                          L.best1, L.best2, L.cand1, L.cand2);
    else
      rc = bc_walk_launch(s, slr_walk_kernel<D>, n, nl, D, L.ctrl, L.ix, n, nl, L.colour, L.bcol, L.best1, L.best2,
                          L.cand1, L.cand2);
    if (rc) return rc;
    slr_tie_kernel<<<sl_grid(n), 256, 0, s>>>(L.ctrl, L.colour, L.cand1, L.cand2, L.best1, L.best2, n);
    slr_hook_kernel<<<sl_grid(n), 256, 0, s>>>(L.ctrl, L.colour, L.pos, L.best1, L.best2, L.parent, L.mst1, L.mst2, n);
    for (int j = 0; j < jumps; ++j) sl_jump_kernel<<<sl_grid(n), 256, 0, s>>>(L.ctrl, L.colour, L.parent, n, j);
    sl_relabel_kernel<<<sl_grid(n), 256, 0, s>>>(L.ctrl, L.colour, L.parent, n);
    sl_round_end_kernel<<<1, 1, 0, s>>>(L.ctrl);
    B2D_CUDA(cudaGetLastError());
  }
  // the edges in (s, min row, max row) order: stable radix sorts by the max row, then by (s, min row)
  const int ne = n - 1;
  cub::DoubleBuffer<int> k2(L.mst2, L.cand2);
  cub::DoubleBuffer<long long> k1(L.mst1, L.cand1);
  size_t need = 0;
  B2D_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, need, k2, k1, ne, 0, 32, s));
  if (need > L.sort_bytes) return fail(B2D_ERR_WORKSPACE, "internal: radix sort scratch " + std::to_string(need) + " bytes");
  B2D_CUDA(cub::DeviceRadixSort::SortPairs(L.sort_tmp, need, k2, k1, ne, 0, 32, s));
  B2D_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, need, k1, k2, ne, 0, 64, s));
  if (need > L.sort_bytes) return fail(B2D_ERR_WORKSPACE, "internal: radix sort scratch " + std::to_string(need) + " bytes");
  B2D_CUDA(cub::DeviceRadixSort::SortPairs(L.sort_tmp, need, k1, k2, ne, 0, 64, s));
  slr_emit_kernel<<<sl_grid(ne), 256, 0, s>>>(L.ctrl, k1.Current(), k2.Current(), ne, root, out_src, out_dst, out_w);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

// The model of b2d_hdbscan_rbc_fit_model (256-byte aligned regions): the fit's index (bc_layout, so one copy moves it),
// then HdbModel's arrays, the clusters bounded by m.
struct HdbModelLayout {
  HdbModel M;
  size_t index_bytes;
  size_t bytes;
};

static HdbModelLayout hdb_model_layout(void* base, int64_t m, int64_t d, int64_t nl)
{
  const BcLayout I = bc_layout(base, m, d, nl);
  Carve c(base ? static_cast<char*>(base) + I.bytes : nullptr, 256);
  HdbModelLayout L{};
  L.M.ix         = I.ix;
  L.index_bytes  = I.bytes;
  L.M.core       = c.take<float>(m);
  L.M.cmin       = c.take<float>(nl);
  L.M.pos        = c.take<int>(m);
  L.M.row_parent = c.take<int>(m);
  L.M.row_lambda = c.take<double>(m);
  L.M.parent     = c.take<int>(m);
  L.M.owner      = c.take<int>(m);
  L.M.label      = c.take<int>(m);
  L.M.birth      = c.take<double>(m);
  L.M.death      = c.take<double>(m);
  L.M.head       = c.take<HdbModelHead>(1);
  L.bytes        = I.bytes + c.bytes;
  return L;
}

static int emst_dispatch(cudaStream_t s, const EmstLayout& L, int metric, const float* x, int64_t ldx, int64_t m,
                         int64_t d, int64_t nl, uint64_t seed, int* out_src, int* out_dst, float* out_w,
                         int min_samples = 0)
{
  const int root = metric == B2D_L2SqrtUnexpanded;
  const int n = static_cast<int>(m), l = static_cast<int>(nl);
  return d == 2 ? emst_run<2>(s, L, root, x, ldx, n, l, seed, out_src, out_dst, out_w, min_samples)
                : emst_run<3>(s, L, root, x, ldx, n, l, seed, out_src, out_dst, out_w, min_samples);
}
}  // namespace

size_t b2d_mst_workspace_bytes(int64_t n_vertices, int64_t n_edges)
{
  if (n_vertices < 0 || n_edges < 0) return static_cast<size_t>(-1);
  return mst_layout(nullptr, n_vertices).bytes;
}

int b2d_mst(void* stream, const int32_t* src, const int32_t* dst, const float* w, int64_t n_vertices, int64_t n_edges,
            int32_t* out_src, int32_t* out_dst, float* out_w, int32_t* out_colour, int32_t* out_count, void* workspace,
            size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int64_t n = n_vertices, E = n_edges;
  if (n < 0 || E < 0) return fail(B2D_ERR_INVALID_ARG, "negative extent");
  if (n >= kSlMaxRows) return fail(B2D_ERR_UNSUPPORTED, "mst: n_vertices must be below 2^30");
  if (E >= kSlMaxEdges) return fail(B2D_ERR_UNSUPPORTED, "mst: n_edges must be below 2^32 - 1");
  if (E > 0 && (!src || !dst || !w)) return fail(B2D_ERR_INVALID_ARG, "null src / dst / w");
  if (!out_count || (n > 0 && !out_colour) || (n > 1 && (!out_src || !out_dst || !out_w)))
    return fail(B2D_ERR_INVALID_ARG, "null out_src / out_dst / out_w / out_colour / out_count");
  int rc = check_workspace(workspace, workspace_bytes, mst_layout(nullptr, n).bytes);
  if (rc) return rc;
  if (n == 0) {
    B2D_CUDA(cudaMemsetAsync(out_count, 0, sizeof(int32_t), s));
    return B2D_OK;
  }
  const MstLayout L = mst_layout(workspace, n);
  sl_mst_init_kernel<<<sl_grid(n), 256, 0, s>>>(L.ctrl, L.colour, L.keys, n);
  B2D_CUDA(cudaGetLastError());
  rc = mst_rounds(s, L, src, dst, w, n, 0, E, n);
  if (rc) return rc;
  rc = mst_emit(s, L, src, dst, w, n, 0, out_src, out_dst, out_w, out_count);
  if (rc) return rc;
  sl_fill_kernel<<<sl_grid(n), 256, 0, s>>>(L.parent, 0x7fffffff, n);
  sl_min_vertex_kernel<<<sl_grid(n), 256, 0, s>>>(L.colour, L.parent, n);
  sl_colour_out_kernel<<<sl_grid(n), 256, 0, s>>>(L.colour, L.parent, out_colour, n);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

size_t b2d_single_linkage_workspace_bytes(int64_t m, int64_t d, int c)
{
  if (m < 0 || d < 0) return static_cast<size_t>(-1);
  const int64_t n_nb = sl_neighbors(m, c);
  if (n_nb > KNN_MAX_K || m >= kSlMaxRows) return static_cast<size_t>(-1);
  return sl_layout(nullptr, m, d, n_nb).bytes;
}

int b2d_single_linkage(void* stream, int metric, const float* x, int64_t ldx, int64_t m, int64_t d, int c, int n_clusters,
                       int32_t* children, float* deltas, int32_t* sizes, int32_t* labels, int32_t* n_components_out,
                       void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (metric != B2D_L2Expanded && metric != B2D_L2SqrtExpanded)
    return fail(B2D_ERR_UNSUPPORTED, "single_linkage supports the L2Expanded and L2SqrtExpanded metrics");
  if (m < 1 || d < 1) return fail(B2D_ERR_INVALID_ARG, "m and d must be positive");
  if (d > 320) return fail(B2D_ERR_UNSUPPORTED, "single_linkage supports d <= 320 (the fused kNN's limit)");
  if (m >= kSlMaxRows) return fail(B2D_ERR_UNSUPPORTED, "single_linkage: m must be below 2^30");
  if (n_clusters < 1 || n_clusters > m) return fail(B2D_ERR_INVALID_ARG, "n_clusters must be in [1, m]");
  const int64_t n_nb = sl_neighbors(m, c);
  if (n_nb > KNN_MAX_K)
    return fail(B2D_ERR_UNSUPPORTED, "single_linkage: min(m, max(2, floor(log2 m) + c)) = " + std::to_string(n_nb) +
                                         " neighbours exceeds 64: lower c (" + std::to_string(c) + ")");
  if (m * n_nb + m >= kSlMaxEdges)
    return fail(B2D_ERR_UNSUPPORTED, "single_linkage: m * (n_nb + 1) edges must stay below 2^32 - 1");
  if (!x || !labels || !n_components_out || (m > 1 && (!children || !deltas || !sizes)))
    return fail(B2D_ERR_INVALID_ARG, "null x / children / deltas / sizes / labels / n_components_out");
  if (ldx < d) return fail(B2D_ERR_INVALID_ARG, "leading dimension smaller than d");
  int rc = check_workspace(workspace, workspace_bytes, sl_layout(nullptr, m, d, n_nb).bytes);
  if (rc) return rc;
  const SlLayout L = sl_layout(workspace, m, d, n_nb);
  const MstLayout& T = L.mst;
  SlCtrl h;
  sl_mst_init_kernel<<<sl_grid(m), 256, 0, s>>>(T.ctrl, T.colour, T.keys, m);
  sl_finite_kernel<<<km_grid(m * d), 256, 0, s>>>(x, ldx, m, static_cast<int>(d), T.ctrl);
  B2D_CUDA(cudaGetLastError());
  // 1. the kNN graph (squared distances, whatever the metric)
  if (m > 1) {
    rc = b2d_knn(s, L.idx, L.dist, B2D_L2Expanded, x, ldx, x, ldx, m, m, d, n_nb, L.knn_ws, L.knn_bytes);
    if (rc) return rc;
    sl_knn_edges_kernel<<<sl_grid(m * n_nb), 256, 0, s>>>(L.idx, L.dist, m, static_cast<int>(n_nb), L.src, L.dst, L.w);
    B2D_CUDA(cudaGetLastError());
    // 2.-3. its minimum spanning forest
    rc = mst_rounds(s, T, L.src, L.dst, L.w, m, 0, m * n_nb, m);
    if (rc) return rc;
  }
  rc = sl_read_ctrl(s, T.ctrl, &h);
  if (rc) return rc;
  if (h.bad & 1u) return fail(B2D_ERR_INVALID_ARG, "single_linkage: X holds a non-finite value");
  int64_t comps = m - h.n_mst;
  *n_components_out = static_cast<int32_t>(comps);
  // 4. connect_components: each round at least halves the components
  int64_t e = m * n_nb;
  while (comps > 1) {
    rc = sl_connect(s, L, x, ldx, m, d, comps, e);
    if (rc) return rc;
    sl_rearm_kernel<<<1, 1, 0, s>>>(T.ctrl);
    B2D_CUDA(cudaGetLastError());
    rc = mst_rounds(s, T, L.src, L.dst, L.w, m, e, e + comps, comps);
    if (rc) return rc;
    e += comps;
    rc = sl_read_ctrl(s, T.ctrl, &h);
    if (rc) return rc;
    const int64_t next = m - h.n_mst;
    if ((h.bad & 2u) || 2 * next > comps)
      return fail(B2D_ERR_CUDA, "internal: connect_components left " + std::to_string(next) + " of " +
                                    std::to_string(comps) + " components");
    comps = next;
  }
  // 5. dendrogram: the m - 1 forest edges in key order, union-find on the host
  std::vector<int> hs(m - 1), hd(m - 1);
  if (m > 1) {
    rc = mst_emit(s, T, L.src, L.dst, L.w, m, metric == B2D_L2SqrtExpanded ? 1 : 0, L.hsrc, L.hdst, deltas, nullptr);
    if (rc) return rc;
    B2D_CUDA(cudaMemcpyAsync(hs.data(), L.hsrc, (m - 1) * sizeof(int), cudaMemcpyDeviceToHost, s));
    B2D_CUDA(cudaMemcpyAsync(hd.data(), L.hdst, (m - 1) * sizeof(int), cudaMemcpyDeviceToHost, s));
    B2D_CUDA(cudaStreamSynchronize(s));
  }
  return sl_dendrogram(s, m, n_clusters, hs, hd, children, sizes, labels);
}

int b2d_debug_single_linkage_plan(int64_t m, int64_t comps, int64_t* out)
{
  if (!out) return fail(B2D_ERR_INVALID_ARG, "null out");
  if (m < 2 || m >= kSlMaxRows) return fail(B2D_ERR_INVALID_ARG, "m must be in [2, 2^30)");
  if (comps < 2 || comps > m) return fail(B2D_ERR_INVALID_ARG, "comps must be in [2, m]");
  const int64_t mc = sl_chunk_rows(m, comps);
  const KmSortPlan P = km_sort_plan(m, comps);
  out[0] = mc;
  out[1] = (m + mc - 1) / mc;
  out[2] = P.rb;
  out[3] = P.nblk;
  return B2D_OK;
}

size_t b2d_emst_rbc_workspace_bytes(int64_t m, int64_t d, int64_t n_landmarks)
{
  if (!emst_extents_ok(m, d, n_landmarks)) return static_cast<size_t>(-1);
  return emst_layout(nullptr, m, d, bc_landmarks(m, n_landmarks), false).bytes;
}

int b2d_emst_rbc(void* stream, int metric, const float* x, int64_t ldx, int64_t m, int64_t d, int64_t n_landmarks,
                 uint64_t seed, int32_t* out_src, int32_t* out_dst, float* out_w, void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  int rc         = emst_args("emst rbc", metric, x, ldx, m, d, n_landmarks);
  if (rc) return rc;
  if (m > 1 && (!out_src || !out_dst || !out_w)) return fail(B2D_ERR_INVALID_ARG, "null out_src / out_dst / out_w");
  const int64_t nl = bc_landmarks(m, n_landmarks);
  rc = check_workspace(workspace, workspace_bytes, emst_layout(nullptr, m, d, nl, false).bytes);
  if (rc) return rc;
  const EmstLayout L = emst_layout(workspace, m, d, nl, false);
  return emst_dispatch(s, L, metric, x, ldx, m, d, nl, seed, out_src, out_dst, out_w);
}

size_t b2d_single_linkage_rbc_workspace_bytes(int64_t m, int64_t d, int64_t n_landmarks)
{
  if (!emst_extents_ok(m, d, n_landmarks)) return static_cast<size_t>(-1);
  return emst_layout(nullptr, m, d, bc_landmarks(m, n_landmarks), true).bytes;
}

int b2d_single_linkage_rbc(void* stream, int metric, const float* x, int64_t ldx, int64_t m, int64_t d,
                           int64_t n_landmarks, uint64_t seed, int n_clusters, int32_t* children, float* deltas,
                           int32_t* sizes, int32_t* labels, void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  int rc         = emst_args("single_linkage rbc", metric, x, ldx, m, d, n_landmarks);
  if (rc) return rc;
  if (n_clusters < 1 || n_clusters > m) return fail(B2D_ERR_INVALID_ARG, "n_clusters must be in [1, m]");
  if (!labels || (m > 1 && (!children || !deltas || !sizes)))
    return fail(B2D_ERR_INVALID_ARG, "null children / deltas / sizes / labels");
  const int64_t nl = bc_landmarks(m, n_landmarks);
  rc = check_workspace(workspace, workspace_bytes, emst_layout(nullptr, m, d, nl, true).bytes);
  if (rc) return rc;
  const EmstLayout L = emst_layout(workspace, m, d, nl, true);
  // 1.-3. the tree edges in order, their weights (the metric's distance) straight into deltas
  rc = emst_dispatch(s, L, metric, x, ldx, m, d, nl, seed, L.hsrc, L.hdst, deltas);
  if (rc) return rc;
  sl_finite_kernel<<<km_grid(m * d), 256, 0, s>>>(x, ldx, m, static_cast<int>(d), L.ctrl);
  B2D_CUDA(cudaGetLastError());
  // 4. the dendrogram on the host (the one synchronisation before it reads the control words and the edges)
  SlCtrl h;
  std::vector<int> hs(m - 1), hd(m - 1);
  B2D_CUDA(cudaMemcpyAsync(&h, L.ctrl, sizeof(SlCtrl), cudaMemcpyDeviceToHost, s));
  if (m > 1) {
    B2D_CUDA(cudaMemcpyAsync(hs.data(), L.hsrc, (m - 1) * sizeof(int), cudaMemcpyDeviceToHost, s));
    B2D_CUDA(cudaMemcpyAsync(hd.data(), L.hdst, (m - 1) * sizeof(int), cudaMemcpyDeviceToHost, s));
  }
  B2D_CUDA(cudaStreamSynchronize(s));
  if (h.bad & 1u) return fail(B2D_ERR_INVALID_ARG, "single_linkage rbc: X holds a non-finite value");
  if (m > 1 && h.n_mst != static_cast<unsigned>(m - 1))
    return fail(B2D_ERR_CUDA, "internal: the rounds chose " + std::to_string(h.n_mst) + " of " + std::to_string(m - 1) +
                                  " tree edges");
  return sl_dendrogram(s, m, n_clusters, hs, hd, children, sizes, labels);
}

// ------------------------------------------------------------------------------------------
// HDBSCAN of 2-D and 3-D points (hdbscan_rbc.cuh, hdbscan_tree.cuh): the core distances and the mutual-reachability tree
// by the EMST's rounds, then the tree stages on the host.

size_t b2d_hdbscan_rbc_workspace_bytes(int64_t m, int64_t d, int64_t n_landmarks)
{
  if (!emst_extents_ok(m, d, n_landmarks)) return static_cast<size_t>(-1);
  return emst_layout(nullptr, m, d, bc_landmarks(m, n_landmarks), false, true).bytes;
}

size_t b2d_hdbscan_rbc_model_bytes(int64_t m, int64_t d, int64_t n_landmarks)
{
  if (!emst_extents_ok(m, d, n_landmarks)) return static_cast<size_t>(-1);
  return hdb_model_layout(nullptr, m, d, bc_landmarks(m, n_landmarks)).bytes;
}

namespace {
// b2d_hdbscan_rbc_fit, and with with_model b2d_hdbscan_rbc_fit_model, whose model is checked after the fit's arguments
int hdbscan_fit(void* stream, int metric, const float* x, int64_t ldx, int64_t m, int64_t d, int min_samples,
                int min_cluster_size, double cluster_selection_epsilon, int method, int allow_single_cluster,
                int64_t n_landmarks, uint64_t seed, int32_t* labels, float* probabilities, int32_t* mst_src,
                int32_t* mst_dst, float* mst_w, int32_t* n_clusters, void* workspace, size_t workspace_bytes, void* model,
                bool with_model)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  int rc         = emst_args("hdbscan rbc", metric, x, ldx, m, d, n_landmarks);
  if (rc) return rc;
  if (min_samples < 1 || min_samples > std::min<int64_t>(KNN_MAX_K, m))
    return fail(B2D_ERR_INVALID_ARG, "min_samples must be in [1, min(64, m)], got " + std::to_string(min_samples));
  if (min_cluster_size < 2)
    return fail(B2D_ERR_INVALID_ARG, "min_cluster_size must be at least 2, got " + std::to_string(min_cluster_size));
  if (!(cluster_selection_epsilon >= 0.0) || std::isinf(cluster_selection_epsilon))
    return fail(B2D_ERR_INVALID_ARG, "cluster_selection_epsilon must be finite and non-negative");
  if (method != B2D_HDBSCAN_EOM && method != B2D_HDBSCAN_LEAF)
    return fail(B2D_ERR_INVALID_ARG, "method must be B2D_HDBSCAN_EOM or B2D_HDBSCAN_LEAF, got " + std::to_string(method));
  if (allow_single_cluster != 0 && allow_single_cluster != 1)
    return fail(B2D_ERR_INVALID_ARG, "allow_single_cluster must be 0 or 1");
  if (!labels || !probabilities || !n_clusters || (m > 1 && (!mst_src || !mst_dst || !mst_w)))
    return fail(B2D_ERR_INVALID_ARG, "null labels / probabilities / mst_src / mst_dst / mst_w / n_clusters");
  const int64_t nl = bc_landmarks(m, n_landmarks);
  rc = check_workspace(workspace, workspace_bytes, emst_layout(nullptr, m, d, nl, false, true).bytes);
  if (rc) return rc;
  if (with_model && !model) return fail(B2D_ERR_INVALID_ARG, "null model");
  if (with_model && reinterpret_cast<uintptr_t>(model) % 256)
    return fail(B2D_ERR_INVALID_ARG, "model must be 256-byte aligned");
  const EmstLayout L = emst_layout(workspace, m, d, nl, false, true);
  // 1.-2. the index, the core distances and the tree edges in (w, min row, max row) order
  rc = emst_dispatch(s, L, metric, x, ldx, m, d, nl, seed, mst_src, mst_dst, mst_w, min_samples);
  if (rc) return rc;
  const HdbModelLayout ML = hdb_model_layout(model, m, d, nl);
  if (model) {   // the index lies at the workspace's start in the model's own layout
    B2D_CUDA(cudaMemcpyAsync(model, workspace, ML.index_bytes, cudaMemcpyDeviceToDevice, s));
    B2D_CUDA(cudaMemcpyAsync(ML.M.pos, L.pos, m * sizeof(int), cudaMemcpyDeviceToDevice, s));
    if (m > 1) {
      B2D_CUDA(cudaMemcpyAsync(ML.M.core, L.core, m * sizeof(float), cudaMemcpyDeviceToDevice, s));
      B2D_CUDA(cudaMemcpyAsync(ML.M.cmin, L.cmin, nl * sizeof(float), cudaMemcpyDeviceToDevice, s));
    } else {   // one row: its core distance is s(0, 0) = 0 (the rounds computed none)
      B2D_CUDA(cudaMemsetAsync(ML.M.core, 0, sizeof(float), s));
      B2D_CUDA(cudaMemsetAsync(ML.M.cmin, 0, nl * sizeof(float), s));
    }
  }
  sl_finite_kernel<<<km_grid(m * d), 256, 0, s>>>(x, ldx, m, static_cast<int>(d), L.ctrl);
  B2D_CUDA(cudaGetLastError());
  // 3. the tree stages on the host (the one synchronisation before it reads the control words and the edges)
  SlCtrl h;
  std::vector<int> hs(m - 1), hd(m - 1), hl(m);
  std::vector<float> hw(m - 1), hp(m);
  B2D_CUDA(cudaMemcpyAsync(&h, L.ctrl, sizeof(SlCtrl), cudaMemcpyDeviceToHost, s));
  if (m > 1) {
    B2D_CUDA(cudaMemcpyAsync(hs.data(), mst_src, (m - 1) * sizeof(int), cudaMemcpyDeviceToHost, s));
    B2D_CUDA(cudaMemcpyAsync(hd.data(), mst_dst, (m - 1) * sizeof(int), cudaMemcpyDeviceToHost, s));
    B2D_CUDA(cudaMemcpyAsync(hw.data(), mst_w, (m - 1) * sizeof(float), cudaMemcpyDeviceToHost, s));
  }
  B2D_CUDA(cudaStreamSynchronize(s));
  if (h.bad & 1u) return fail(B2D_ERR_INVALID_ARG, "hdbscan rbc: X holds a non-finite value");
  if (m > 1 && h.n_mst != static_cast<unsigned>(m - 1))
    return fail(B2D_ERR_CUDA, "internal: the rounds chose " + std::to_string(h.n_mst) + " of " + std::to_string(m - 1) +
                                  " tree edges");
  const HdbTreeParams P{min_cluster_size, cluster_selection_epsilon, method == B2D_HDBSCAN_LEAF, allow_single_cluster != 0};
  HdbTreeExport ex;
  const int nc = hdbscan_tree(m, hs.data(), hd.data(), hw.data(), P, hl.data(), hp.data(), model ? &ex : nullptr);
  if (nc < 0) return fail(B2D_ERR_CUDA, "internal: the spanning tree has a cycle");
  B2D_CUDA(cudaMemcpyAsync(labels, hl.data(), m * sizeof(int), cudaMemcpyHostToDevice, s));
  B2D_CUDA(cudaMemcpyAsync(probabilities, hp.data(), m * sizeof(float), cudaMemcpyHostToDevice, s));
  const size_t nci = ex.parent.size();
  const HdbModelHead head{ex.thr, ex.single_root ? 1 : 0, static_cast<int>(nci)};
  if (model) {
    const HdbModel& M = ML.M;
    B2D_CUDA(cudaMemcpyAsync(M.row_parent, ex.row_parent.data(), m * sizeof(int), cudaMemcpyHostToDevice, s));
    B2D_CUDA(cudaMemcpyAsync(M.row_lambda, ex.row_lambda.data(), m * sizeof(double), cudaMemcpyHostToDevice, s));
    B2D_CUDA(cudaMemcpyAsync(M.parent, ex.parent.data(), nci * sizeof(int), cudaMemcpyHostToDevice, s));
    B2D_CUDA(cudaMemcpyAsync(M.owner, ex.owner.data(), nci * sizeof(int), cudaMemcpyHostToDevice, s));
    B2D_CUDA(cudaMemcpyAsync(M.label, ex.label.data(), nci * sizeof(int), cudaMemcpyHostToDevice, s));
    B2D_CUDA(cudaMemcpyAsync(M.birth, ex.birth.data(), nci * sizeof(double), cudaMemcpyHostToDevice, s));
    B2D_CUDA(cudaMemcpyAsync(M.death, ex.death.data(), nci * sizeof(double), cudaMemcpyHostToDevice, s));
    B2D_CUDA(cudaMemcpyAsync(M.head, &head, sizeof(head), cudaMemcpyHostToDevice, s));
  }
  B2D_CUDA(cudaStreamSynchronize(s));
  *n_clusters = nc;
  return B2D_OK;
}
}  // namespace

int b2d_hdbscan_rbc_fit(void* stream, int metric, const float* x, int64_t ldx, int64_t m, int64_t d, int min_samples,
                        int min_cluster_size, double cluster_selection_epsilon, int method, int allow_single_cluster,
                        int64_t n_landmarks, uint64_t seed, int32_t* labels, float* probabilities, int32_t* mst_src,
                        int32_t* mst_dst, float* mst_w, int32_t* n_clusters, void* workspace, size_t workspace_bytes)
{
  return hdbscan_fit(stream, metric, x, ldx, m, d, min_samples, min_cluster_size, cluster_selection_epsilon, method,
                     allow_single_cluster, n_landmarks, seed, labels, probabilities, mst_src, mst_dst, mst_w, n_clusters,
                     workspace, workspace_bytes, nullptr, false);
}

int b2d_hdbscan_rbc_fit_model(void* stream, int metric, const float* x, int64_t ldx, int64_t m, int64_t d,
                              int min_samples, int min_cluster_size, double cluster_selection_epsilon, int method,
                              int allow_single_cluster, int64_t n_landmarks, uint64_t seed, int32_t* labels,
                              float* probabilities, int32_t* mst_src, int32_t* mst_dst, float* mst_w, int32_t* n_clusters,
                              void* workspace, size_t workspace_bytes, void* model)
{
  return hdbscan_fit(stream, metric, x, ldx, m, d, min_samples, min_cluster_size, cluster_selection_epsilon, method,
                     allow_single_cluster, n_landmarks, seed, labels, probabilities, mst_src, mst_dst, mst_w, n_clusters,
                     workspace, workspace_bytes, model, true);
}

int b2d_hdbscan_rbc_approximate_predict(void* stream, const void* model, int64_t m, int64_t d, int metric,
                                        int64_t n_landmarks, int min_samples, const float* q, int64_t ldq, int64_t mq,
                                        int32_t* labels, float* probabilities, int32_t* nn_rows, float* nn_w)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (metric != B2D_L2Unexpanded && metric != B2D_L2SqrtUnexpanded)
    return fail(B2D_ERR_UNSUPPORTED, "hdbscan approximate_predict supports the L2Unexpanded and L2SqrtUnexpanded metrics, "
                                     "got metric " + std::to_string(metric));
  if (d != 2 && d != 3)
    return fail(B2D_ERR_UNSUPPORTED, "hdbscan approximate_predict supports d = 2 and d = 3, got d = " + std::to_string(d));
  if (m < 1 || m >= kSlMaxRows) return fail(B2D_ERR_INVALID_ARG, "m must be in [1, 2^30)");
  if (n_landmarks < 0 || n_landmarks > m)
    return fail(B2D_ERR_INVALID_ARG, "n_landmarks must be in [0, m] (0: ceil(sqrt(m)))");
  if (min_samples < 1 || min_samples > std::min<int64_t>(KNN_MAX_K, m))
    return fail(B2D_ERR_INVALID_ARG, "min_samples must be in [1, min(64, m)], got " + std::to_string(min_samples));
  if (!model) return fail(B2D_ERR_INVALID_ARG, "null model");
  if (reinterpret_cast<uintptr_t>(model) % 256) return fail(B2D_ERR_INVALID_ARG, "model must be 256-byte aligned");
  if (mq < 0 || mq > 0x7fffffffll) return fail(B2D_ERR_INVALID_ARG, "mq must be in [0, 2^31)");
  if (mq > 0 && !q) return fail(B2D_ERR_INVALID_ARG, "null queries");
  if (ldq < d) return fail(B2D_ERR_INVALID_ARG, "ldq smaller than d");
  if (mq > 0 && (!labels || !probabilities)) return fail(B2D_ERR_INVALID_ARG, "null labels / probabilities");
  if (mq == 0) return B2D_OK;
  const int64_t nl = bc_landmarks(m, n_landmarks);
  const HdbModel M = hdb_model_layout(const_cast<void*>(model), m, d, nl).M;
  const int root   = metric == B2D_L2SqrtUnexpanded;
  const int n = static_cast<int>(m), nli = static_cast<int>(nl), mqi = static_cast<int>(mq);
  return d == 2 ? bc_walk_launch(s, hdb_predict_kernel<2>, mq, nl, d, M, n, nli, min_samples, root, q, ldq, mqi, labels,
                                 probabilities, nn_rows, nn_w)
                : bc_walk_launch(s, hdb_predict_kernel<3>, mq, nl, d, M, n, nli, min_samples, root, q, ldq, mqi, labels,
                                 probabilities, nn_rows, nn_w);
}
