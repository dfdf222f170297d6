// DBSCAN (dbscan.cuh) on the epsilon neighbourhood of the tensor path, and on the random ball cover for 2-D and 3-D points.
#include <cuda_runtime.h>
#include <algorithm>
#include <cmath>
#include <string>

#include "host.cuh"
#include "dbscan.cuh"

using namespace b2d;

// ------------------------------------------------------------------------------------------
// DBSCAN (dbscan.cuh): the epsilon neighbourhood of x against itself in column batches of the prepared rows, a device
// union-find over the core points and the border rule.  Only enqueues work.
namespace {
constexpr int64_t kDbDefaultBatchBytes = 1ll << 30;

// The degrees and the union-find forest of both fits, and the scans that number its roots and core rows.
struct DbForest {
  unsigned* deg;     // the degrees (db_core_kernel's layout)
  int* parent;       // [m] union-find forest over the core rows (-1: not core)
  int* border;       // [m] smallest root reaching a non-core row (INT_MAX: none)
  unsigned* root;    // [m] root flags, scanned into cluster numbers
  unsigned* core;    // [m] core flags, scanned into core_sample_indices positions
  unsigned* tiles;   // scan tile sums
  KmCtrl* ctrl;      // [2] scan totals: clusters, core rows
};

static DbForest db_forest(Carve& c, int64_t m, int64_t deg_rows)
{
  DbForest F;
  F.deg    = c.take<unsigned>(deg_rows);
  F.parent = c.take<int>(m);
  F.border = c.take<int>(m);
  F.root   = c.take<unsigned>(m);
  F.core   = c.take<unsigned>(m);
  F.tiles  = c.take<unsigned>((m + kKmScanTile - 1) / kKmScanTile);
  F.ctrl   = c.take<KmCtrl>(2);
  return F;
}

// the labels from the compressed forest and the border roots: cluster numbers = ranks of the roots, core_sample_indices
// positions = ranks of the core rows
static int db_label(cudaStream_t s, const DbForest& F, int64_t m, int32_t* labels, int32_t* core_sample_indices,
                    int32_t* n_clusters)
{
  int rc = km_scan(s, nullptr, F.root, m, F.tiles, F.ctrl);
  if (rc) return rc;
  rc = km_scan(s, nullptr, F.core, m, F.tiles, F.ctrl + 1);
  if (rc) return rc;
  db_label_kernel<<<sl_grid(m), 256, 0, s>>>(F.parent, F.border, F.root, F.core, m, &F.ctrl[0].total, &F.ctrl[1].total,
                                             labels, core_sample_indices, n_clusters);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

// columns per batch: min(m, max(256, floor(max_bytes / m / 256) * 256)); max_bytes 0 means 2^30
static int64_t db_batch(int64_t m, int64_t max_bytes)
{
  const int64_t mm = std::max<int64_t>(m, 1);
  const int64_t mb = max_bytes > 0 ? max_bytes : kDbDefaultBatchBytes;
  return std::min(mm, std::max<int64_t>(256, mb / mm / 256 * 256));
}

struct DbLayout {
  TcWorkspace tc;    // x prepared once, as both operands
  int64_t b, nb;     // columns per batch, batches
  int64_t ld;        // adjacency row pitch: b rounded up to 16
  DbForest f;        // deg [m + nb]: per-column degrees, each batch's total behind its columns
  uint8_t* adj;      // [m][ld] adjacency of one batch
  size_t bytes;
};

static DbLayout db_layout(void* base, int64_t m, int64_t d, int64_t max_bytes)
{
  Carve c(base, 1024);
  DbLayout L{};
  L.tc     = tc_layout(c, m, m, d, false);
  L.b      = db_batch(m, max_bytes);
  L.nb     = (m + L.b - 1) / L.b;
  L.ld     = (L.b + 15) / 16 * 16;
  L.f      = db_forest(c, m, m + L.nb);
  L.adj    = c.take<uint8_t>(static_cast<size_t>(m) * L.ld);
  L.bytes  = c.bytes;
  return L;
}

// One EPI_EPS launch over the columns [s, s + w) of the prepared x (batch t): the adjacency into L.adj (adj) and / or
// the degrees of those columns into deg[s + t, s + t + w] (deg).  diag_off = s keeps the self pairs.
static int db_eps(cudaStream_t s, const DbLayout& L, int64_t m, int64_t d, float e, int64_t t, bool adj, bool deg)
{
  const int64_t c0 = t * L.b, w = std::min(L.b, m - c0);
  TcParams p{};
  p.m = m; p.n = w;
  p.adj = adj ? L.adj : nullptr; p.ld_adj = L.ld;
  p.vd = deg ? L.f.deg + c0 + t : nullptr; p.vd64 = 0; p.eps = e;
  p.diag_off = c0;
  p.tma_store = (adj && w % 16 == 0) ? 1 : 0;   // (L.adj is 1024-byte aligned and L.ld a multiple of 16)
  return launch_tc(s, tc_rows(L.tc, 1, c0, d), p, d, EPI_EPS, POST_CLAMP);
}

static unsigned db_warp_grid(int64_t m) { return static_cast<unsigned>(std::min<int64_t>((m + 7) / 8, 1 << 16)); }
}  // namespace

size_t b2d_dbscan_workspace_bytes(int64_t m, int64_t d, int64_t max_bytes_per_batch)
{
  if (m < 0 || d < 0 || max_bytes_per_batch < 0) return static_cast<size_t>(-1);
  return db_layout(nullptr, m, d, max_bytes_per_batch).bytes;
}

int b2d_dbscan_fit(void* stream, int metric, const float* x, int64_t ldx, int64_t m, int64_t d, double eps,
                   int64_t min_samples, int64_t max_bytes_per_batch, int32_t* labels, int32_t* core_sample_indices,
                   int32_t* n_clusters, void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  TcMetric tm;
  if ((metric != B2D_L2SqrtExpanded && metric != B2D_L2Expanded && metric != B2D_CosineExpanded) || !tc_metric(metric, d, &tm))
    return fail(B2D_ERR_UNSUPPORTED, "dbscan supports the L2SqrtExpanded, L2Expanded and CosineExpanded metrics");
  if (m < 0 || d < 0 || max_bytes_per_batch < 0) return fail(B2D_ERR_INVALID_ARG, "negative extent or batch size");
  if (m == 0) return B2D_OK;
  if (m > 0x7fffffffll) return fail(B2D_ERR_INVALID_ARG, "dbscan: m must be below 2^31");
  if (d < 1) return fail(B2D_ERR_INVALID_ARG, "d must be positive");
  if (d > 320) return fail(B2D_ERR_UNSUPPORTED, "dbscan supports d <= 320 (the whole distance at once)");
  if (min_samples < 1) return fail(B2D_ERR_INVALID_ARG, "min_samples must be >= 1");
  if (!x || !labels) return fail(B2D_ERR_INVALID_ARG, "null x / labels");
  if (ldx < d) return fail(B2D_ERR_INVALID_ARG, "leading dimension smaller than d");
  int rc = check_workspace(workspace, workspace_bytes, db_layout(nullptr, m, d, max_bytes_per_batch).bytes);
  if (rc) return rc;
  const DbLayout L  = db_layout(workspace, m, d, max_bytes_per_batch);
  const DbForest& F = L.f;
  // the threshold on the distance the kernel compares: eps^2 (rounded once from fp64) for L2SqrtExpanded; a NaN or
  // negative eps matches nothing (every distance is >= 0 or NaN)
  const float e = !(eps >= 0.0) ? -INFINITY : static_cast<float>(metric == B2D_L2SqrtExpanded ? eps * eps : eps);
  const unsigned ms = static_cast<unsigned>(std::min<int64_t>(min_samples, m + 1));
  // 0. x prepared once, as both operands; every batch takes a window of the y side
  rc = launch_prep<float>(s, L.tc, x, ldx, 1, m, x, ldx, 1, m, d, nullptr, nullptr, tm);
  if (rc) return rc;
  // 1. degrees, then the core flags (one batch: the adjacency in the same launch)
  B2D_CUDA(cudaMemsetAsync(F.deg, 0, static_cast<size_t>(m + L.nb) * sizeof(unsigned), s));
  const bool one = L.nb == 1;
  for (int64_t t = 0; t < L.nb; ++t) {
    rc = db_eps(s, L, m, d, e, t, one, true);
    if (rc) return rc;
  }
  db_core_kernel<<<sl_grid(m), 256, 0, s>>>(F.deg, m, L.b, ms, F.parent, F.border, F.core);
  B2D_CUDA(cudaGetLastError());
  // 2. links between core points
  for (int64_t t = 0; t < L.nb; ++t) {
    const int64_t c0 = t * L.b, w = std::min(L.b, m - c0);
    if (!one) {
      rc = db_eps(s, L, m, d, e, t, true, false);
      if (rc) return rc;
    }
    db_link_kernel<<<db_warp_grid(m), kDbThreads, 0, s>>>(L.adj, L.ld, m, c0, w, F.core, F.parent);
    B2D_CUDA(cudaGetLastError());
  }
  db_compress_kernel<<<sl_grid(m), 256, 0, s>>>(F.parent, m, F.root);
  B2D_CUDA(cudaGetLastError());
  // 3. border points
  for (int64_t t = 0; t < L.nb; ++t) {
    const int64_t c0 = t * L.b, w = std::min(L.b, m - c0);
    if (!one) {
      rc = db_eps(s, L, m, d, e, t, true, false);
      if (rc) return rc;
    }
    db_border_kernel<<<db_warp_grid(m), kDbThreads, 0, s>>>(L.adj, L.ld, m, c0, w, F.parent, F.border);
    B2D_CUDA(cudaGetLastError());
  }
  // 4. the labels
  return db_label(s, F, m, labels, core_sample_indices, n_clusters);
}

// ------------------------------------------------------------------------------------------
// DBSCAN on the random ball cover (dbscan.cuh, db_rbc_*): the index of x, then the degree, link and border walks over it.
// Only enqueues work.
namespace {

// The index, then the build's scratch, which is dead once the index is built: the fit's arrays overlap it.
struct DbRbcLayout {
  BcIndex ix;
  BcBuildLayout build;
  DbForest f;        // deg [m]: hits per row, up to min_samples
  size_t bytes;
};

static DbRbcLayout db_rbc_layout(void* base, int64_t m, int64_t d, int64_t nl)
{
  BcOverlay o(base, m, d, nl);
  DbRbcLayout L{};
  L.ix    = o.ix;
  L.build = o.build;
  L.f     = db_forest(o.rest, m, m);
  L.bytes = o.bytes();
  return L;
}

template <int D>
static int db_rbc_fit(cudaStream_t s, const DbRbcLayout& L, int root, const float* x, int64_t ldx, int n, int nl, float e,
                      unsigned ms, uint64_t seed)
{
  const DbForest& F = L.f;
  // 0. the index of x
  int rc = bc_build<D>(s, L.ix, L.build, x, ldx, n, nl, seed);
  if (rc) return rc;
  // 1. degrees, then the core flags; a NaN or negative eps matches nothing
  if (e >= 0.f) {
    rc = bc_walk_launch(s, db_rbc_degree_kernel<D>, n, nl, D, L.ix, n, nl, root, e, ms, F.deg);
    if (rc) return rc;
  } else {
    B2D_CUDA(cudaMemsetAsync(F.deg, 0, static_cast<size_t>(n) * sizeof(unsigned), s));
  }
  db_core_kernel<<<sl_grid(n), 256, 0, s>>>(F.deg, n, n, ms, F.parent, F.border, F.core);
  B2D_CUDA(cudaGetLastError());
  // 2. links between core points; 3. border points (no core point without a hit)
  if (e >= 0.f) {
    rc = bc_walk_launch(s, db_rbc_link_kernel<D>, n, nl, D, L.ix, n, nl, root, e, static_cast<const unsigned*>(F.core),
                        F.parent);
    if (rc) return rc;
  }
  db_compress_kernel<<<sl_grid(n), 256, 0, s>>>(F.parent, n, F.root);
  B2D_CUDA(cudaGetLastError());
  if (e >= 0.f) {
    rc = bc_walk_launch(s, db_rbc_border_kernel<D>, n, nl, D, L.ix, n, nl, root, e, static_cast<const int*>(F.parent),
                        F.border);
    if (rc) return rc;
  }
  return B2D_OK;
}
}  // namespace

size_t b2d_dbscan_rbc_workspace_bytes(int64_t m, int64_t d, int64_t n_landmarks)
{
  if (m < 0 || m > 0x7fffffffll || (d != 2 && d != 3) || n_landmarks < 0 || n_landmarks > m) return static_cast<size_t>(-1);
  return db_rbc_layout(nullptr, m, d, bc_landmarks(m, n_landmarks)).bytes;
}

int b2d_dbscan_rbc_fit(void* stream, int metric, const float* x, int64_t ldx, int64_t m, int64_t d, double eps,
                       int64_t min_samples, int64_t n_landmarks, uint64_t seed, int32_t* labels,
                       int32_t* core_sample_indices, int32_t* n_clusters, void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (metric != B2D_L2Unexpanded && metric != B2D_L2SqrtUnexpanded)
    return fail(B2D_ERR_UNSUPPORTED, "dbscan rbc supports the L2Unexpanded and L2SqrtUnexpanded metrics, got metric " +
                                         std::to_string(metric));
  if (m < 0 || n_landmarks < 0) return fail(B2D_ERR_INVALID_ARG, "negative extent or n_landmarks");
  if (m == 0) return B2D_OK;
  if (m > 0x7fffffffll) return fail(B2D_ERR_INVALID_ARG, "dbscan: m must be below 2^31");
  if (d != 2 && d != 3) return fail(B2D_ERR_UNSUPPORTED, "dbscan rbc supports d = 2 and d = 3, got d = " + std::to_string(d));
  if (n_landmarks > m) return fail(B2D_ERR_INVALID_ARG, "n_landmarks must be in [0, m] (0: ceil(sqrt(m)))");
  if (min_samples < 1) return fail(B2D_ERR_INVALID_ARG, "min_samples must be >= 1");
  if (!x || !labels) return fail(B2D_ERR_INVALID_ARG, "null x / labels");
  if (ldx < d) return fail(B2D_ERR_INVALID_ARG, "leading dimension smaller than d");
  const int64_t nl = bc_landmarks(m, n_landmarks);
  int rc           = check_workspace(workspace, workspace_bytes, db_rbc_layout(nullptr, m, d, nl).bytes);
  if (rc) return rc;
  const DbRbcLayout L = db_rbc_layout(workspace, m, d, nl);
  // the ball cover's comparison: f <= fp32(eps) with f = s or sqrt(s) (a NaN or negative eps matches nothing)
  const float e     = static_cast<float>(eps);
  const unsigned ms = static_cast<unsigned>(std::min<int64_t>(min_samples, m + 1));
  const int root    = metric == B2D_L2SqrtUnexpanded;
  rc = d == 2 ? db_rbc_fit<2>(s, L, root, x, ldx, static_cast<int>(m), static_cast<int>(nl), e, ms, seed)
              : db_rbc_fit<3>(s, L, root, x, ldx, static_cast<int>(m), static_cast<int>(nl), e, ms, seed);
  if (rc) return rc;
  // 4. the labels
  return db_label(s, L.f, m, labels, core_sample_indices, n_clusters);
}
