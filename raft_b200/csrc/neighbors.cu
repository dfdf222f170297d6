// Fused brute-force kNN (knn.cuh) and the epsilon neighbourhood, both on the tensor path without the m x n matrix.
#include <cuda_runtime.h>
#include <algorithm>

#include "host.cuh"
#include "knn.cuh"

using namespace b2d;

// ------------------------------------------------------------------------------------------
// Fused brute-force kNN (SURVEY.md 8(f2)): raft::neighbors::brute_force::knn / fused_l2_knn for the
// L2 metrics without ever writing the m x n matrix (expanded_tc.cuh, EPI_TOPK).

namespace b2d {
KnnLayout knn_layout(void* base, int64_t m, int64_t n, int64_t k, int64_t n_neighbors)
{
  Carve c(base, 1024);
  KnnLayout L;
  L.w         = tc_layout(c, m, n, k, true);
  L.thr       = reinterpret_cast<float*>(L.w.aux);
  L.cnt       = L.w.aux ? reinterpret_cast<unsigned*>(L.w.aux) + m : nullptr;
  L.topk      = c.take<long long>(static_cast<size_t>(m) * n_neighbors);
  L.dropmin   = c.take<long long>(m);
  L.dirty     = c.take<int>(m);
  L.repaired  = c.take<unsigned>(m);
  L.rep_list  = c.take<int>(m);
  L.dirty_cnt = c.take<unsigned>(65);
  L.rep_cnt   = L.dirty_cnt ? L.dirty_cnt + 64 : nullptr;
  L.bytes     = c.bytes;
  return L;
}
}  // namespace b2d

size_t b2d_knn_l2_workspace_bytes(int64_t m, int64_t n, int64_t k, int64_t n_neighbors)
{
  if (m < 0 || n < 0 || k < 0 || n_neighbors < 1 || n_neighbors > KNN_MAX_K) return static_cast<size_t>(-1);
  return knn_layout(nullptr, m, n, k, n_neighbors).bytes;
}

namespace {
struct KnnCtx {
  cudaStream_t s;
  KnnLayout L;
  TcParams p;       // m, knn_* set; n / idx_offset per pass
  int64_t k;
  bool any_fix;         // a knn_fix_kernel was launched
  int pass;
  const float* x; int64_t ldx;
  const float* y; int64_t ldy;
  int family, center;
  int kk;
};
}  // namespace

// one pass over y rows [off, off + width): append, fold into the top-k, redo the rows whose lists overflowed in a way
// that matters (knn_merge_kernel / knn_fix_kernel) -- all on the device: the call only enqueues work
static int knn_pass(KnnCtx& c, int64_t off, int64_t width)
{
  const KnnLayout& L = c.L;
  TcWorkspace w2 = tc_rows(L.w, 1, off, c.k);
  TcParams p     = c.p;
  p.n            = width;
  p.idx_offset   = off;
  int rc         = launch_tc(c.s, w2, p, c.k, EPI_TOPK, POST_NONE);
  if (rc) return rc;
  unsigned* dc = L.dirty_cnt + (c.pass & 63);
  knn_merge_kernel<<<static_cast<unsigned>((c.p.m + 7) / 8), 256, 0, c.s>>>(L.topk, c.p.knn_cand, L.cnt, L.thr, L.dropmin, L.dirty,
                                                                            dc, L.repaired, L.rep_list, L.rep_cnt, c.p.m, c.kk);
  B2D_CUDA(cudaGetLastError());
  if (width > KNN_CAP) {  // (a pass of at most KNN_CAP columns cannot overflow)
    int sms = 0;
    rc = device_sms(&sms);
    if (rc) return rc;
    knn_fix_kernel<<<sms * 2, 256, 0, c.s>>>(L.topk, L.thr, L.dirty, dc, c.x, c.ldx, c.y, c.ldy, static_cast<int>(c.k), c.kk, off,
                                             width, c.family, c.center);
    B2D_CUDA(cudaGetLastError());
    c.any_fix = true;
  }
  ++c.pass;
  return B2D_OK;
}

int b2d_knn_l2(void* stream, int64_t* out_idx, float* out_dist, const float* x, int64_t ldx, const float* y,
               int64_t ldy, int64_t m, int64_t n, int64_t k, int64_t n_neighbors, int do_sqrt, void* workspace,
               size_t workspace_bytes)
{
  return b2d_knn(stream, out_idx, out_dist, do_sqrt ? B2D_L2SqrtExpanded : B2D_L2Expanded, x, ldx, y, ldy, m, n, k,
                 n_neighbors, workspace, workspace_bytes);
}

int b2d_knn(void* stream, int64_t* out_idx, float* out_dist, int metric, const float* x, int64_t ldx, const float* y,
            int64_t ldy, int64_t m, int64_t n, int64_t k, int64_t n_neighbors, void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (metric == B2D_L2Unexpanded) metric = B2D_L2Expanded;   // (the same distance)
  if (metric == B2D_L2SqrtUnexpanded) metric = B2D_L2SqrtExpanded;
  TcMetric tm;
  if ((metric != B2D_L2Expanded && metric != B2D_L2SqrtExpanded && metric != B2D_CosineExpanded &&
       metric != B2D_CorrelationExpanded) || !tc_metric(metric, k, &tm))
    return fail(B2D_ERR_UNSUPPORTED, "kNN supports the L2 metrics, CosineExpanded and CorrelationExpanded");
  if (m < 0 || n < 0 || k < 0) return fail(B2D_ERR_INVALID_ARG, "negative extent");
  if (n_neighbors < 1 || n_neighbors > n) return fail(B2D_ERR_INVALID_ARG, "n_neighbors must be in [1, n]");
  if (n_neighbors > KNN_MAX_K) return fail(B2D_ERR_UNSUPPORTED, "n_neighbors > 64 is not supported");
  if (m == 0) return B2D_OK;
  if (k == 0) return fail(B2D_ERR_INVALID_ARG, "k must be positive");
  if (k > 320) return fail(B2D_ERR_UNSUPPORTED, "kNN supports k <= 320 (see DESIGN.md section 3)");
  if (!out_idx || !out_dist || !x || !y) return fail(B2D_ERR_INVALID_ARG, "null out / x / y");
  if (ldx < k || ldy < k) return fail(B2D_ERR_INVALID_ARG, "leading dimension smaller than k");
  if (n > 0xFFFFFFFFll) return fail(B2D_ERR_INVALID_ARG, "index range exceeds 32 bits");
  const KnnLayout need = knn_layout(nullptr, m, n, k, n_neighbors);
  if (m * static_cast<int64_t>(KNN_CAP) > need.w.cand_cap)
    return fail(B2D_ERR_UNSUPPORTED, "kNN: too many query rows for one call (m * 128 must stay below 2^31): split the queries");
  int rc = check_workspace(workspace, workspace_bytes, need.bytes);
  if (rc) return rc;
  KnnCtx c;
  c.s   = s;
  c.L   = knn_layout(workspace, m, n, k, n_neighbors);
  c.k   = k;
  c.kk  = static_cast<int>(n_neighbors);
  c.pass = 0; c.any_fix = false; c.x = x; c.ldx = ldx; c.y = y; c.ldy = ldy;
  c.family = tm.mode == PREP_COSINE ? 1 : 0; c.center = tm.center;
  const KnnLayout& L = c.L;
  rc = launch_prep<float>(s, L.w, x, ldx, 1, m, y, ldy, 1, n, k, nullptr, nullptr, tm);
  if (rc) return rc;
  const int64_t total = m * n_neighbors;
  knn_init_kernel<<<static_cast<unsigned>((std::max<int64_t>(std::max<int64_t>(total, m), 65) + 255) / 256), 256, 0, s>>>(L.topk, L.thr, L.cnt, L.dropmin, L.dirty_cnt, L.repaired, m, c.kk);
  B2D_CUDA(cudaGetLastError());
  c.p   = TcParams{};
  c.p.m = m;
  c.p.knn_thr = L.thr; c.p.knn_cnt = L.cnt; c.p.knn_cand = reinterpret_cast<long long*>(L.w.cand);
  c.p.knn_cap = KNN_CAP; c.p.knn_dropmin = L.dropmin;
  // pass widths KNN_CAP, KNN_CAP, 2 KNN_CAP, 4 KNN_CAP, ...: with the k-th best of the s columns seen so far as
  // threshold, a pass over the next s columns appends ~n_neighbors entries per row on unordered data
  int64_t off = 0;
  while (off < n) {
    const int64_t width = std::min<int64_t>(off == 0 ? KNN_CAP : off, n - off);
    rc = knn_pass(c, off, width);
    if (rc) return rc;
    off += width;
  }
  if (c.any_fix) {  // every row repaired in some pass: measured again over all n columns, so one arithmetic ranks it
    int sms = 0;
    rc = device_sms(&sms);
    if (rc) return rc;
    knn_fix_kernel<<<sms * 2, 256, 0, s>>>(L.topk, L.thr, L.rep_list, L.rep_cnt, x, ldx, y, ldy, static_cast<int>(k), c.kk, 0, n,
                                           c.family, c.center);
    B2D_CUDA(cudaGetLastError());
  }
  knn_finalize_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, s>>>(out_idx, out_dist, L.topk, total,
                                                                                 tm.post == POST_CLAMP_SQRT ? 1 : 0);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

// ------------------------------------------------------------------------------------------
// Epsilon neighbourhood (raft::neighbors::epsilon_neighborhood): the L2Expanded distance of pairwise_distance compared with
// eps in the epilogue of the tensor kernel (expanded_tc.cuh, EPI_EPS), so the m x n matrix is never written.

size_t b2d_eps_neighbors_l2sq_workspace_bytes(int64_t m, int64_t n, int64_t k)
{
  if (m < 0 || n < 0 || k < 0) return static_cast<size_t>(-1);
  return tc_layout(nullptr, m, n, k, false).bytes;
}

int b2d_eps_neighbors_l2sq(void* stream, uint8_t* adj, int64_t ld_adj, void* vd, int vd_int64, int init_vd,
                           const float* x, int64_t ldx, const float* y, int64_t ldy, int64_t m, int64_t n, int64_t k,
                           float eps, void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (m < 0 || n < 0 || k < 0) return fail(B2D_ERR_INVALID_ARG, "negative extent");
  if (!adj && !vd) return fail(B2D_ERR_INVALID_ARG, "adj and vd are both null: nothing to compute");
  if (m > 0x7fffffffll || n > 0x7fffffffll) return fail(B2D_ERR_INVALID_ARG, "m and n must be below 2^31");
  const bool work = m > 0 && n > 0;
  if (work) {
    if (k == 0) return fail(B2D_ERR_INVALID_ARG, "k must be positive");
    if (k > 320) return fail(B2D_ERR_UNSUPPORTED, "eps_neighbors_l2sq supports k <= 320 (the whole distance at once)");
    if (!x || !y) return fail(B2D_ERR_INVALID_ARG, "null x / y");
    if (adj && ld_adj < n) return fail(B2D_ERR_INVALID_ARG, "ld_adj smaller than n");
    if (ldx < k || ldy < k) return fail(B2D_ERR_INVALID_ARG, "leading dimension smaller than k");
    const int rc = check_workspace(workspace, workspace_bytes, tc_layout(nullptr, m, n, k, false).bytes);
    if (rc) return rc;
  }
  if (vd && init_vd) B2D_CUDA(cudaMemsetAsync(vd, 0, static_cast<size_t>(n + 1) * (vd_int64 ? 8 : 4), s));
  if (!work) return B2D_OK;
  TcWorkspace w = tc_layout(workspace, m, n, k, false);
  int rc = launch_prep<float>(s, w, x, ldx, 1, m, y, ldy, 1, n, k, nullptr, nullptr, TC_L2);
  if (rc) return rc;
  TcParams p{};
  p.m = m; p.n = n;
  p.adj = adj; p.ld_adj = ld_adj; p.vd = vd; p.vd64 = vd_int64 ? 1 : 0; p.eps = eps;
  // y is a window of x's rows (same memory, same pitch): row j of y is row j + off of x
  const intptr_t dy = reinterpret_cast<intptr_t>(y) - reinterpret_cast<intptr_t>(x);
  if (ldx == ldy && dy % (ldx * static_cast<intptr_t>(sizeof(float))) == 0)
    p.diag_off = dy / (ldx * static_cast<intptr_t>(sizeof(float)));
  // adj leaves through the staging boxes where TMA can address it: 16-byte aligned base and pitch, and rows that end on a
  // 16-byte boundary (the byte analogue of pairwise_distance's n % 4 rule for fp32 above); coordinates fit int32 (m, n <
  // 2^31 above).  Otherwise the epilogue stores from registers.
  p.tma_store = (adj && reinterpret_cast<uintptr_t>(adj) % 16 == 0 && ld_adj % 16 == 0 && n % 16 == 0) ? 1 : 0;
  ProfileScope prof(s);
  return launch_tc(s, w, p, k, EPI_EPS, POST_CLAMP);
}
