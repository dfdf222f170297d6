// Dense pairwise distances and Gram matrices: the tensor path (expanded metrics, fp32 / fp16), the SIMT kernels of the
// unexpanded metrics (unexpanded_simt.cuh) and the fp64 SIMT path (fp64_simt.cuh).
#include <cuda.h>
#include <cuda_runtime.h>
#include <cmath>
#include <cstring>
#include <string>

#include "host.cuh"
#include "dispatch_plan.cuh"
#include "fp64_simt.cuh"
#include "unexpanded_simt.cuh"

namespace b2d {

static bool is_unexpanded(int metric)
{
  return metric == B2D_L1 || metric == B2D_L2Unexpanded || metric == B2D_L2SqrtUnexpanded ||
         metric == B2D_Linf || metric == B2D_Canberra || metric == B2D_LpUnexpanded ||
         metric == B2D_HammingUnexpanded || metric == B2D_KLDivergence || metric == B2D_JensenShannon ||
         metric == B2D_BrayCurtis;
}

template <int kMetric>
static int launch_ux_inst(cudaStream_t s, const UxParams& p, int64_t tiles, bool tma)
{
  if (tma) {  // TMA-legal operands: hardware-staged tiles of 32 floats x 128 rows, SWIZZLE_128B
    CUtensorMap mx, my;
    int rc = encode_2d(&mx, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, p.x, p.k, p.m, p.xrs * 4, UX_KB, UX_BM,
                       CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "(f32 operand)");
    if (rc) return rc;
    rc = encode_2d(&my, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, p.y, p.k, p.n, p.yrs * 4, UX_KB, UX_BM,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "(f32 operand)");
    if (rc) return rc;
    B2D_CUDA(cudaFuncSetAttribute(unexpanded_tma_kernel<kMetric>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  UX_TMA_SMEM_BYTES));
    unexpanded_tma_kernel<kMetric><<<static_cast<unsigned>(tiles), UX_THREADS, UX_TMA_SMEM_BYTES, s>>>(mx, my, p);
    B2D_CUDA(cudaGetLastError());
    return B2D_OK;
  }
  cudaError_t e = cudaFuncSetAttribute(unexpanded_simt_kernel<kMetric>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       UX_SMEM_BYTES);
  B2D_CUDA(e);
  unexpanded_simt_kernel<kMetric><<<static_cast<unsigned>(tiles), UX_THREADS, UX_SMEM_BYTES, s>>>(p);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

}  // namespace b2d

using namespace b2d;

// fp64 path: one SIMT kernel per metric (fp64_simt.cuh)
template <int kMetric>
static int launch_f64_inst(cudaStream_t s, const F64Params& p, int64_t tiles)
{
  f64_pairwise_kernel<kMetric><<<static_cast<unsigned>(tiles), 256, 0, s>>>(p);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

static int pairwise_f64(cudaStream_t s, int metric, const double* x, int64_t xrs, int64_t xcs, const double* y, int64_t yrs,
                        int64_t ycs, double* dist, int64_t ldd, int64_t m, int64_t n, int64_t k, int swapped, double metric_arg,
                        void* workspace, size_t workspace_bytes, double gamma = 0.0, double coef0 = 0.0, int degree = 0)
{
  const int rc = check_workspace(workspace, workspace_bytes, align_up(static_cast<size_t>(m + n) * 16, 1024), 1);
  if (rc) return rc;
  double* xs = static_cast<double*>(workspace);
  double* ys = xs + 2 * m;
  f64_row_stats_kernel<<<static_cast<unsigned>((m + 7) / 8), 256, 0, s>>>(xs, x, xrs, xcs, m, static_cast<int>(k));
  f64_row_stats_kernel<<<static_cast<unsigned>((n + 7) / 8), 256, 0, s>>>(ys, y, yrs, ycs, n, static_cast<int>(k));
  B2D_CUDA(cudaGetLastError());
  F64Params p;
  p.x = x; p.y = y; p.dist = dist; p.xrs = xrs; p.xcs = xcs; p.yrs = yrs; p.ycs = ycs; p.ldd = ldd; p.m = m; p.n = n;
  p.k = static_cast<int>(k); p.metric = metric; p.swapped = swapped; p.p = metric_arg; p.inv_p = 1.0 / metric_arg;
  p.xs = xs; p.ys = ys;
  p.gamma = gamma; p.coef0 = coef0; p.degree = degree;
  p.tiles_n = static_cast<int>((n + F64_T - 1) / F64_T);
  const int64_t tiles = ((m + F64_T - 1) / F64_T) * p.tiles_n;
  switch (metric) {
#define B2D_F64_CASE(M) case M: return launch_f64_inst<M>(s, p, tiles);
    B2D_F64_CASE(B2D_L2Expanded) B2D_F64_CASE(B2D_L2SqrtExpanded) B2D_F64_CASE(B2D_CosineExpanded) B2D_F64_CASE(B2D_L1)
    B2D_F64_CASE(B2D_L2Unexpanded) B2D_F64_CASE(B2D_L2SqrtUnexpanded) B2D_F64_CASE(B2D_InnerProduct) B2D_F64_CASE(B2D_Linf)
    B2D_F64_CASE(B2D_Canberra) B2D_F64_CASE(B2D_LpUnexpanded) B2D_F64_CASE(B2D_CorrelationExpanded)
    B2D_F64_CASE(B2D_JaccardExpanded) B2D_F64_CASE(B2D_HellingerExpanded) B2D_F64_CASE(B2D_BrayCurtis)
    B2D_F64_CASE(B2D_JensenShannon) B2D_F64_CASE(B2D_HammingUnexpanded) B2D_F64_CASE(B2D_KLDivergence)
    B2D_F64_CASE(B2D_RusselRaoExpanded) B2D_F64_CASE(B2D_DiceExpanded)
    B2D_F64_CASE(F64_GRAM_POLY) B2D_F64_CASE(F64_GRAM_RBF) B2D_F64_CASE(F64_GRAM_TANH)
#undef B2D_F64_CASE
    default: return fail(B2D_ERR_UNSUPPORTED, "metric");
  }
}

// The tensor path of b2d_pairwise_distance and b2d_gram_matrix: x [ma, k] and y [na, k] with element strides (xrs, xcs) and
// (yrs, ycs) (a column-major call arrives with the operands exchanged), dist [ma][ldd]; gamma, coef0 and degree are the
// kernel parameters of the Gram matrices (gram_post).
static int tc_store(cudaStream_t s, const TcMetric& tm, float gamma, float coef0, int degree, int dtype, const void* xa,
                    int64_t xrs, int64_t xcs, int64_t ma, const void* ya, int64_t yrs, int64_t ycs, int64_t na, int64_t k,
                    float* dist, int64_t ldd, void* workspace, size_t workspace_bytes)
{
  int rc = check_workspace(workspace, workspace_bytes, tc_layout(nullptr, ma, na, k, false).bytes);
  if (rc) return rc;
  TcWorkspace w = tc_layout(workspace, ma, na, k, false);
  rc = dtype == B2D_F32 ? launch_prep<float>(s, w, xa, xrs, xcs, ma, ya, yrs, ycs, na, k, nullptr, nullptr, tm)
                        : launch_prep<__half>(s, w, xa, xrs, xcs, ma, ya, yrs, ycs, na, k, nullptr, nullptr, tm);
  if (rc) return rc;
  TcParams p{};
  p.m = ma; p.n = na; p.dist = dist; p.ldd = ldd;
  p.diag_off = tc_self_diag(tm, xa, xrs, xcs, ma, ya, yrs, ycs, na);
  p.gamma = gamma; p.coef0 = coef0; p.degree = degree;
  // (dispatch_plan.cuh: TMA or register stores; k > 320: K chunks accumulated in dist, post-processed on the last)
  const TcStorePlan pl = tc_store_plan(tm.post, ma, na, k, reinterpret_cast<uintptr_t>(dist), ldd);
  p.tma_store = pl.tma_store;
  ProfileScope prof(s);  // the main kernel(s) only: the operand preparation above is outside
  for (int i = 0; i < pl.launches; ++i) {
    const TcStoreLaunch l = tc_store_launch(pl, i);
    p.acc_mode = l.acc_mode;
    rc = launch_tc(s, w, p, k, EPI_STORE, tm.post, l.kb0, l.nkb);
    if (rc) return rc;
  }
  return B2D_OK;
}

size_t b2d_pairwise_workspace_bytes(int metric, int dtype, int64_t m, int64_t n, int64_t k)
{
  if (dtype != B2D_F32 && dtype != B2D_F16 && dtype != B2D_F64) return static_cast<size_t>(-1);
  if (m < 0 || n < 0 || k < 0) return static_cast<size_t>(-1);
  TcMetric tm;
  const bool expanded = tc_metric(metric, k, &tm);
  if (dtype == B2D_F64)   // per-row (sum, sum of squares) of x and y
    return (expanded || is_unexpanded(metric)) ? align_up(static_cast<size_t>(m + n) * 16, 1024) : static_cast<size_t>(-1);
  if (is_unexpanded(metric)) return dtype == B2D_F32 ? 0 : static_cast<size_t>(-1);
  if (!expanded) return static_cast<size_t>(-1);
  return tc_layout(nullptr, m, n, k, false).bytes;
}

// The argument checks of b2d_pairwise_distance.  *empty: nothing to compute (m or n is 0).
static int pairwise_check(int metric, int dtype, const void* x, int64_t ldx, const void* y, int64_t ldy, const void* dist,
                          int64_t ldd, int64_t m, int64_t n, int64_t k, int row_major, float metric_arg, bool* empty)
{
  *empty = false;
  if (m < 0 || n < 0 || k < 0) return fail(B2D_ERR_INVALID_ARG, "negative extent");
  if (m == 0 || n == 0) { *empty = true; return B2D_OK; }
  if (k == 0) return fail(B2D_ERR_INVALID_ARG, "k must be positive");
  if (!x || !y || !dist) return fail(B2D_ERR_INVALID_ARG, "null x / y / dist");
  if (m > 0x7fffffffll * 128 || n > 0x7fffffffll || k > (1 << 24)) return fail(B2D_ERR_INVALID_ARG, "extent too large");
  if (row_major) {
    if (ldx < k || ldy < k || ldd < n) return fail(B2D_ERR_INVALID_ARG, "leading dimension smaller than the row length");
  } else {
    if (ldx < m || ldy < n || ldd < m) return fail(B2D_ERR_INVALID_ARG, "leading dimension smaller than the column length");
  }
  TcMetric tm;
  const bool expanded = tc_metric(metric, k, &tm);
  if (!expanded && !is_unexpanded(metric))
    return fail(B2D_ERR_UNSUPPORTED, "metric " + std::to_string(metric) + " is not on the tensor-core / SIMT distance path");
  if (dtype != B2D_F32 && dtype != B2D_F16 && dtype != B2D_F64) return fail(B2D_ERR_UNSUPPORTED, "dtype");
  if (metric == B2D_LpUnexpanded && !(metric_arg > 0.f)) return fail(B2D_ERR_INVALID_ARG, "LpUnexpanded needs p > 0");
  if (dtype == B2D_F16 && !expanded) return fail(B2D_ERR_UNSUPPORTED, "unexpanded metrics take fp32 inputs");
  return B2D_OK;
}

// The operands as the fp32 / fp16 kernels take them: dist is always written as a row-major [ma][ldd] matrix.
// Fortran order: D^T (row-major [n,m]) = metric(y_j, x_i).  Every metric here is symmetric except
// KLDivergence, which switches to the kernel with the operand roles exchanged (UX_KL_REV).
struct PairwiseOperands {
  const void *xa, *ya;
  int64_t ma, na, xrs, xcs, yrs, ycs;
};
static PairwiseOperands pairwise_operands(const void* x, int64_t ldx, const void* y, int64_t ldy, int64_t m, int64_t n,
                                          int row_major)
{
  if (row_major) return PairwiseOperands{x, y, m, n, ldx, 1, ldy, 1};
  return PairwiseOperands{y, x, n, m, 1, ldy, 1, ldx};
}

int b2d_debug_pairwise_plan(int metric, int dtype, const void* x, int64_t ldx, const void* y, int64_t ldy, const void* dist,
                            int64_t ldd, int64_t m, int64_t n, int64_t k, int row_major, int* out, int out_len)
{
  if (!out || out_len < 6) return fail(B2D_ERR_INVALID_ARG, "out must hold at least 6 words");
  bool empty = false;
  const int rc = pairwise_check(metric, dtype, x, ldx, y, ldy, dist, ldd, m, n, k, row_major, 2.0f, &empty);
  if (rc) return rc;
  for (int i = 0; i < out_len; ++i) out[i] = 0;
  if (empty) { out[0] = B2D_PLAN_NONE; return B2D_OK; }
  if (dtype == B2D_F64) { out[0] = B2D_PLAN_F64_SIMT; return B2D_OK; }
  const PairwiseOperands o = pairwise_operands(x, ldx, y, ldy, m, n, row_major);
  TcMetric tm;
  if (tc_metric(metric, k, &tm)) {
    const TcStorePlan pl = tc_store_plan(tm.post, o.ma, o.na, k, reinterpret_cast<uintptr_t>(dist), ldd);
    out[0] = B2D_PLAN_TENSOR; out[1] = pl.tma_store; out[2] = pl.vec2; out[5] = pl.launches;
    for (int i = 0; i < pl.launches && 6 + 4 * i + 3 < out_len; ++i) {
      const TcStoreLaunch l = tc_store_launch(pl, i);
      out[6 + 4 * i] = l.kb0; out[7 + 4 * i] = l.nkb; out[8 + 4 * i] = l.acc_mode; out[9 + 4 * i] = l.resident;
    }
    return B2D_OK;
  }
  const UxPlan ux = ux_plan(o.xrs, o.xcs, reinterpret_cast<uintptr_t>(o.xa), o.yrs, o.ycs, reinterpret_cast<uintptr_t>(o.ya), k);
  out[0] = ux.tma ? B2D_PLAN_F32_TMA : B2D_PLAN_F32_SIMT; out[3] = ux.vec_x; out[4] = ux.vec_y;
  out[5] = 1;
  return B2D_OK;
}

int b2d_pairwise_distance(void* stream, int metric, int dtype, const void* x, int64_t ldx, const void* y,
                          int64_t ldy, void* dist_v, int64_t ldd, int64_t m, int64_t n, int64_t k,
                          int row_major, float metric_arg, void* workspace, size_t workspace_bytes)
{
  float* dist = static_cast<float*>(dist_v);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  bool empty = false;
  int rc = pairwise_check(metric, dtype, x, ldx, y, ldy, dist_v, ldd, m, n, k, row_major, metric_arg, &empty);
  if (rc || empty) return rc;
  if (dtype == B2D_F64) {   // double in / double out: the SIMT fp64 path, every metric
    if (row_major)
      return pairwise_f64(s, metric, static_cast<const double*>(x), ldx, 1, static_cast<const double*>(y), ldy, 1,
                          static_cast<double*>(dist_v), ldd, m, n, k, 0, metric_arg, workspace, workspace_bytes);
    return pairwise_f64(s, metric, static_cast<const double*>(y), 1, ldy, static_cast<const double*>(x), 1, ldx,
                        static_cast<double*>(dist_v), ldd, n, m, k, 1, metric_arg, workspace, workspace_bytes);
  }
  const PairwiseOperands o = pairwise_operands(x, ldx, y, ldy, m, n, row_major);
  TcMetric tm;
  if (tc_metric(metric, k, &tm))
    return tc_store(s, tm, 0.f, 0.f, 0, dtype, o.xa, o.xrs, o.xcs, o.ma, o.ya, o.yrs, o.ycs, o.na, k, dist, ldd, workspace,
                    workspace_bytes);

  UxParams p;
  memset(&p, 0, sizeof(p));
  p.x = static_cast<const float*>(o.xa); p.y = static_cast<const float*>(o.ya); p.dist = dist;
  p.xrs = o.xrs; p.xcs = o.xcs; p.yrs = o.yrs; p.ycs = o.ycs; p.ldd = ldd; p.m = o.ma; p.n = o.na; p.k = static_cast<int>(k);
  const UxPlan ux = ux_plan(o.xrs, o.xcs, reinterpret_cast<uintptr_t>(o.xa), o.yrs, o.ycs, reinterpret_cast<uintptr_t>(o.ya), k);
  p.vec_x = ux.vec_x; p.vec_y = ux.vec_y;
  p.p = metric_arg; p.inv_p = metric == B2D_HammingUnexpanded ? 1.f / static_cast<float>(k) : 1.f / metric_arg;
  p.tiles_n = static_cast<int>((o.na + UX_BN - 1) / UX_BN);
  const int64_t tiles = ((o.ma + UX_BM - 1) / UX_BM) * p.tiles_n;
  int sms = 0;
  rc      = device_sms(&sms);
  if (rc) return rc;
  switch (metric) {
    case B2D_L1: return launch_ux_inst<UX_L1>(s, p, tiles, ux.tma);
    case B2D_L2Unexpanded: return launch_ux_inst<UX_L2>(s, p, tiles, ux.tma);
    case B2D_L2SqrtUnexpanded: return launch_ux_inst<UX_L2SQRT>(s, p, tiles, ux.tma);
    case B2D_Linf: return launch_ux_inst<UX_LINF>(s, p, tiles, ux.tma);
    case B2D_Canberra: return launch_ux_inst<UX_CANBERRA>(s, p, tiles, ux.tma);
    case B2D_HammingUnexpanded: return launch_ux_inst<UX_HAMMING>(s, p, tiles, ux.tma);
    case B2D_KLDivergence:
      return row_major ? launch_ux_inst<UX_KL>(s, p, tiles, ux.tma) : launch_ux_inst<UX_KL_REV>(s, p, tiles, ux.tma);
    case B2D_JensenShannon: return launch_ux_inst<UX_JS>(s, p, tiles, ux.tma);
    case B2D_BrayCurtis: return launch_ux_inst<UX_BRAYCURTIS>(s, p, tiles, ux.tma);
    default: return launch_ux_inst<UX_LP>(s, p, tiles, ux.tma);
  }
}

// ------------------------------------------------------------------------------------------
// Kernel Gram matrices (raft::distance::kernels): pairwise_distance's InnerProduct (LINEAR, POLYNOMIAL, TANH) or
// L2Expanded (RBF) value, transformed in the epilogue of the same kernel (expanded_tc.cuh gram_post; fp64: f64_gram).

// the pairwise metric whose value a kernel transforms
static int gram_base_metric(int kernel) { return kernel == B2D_KERNEL_RBF ? B2D_L2Expanded : B2D_InnerProduct; }
static bool gram_kernel_known(int kernel) { return kernel >= B2D_KERNEL_LINEAR && kernel <= B2D_KERNEL_TANH; }

size_t b2d_gram_matrix_workspace_bytes(int kernel, int dtype, int64_t m, int64_t n, int64_t k)
{
  if (!gram_kernel_known(kernel)) return static_cast<size_t>(-1);
  return b2d_pairwise_workspace_bytes(gram_base_metric(kernel), dtype, m, n, k);
}

int b2d_gram_matrix(void* stream, int kernel, int degree, double gamma, double coef0, int dtype, const void* x, int64_t ldx,
                    const void* y, int64_t ldy, void* out, int64_t ldo, int64_t m, int64_t n, int64_t k, int row_major,
                    void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (!gram_kernel_known(kernel)) return fail(B2D_ERR_INVALID_ARG, "unknown kernel " + std::to_string(kernel));
  if (dtype != B2D_F32 && dtype != B2D_F16 && dtype != B2D_F64) return fail(B2D_ERR_UNSUPPORTED, "dtype");
  // gamma and coef0 in the precision they are used in: double for fp64 inputs, float otherwise
  const bool finite = dtype == B2D_F64 ? std::isfinite(gamma) && std::isfinite(coef0)
                                       : std::isfinite(static_cast<float>(gamma)) && std::isfinite(static_cast<float>(coef0));
  if (!finite) return fail(B2D_ERR_INVALID_ARG, "gamma and coef0 must be finite");
  if (kernel == B2D_KERNEL_POLYNOMIAL && degree < 0) return fail(B2D_ERR_INVALID_ARG, "degree must be >= 0");
  if (m < 0 || n < 0 || k < 0) return fail(B2D_ERR_INVALID_ARG, "negative extent");
  if (m == 0 || n == 0) return B2D_OK;
  if (k == 0) return fail(B2D_ERR_INVALID_ARG, "k must be positive");
  if (!x || !y || !out) return fail(B2D_ERR_INVALID_ARG, "null x / y / out");
  if (m > 0x7fffffffll * 128 || n > 0x7fffffffll || k > (1 << 24)) return fail(B2D_ERR_INVALID_ARG, "extent too large");
  if (row_major) {
    if (ldx < k || ldy < k || ldo < n) return fail(B2D_ERR_INVALID_ARG, "leading dimension smaller than the row length");
  } else {
    if (ldx < m || ldy < n || ldo < m) return fail(B2D_ERR_INVALID_ARG, "leading dimension smaller than the column length");
  }
  if (kernel != B2D_KERNEL_POLYNOMIAL) degree = 0;
  if (dtype == B2D_F64) {
    const int metric = kernel == B2D_KERNEL_LINEAR ? B2D_InnerProduct
                     : kernel == B2D_KERNEL_POLYNOMIAL ? F64_GRAM_POLY
                     : kernel == B2D_KERNEL_RBF ? F64_GRAM_RBF : F64_GRAM_TANH;
    if (row_major)
      return pairwise_f64(s, metric, static_cast<const double*>(x), ldx, 1, static_cast<const double*>(y), ldy, 1,
                          static_cast<double*>(out), ldo, m, n, k, 0, 2.0, workspace, workspace_bytes, gamma, coef0, degree);
    return pairwise_f64(s, metric, static_cast<const double*>(y), 1, ldy, static_cast<const double*>(x), 1, ldx,
                        static_cast<double*>(out), ldo, n, m, k, 1, 2.0, workspace, workspace_bytes, gamma, coef0, degree);
  }
  // the base metric's preparation, its value transformed by the kernel's post.  Fortran order: the row-major [n, m] matrix
  // of K(y_j, x_i), the same values (every kernel is symmetric)
  TcMetric tm;
  tc_metric(gram_base_metric(kernel), k, &tm);
  tm.post = kernel == B2D_KERNEL_LINEAR ? POST_NONE
          : kernel == B2D_KERNEL_POLYNOMIAL ? POST_POLY
          : kernel == B2D_KERNEL_RBF ? POST_RBF : POST_TANH;
  const float g = static_cast<float>(gamma), c0 = static_cast<float>(coef0);
  if (row_major)
    return tc_store(s, tm, g, c0, degree, dtype, x, ldx, 1, m, y, ldy, 1, n, k, static_cast<float*>(out), ldo, workspace,
                    workspace_bytes);
  return tc_store(s, tm, g, c0, degree, dtype, y, 1, ldy, n, x, 1, ldx, m, k, static_cast<float*>(out), ldo, workspace,
                  workspace_bytes);
}
