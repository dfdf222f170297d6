// Kernel density estimation (sklearn.neighbors.KernelDensity.score_samples with atol = rtol = 0) on the tensor path: the
// distances are reduced per row in the epilogue of the tensor kernel (expanded_tc.cuh, EPI_KDE), slab by slab of dataset
// columns, and folded into per-row fp64 accumulators (kde.cuh).  The m x n matrix is never written.
#include <cuda_runtime.h>
#include <algorithm>
#include <cmath>
#include <string>

#include "host.cuh"
#include "kde.cuh"

using namespace b2d;

namespace {

constexpr int64_t kKdeDefaultPartBytes = 1ll << 30;   // the partials of one slab, batch_cols = 0

// columns per slab: batch_cols rounded up to the 256-column y block, or (0) as many as keep the partials at 8 bytes per
// row and 128-column half within about 1 GiB; at least one y block, at most n rounded up
int64_t kde_batch(int64_t m, int64_t n, int64_t batch_cols)
{
  const int64_t all = (n + TC_BN - 1) / TC_BN * TC_BN;
  int64_t cols;
  if (batch_cols > 0) cols = std::min(batch_cols, all) + TC_BN - 1;
  else cols = kKdeDefaultPartBytes / (8 * std::max<int64_t>(m, 1)) * TC_HN;
  return std::max<int64_t>(TC_BN, std::min(cols / TC_BN * TC_BN, all));
}

// The workspace: the tensor path's operands (queries on the x side, dataset on the y side), the column terms and the
// weight sums, the per-row accumulators and the partials of one slab
struct KdeLayout {
  TcWorkspace w;
  int64_t cols;      // dataset columns per slab
  int64_t wblocks;   // blocks of kde_weights_kernel
  float* colw;       // [n]
  double* wpart;     // [wblocks]
  double* wtot;      // [1]
  unsigned* bad;     // [1]
  double2* acc;      // [m]
  float2* part;      // [cols / 128][m]
  size_t bytes;
};

KdeLayout kde_layout(void* base, int64_t m, int64_t n, int64_t d, int64_t batch_cols)
{
  Carve c(base, 1024);
  KdeLayout L;
  L.w       = tc_layout(c, m, n, d, false);
  L.cols    = kde_batch(m, n, batch_cols);
  L.wblocks = (n + kKdeWRows - 1) / kKdeWRows;
  L.colw    = c.take<float>(n);
  L.wpart   = c.take<double>(L.wblocks);
  L.wtot    = c.take<double>(1);
  L.bad     = c.take<unsigned>(1);
  L.acc     = c.take<double2>(m);
  L.part    = c.take<float2>(static_cast<size_t>(L.cols / TC_HN) * m);
  L.bytes   = c.bytes;
  return L;
}

bool kde_lse(int kernel) { return kernel == B2D_KDE_GAUSSIAN || kernel == B2D_KDE_EXPONENTIAL; }

// log of V_n, the volume of the unit n-ball, as sklearn's logVn (n may be -1 there)
double log_vn(double n) { return 0.5 * n * std::log(M_PI) - std::lgamma(0.5 * n + 1.0); }

// log of the integral of t^(d-1) cos(pi t / 2) over [0, 1]: with u = 1 - t it is the sum over k of
// (-1)^k (pi/2)^(2k+1) Gamma(d) / Gamma(d + 2k + 2), an alternating series whose terms fall by at least (pi/2)^2 / 12 per
// step, so it has no cancellation (sklearn's alternating sum of the chain-rule integration has, at every even d)
double log_cos_moment(int64_t d)
{
  const double q = 0.25 * M_PI * M_PI, dd = static_cast<double>(d);
  double sum = 0.0, t = 1.0;
  for (int k = 0; k < 64 && t > 1e-18; ++k) {
    sum += (k % 2 ? -t : t);
    t *= q / ((dd + 2 * k + 2) * (dd + 2 * k + 3));
  }
  return std::log(0.5 * M_PI) - std::log(dd) - std::log(dd + 1.0) + std::log(sum);
}

// sklearn's _log_kernel_norm(h, d, kernel), with the exact normalisation of the cosine kernel
double kde_log_norm(int kernel, double h, int64_t d)
{
  const double dd = static_cast<double>(d), log_2pi = std::log(2.0 * M_PI);
  const double log_s = log_2pi + log_vn(dd - 2.0);   // S_(d-1), the surface of the unit sphere in d dimensions
  double f = 0.0;
  switch (kernel) {
    case B2D_KDE_GAUSSIAN: f = 0.5 * dd * log_2pi; break;
    case B2D_KDE_TOPHAT: f = log_vn(dd); break;
    case B2D_KDE_EPANECHNIKOV: f = log_vn(dd) + std::log(2.0 / (dd + 2.0)); break;
    case B2D_KDE_EXPONENTIAL: f = log_s + std::lgamma(dd); break;
    case B2D_KDE_LINEAR: f = log_vn(dd) - std::log(dd + 1.0); break;
    default: f = log_s + log_cos_moment(d); break;
  }
  return -f - dd * std::log(h);
}

}  // namespace

size_t b2d_kde_workspace_bytes(int64_t m, int64_t n, int64_t d, int64_t batch_cols)
{
  if (m < 0 || n < 0 || d < 0 || batch_cols < 0) return static_cast<size_t>(-1);
  return kde_layout(nullptr, m, n, d, batch_cols).bytes;
}

int b2d_kde_score_samples(void* stream, int kernel, double bandwidth, const float* dataset, int64_t ldy,
                          const float* sample_weight, const float* queries, int64_t ldx, int64_t m, int64_t n, int64_t d,
                          int64_t batch_cols, double* out, void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (kernel < B2D_KDE_GAUSSIAN || kernel > B2D_KDE_COSINE)
    return fail(B2D_ERR_INVALID_ARG, "unknown kernel " + std::to_string(kernel));
  if (m < 0 || n < 0 || d < 0) return fail(B2D_ERR_INVALID_ARG, "negative extent");
  if (batch_cols < 0) return fail(B2D_ERR_INVALID_ARG, "negative batch_cols");
  if (m > 0x7fffffffll || n > 0x7fffffffll) return fail(B2D_ERR_INVALID_ARG, "m and n must be below 2^31");
  if (n == 0 || d == 0) return fail(B2D_ERR_INVALID_ARG, "n and d must be positive");
  if (d > 320) return fail(B2D_ERR_UNSUPPORTED, "kernel_density supports d <= 320 (the whole distance at once)");
  if (!std::isfinite(bandwidth) || !(bandwidth > 0.0)) return fail(B2D_ERR_INVALID_ARG, "bandwidth must be finite and > 0");
  const float h2 = static_cast<float>(bandwidth * bandwidth);
  if (!std::isfinite(0.5f / h2)) return fail(B2D_ERR_INVALID_ARG, "0.5 / bandwidth^2 is not finite in fp32");
  if (m == 0) return B2D_OK;
  if (!dataset || !queries || !out) return fail(B2D_ERR_INVALID_ARG, "null dataset / queries / out");
  if (ldx < d || ldy < d) return fail(B2D_ERR_INVALID_ARG, "leading dimension smaller than d");
  int rc = check_workspace(workspace, workspace_bytes, kde_layout(nullptr, m, n, d, batch_cols).bytes);
  if (rc) return rc;
  const KdeLayout L = kde_layout(workspace, m, n, d, batch_cols);
  const bool lse    = kde_lse(kernel);
  const double h = bandwidth, log2e = 1.0 / std::log(2.0);
  // the factor of kde_row32: base-2 exponents for the log-sum-exp kernels
  double sc = 0.0;
  switch (kernel) {
    case B2D_KDE_GAUSSIAN: sc = 0.5 / (h * h) * log2e; break;
    case B2D_KDE_EPANECHNIKOV: sc = -1.0 / (h * h); break;
    case B2D_KDE_EXPONENTIAL: sc = log2e / h; break;
    case B2D_KDE_LINEAR: sc = -1.0 / h; break;
    case B2D_KDE_COSINE: sc = 0.5 * M_PI / h; break;
    default: break;   // tophat: K = 1
  }
  // 1. the weights: column terms, total, validity (on the device)
  B2D_CUDA(cudaMemsetAsync(L.bad, 0, sizeof(unsigned), s));
  kde_weights_kernel<<<static_cast<unsigned>(L.wblocks), kKdeThreads, 0, s>>>(sample_weight, n, lse ? 1 : 0, L.colw,
                                                                               L.wpart, L.bad);
  B2D_CUDA(cudaGetLastError());
  kde_total_kernel<<<1, kKdeThreads, 0, s>>>(L.wpart, L.wblocks, L.wtot);
  B2D_CUDA(cudaGetLastError());
  // 2. queries and dataset prepared once; every slab is a window of the dataset side
  rc = launch_prep<float>(s, L.w, queries, ldx, 1, m, dataset, ldy, 1, n, d, nullptr, nullptr, TC_L2);
  if (rc) return rc;
  const int64_t self = tc_self_diag(TC_L2, queries, ldx, 1, m, dataset, ldy, 1, n);
  const unsigned rows_grid = static_cast<unsigned>((m + kKdeThreads - 1) / kKdeThreads);
  for (int64_t c0 = 0; c0 < n; c0 += L.cols) {
    const int64_t w = std::min(L.cols, n - c0);
    TcParams p{};
    p.m = m; p.n = w;
    p.diag_off   = self == TC_NO_DIAG ? TC_NO_DIAG : c0;
    p.kde_kernel = kernel;
    p.kde_s      = static_cast<float>(sc);
    p.kde_h2     = h2;
    p.kde_pad    = lse ? -INFINITY : 0.f;
    p.kde_colw   = L.colw + c0;
    p.kde_part   = L.part;
    p.kde_ld     = m;
    {
      ProfileScope prof(s);
      rc = launch_tc(s, tc_rows(L.w, 1, c0, d), p, d, EPI_KDE, POST_CLAMP);
      if (rc) return rc;
    }
    kde_fold_kernel<<<rows_grid, kKdeThreads, 0, s>>>(L.part, m, (w + TC_HN - 1) / TC_HN, m, L.acc, c0 == 0 ? 1 : 0);
    B2D_CUDA(cudaGetLastError());
  }
  // 3. the logs, the weight total, the normalisation
  kde_finish_kernel<<<rows_grid, kKdeThreads, 0, s>>>(L.acc, m, L.wtot, L.bad, kde_log_norm(kernel, h, d), out);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}
