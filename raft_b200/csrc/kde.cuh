// Kernels of kernel_density (kde.cu) around the tensor kernel's EPI_KDE epilogue (expanded_tc.cuh, kde_row32): the
// column weights and their total, the fold of each slab's partials into per-row fp64 accumulators, and the finish.  Every
// sum runs in a fixed order: the result does not depend on the device or on the slab width.
#pragma once
#include <cuda_runtime.h>
#include <cmath>
#include <cstdint>

namespace b2d {

constexpr int kKdeThreads   = 256;
constexpr int64_t kKdeWRows = 8192;   // weights per block of kde_weights_kernel (one fp64 partial sum each)

// fp64 sum of the block's per-thread values v, in a fixed tree order; the result on thread 0
__device__ __forceinline__ double kde_block_sum(double v, double* sh)
{
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int o = kKdeThreads / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
    __syncthreads();
  }
  return sh[0];
}

// Block b: the weights of rows [b kKdeWRows, (b + 1) kKdeWRows) (w null: all 1) into the column terms colw (log2 w for the
// log-sum-exp kernels, w for the compact ones), their fp64 sum into wpart[b], and *bad |= 1 for a negative or non-finite
// weight.
__global__ void __launch_bounds__(kKdeThreads) kde_weights_kernel(const float* w, int64_t n, int lse, float* colw,
                                                                  double* wpart, unsigned* bad)
{
  __shared__ double sh[kKdeThreads];
  const int64_t r0 = blockIdx.x * kKdeWRows, r1 = min(r0 + kKdeWRows, n);
  double acc = 0.0;
  bool b     = false;
  for (int64_t j = r0 + threadIdx.x; j < r1; j += kKdeThreads) {
    const float v = w ? w[j] : 1.f;
    b |= !(v >= 0.f) || isinf(v);
    acc += v;
    colw[j] = lse ? static_cast<float>(log2(static_cast<double>(v))) : v;
  }
  if (b) atomicOr(bad, 1u);
  const double s = kde_block_sum(acc, sh);
  if (threadIdx.x == 0) wpart[blockIdx.x] = s;
}

// *wtot = the sum of wpart[0, nb), one block
__global__ void __launch_bounds__(kKdeThreads) kde_total_kernel(const double* wpart, int64_t nb, double* wtot)
{
  __shared__ double sh[kKdeThreads];
  double acc = 0.0;
  for (int64_t b = threadIdx.x; b < nb; b += kKdeThreads) acc += wpart[b];
  const double s = kde_block_sum(acc, sh);
  if (threadIdx.x == 0) *wtot = s;
}

// One slab: row i's partials part[g * ld + i], g in [0, halves), fold into acc[i] = (M, S) (base-2 log-sum-exp: the row's
// sum is S 2^M), in ascending g; `first` starts from the empty sum (M = -inf, S = 0).  The compact kernels have M = 0 in
// every partial, so this is their plain fp64 sum (2^0 = 1).  A NaN partial makes S NaN.
__global__ void __launch_bounds__(kKdeThreads) kde_fold_kernel(const float2* part, int64_t ld, int64_t halves, int64_t m,
                                                               double2* acc, int first)
{
  const int64_t i = blockIdx.x * static_cast<int64_t>(kKdeThreads) + threadIdx.x;
  if (i >= m) return;
  double2 a = first ? make_double2(-INFINITY, 0.0) : acc[i];
  for (int64_t g = 0; g < halves; ++g) {
    const float2 q = part[g * ld + i];
    const double mh = q.x, sh = q.y;
    if (mh > a.x) {   // a larger maximum (finite: a partial's M is never +inf)
      a.y = a.y * exp2(a.x - mh) + sh;
      a.x = mh;
    } else {          // (M = -inf on both sides: the terms are 0, or NaN)
      a.y += sh * exp2(mh - (a.x == -INFINITY ? 0.0 : a.x));
    }
  }
  acc[i] = a;
}

// out[i] = M ln 2 + ln S - ln W + log_norm, or NaN for every row when *bad or W = 0
__global__ void __launch_bounds__(kKdeThreads) kde_finish_kernel(const double2* acc, int64_t m, const double* wtot,
                                                                 const unsigned* bad, double log_norm, double* out)
{
  const int64_t i = blockIdx.x * static_cast<int64_t>(kKdeThreads) + threadIdx.x;
  if (i >= m) return;
  const double W = *wtot;
  if (*bad != 0u || !(W > 0.0)) {
    out[i] = NAN;
    return;
  }
  const double2 a = acc[i];
  out[i] = (a.x * 0.69314718055994530942 + log(a.y)) - log(W) + log_norm;
}

}  // namespace b2d
