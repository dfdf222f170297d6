// fp64 pairwise distances (SURVEY.md 8(a2): "fp32 in/acc/out (also fp64 ...)", 8(f4)): one register-tiled SIMT kernel
// for every metric of the enum, in double precision end to end.  The fp64 tensor-core path (DMMA) is not worth it for
// this shape (DESIGN.md), and the reference's own fp64 instantiation was a SIMT kernel too, so this is a plain
// 64 x 64 tile, 256 threads x (4 x 4) outputs, 16-deep k-blocks through shared memory; any row / column stride,
// zero-filled tails.  Expanded metrics are evaluated from <x,y> and per-row statistics (sum, sum of squares) computed by
// f64_row_stats_kernel; the L2 family uses the difference form (no cancellation to speak of in fp64, and exact zeros on
// the diagonal).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include "../../include/raft_b200.h"

namespace b2d {

struct F64Params {
  const double* x;
  const double* y;
  double* dist;
  int64_t xrs, xcs, yrs, ycs;  // element strides
  int64_t ldd, m, n;
  int k;
  int metric;       // B2D_* metric id
  int swapped;      // column-major entry: x and y were exchanged (KLDivergence swaps the operand roles back)
  double p, inv_p;  // LpUnexpanded
  const double* xs; // [m][2] (sum, sum of squares) of the rows of x (after the sqrt transform for Hellinger)
  const double* ys; // [n][2]
  int tiles_n;
  double gamma, coef0;  // kernel Gram matrices (F64_GRAM_*)
  int degree;
};

// Internal metric ids of the kernel Gram matrices (b2d_gram_matrix; no public DistanceType): the value of f64_acc /
// f64_fin for the base metric, then f64_gram.  The linear kernel is B2D_InnerProduct itself.
enum { F64_GRAM_POLY = 1001, F64_GRAM_RBF = 1002, F64_GRAM_TANH = 1003 };

__global__ void f64_row_stats_kernel(double* out, const double* x, int64_t rs, int64_t cs, int64_t rows, int k)
{
  const int lane  = threadIdx.x & 31;
  const int64_t r = static_cast<int64_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= rows) return;
  double s = 0.0, ss = 0.0;
  for (int t = lane; t < k; t += 32) {
    const double v = x[r * rs + t * cs];
    s += v;
    ss += v * v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    ss += __shfl_xor_sync(0xffffffffu, ss, o);
  }
  if (lane == 0) { out[2 * r] = s; out[2 * r + 1] = ss; }
}

// metric classes: what one (x_t, y_t) pair adds to the running value(s)
__device__ __forceinline__ void f64_acc(int metric, int swapped, double p, double a, double b, double& acc, double& aux)
{
  switch (metric) {
    case B2D_L2Expanded: case B2D_L2SqrtExpanded: case B2D_L2Unexpanded: case B2D_L2SqrtUnexpanded: case F64_GRAM_RBF: {
      const double d = a - b; acc = fma(d, d, acc); break; }
    case B2D_L1: acc += fabs(a - b); break;
    case B2D_Linf: acc = fmax(acc, fabs(a - b)); break;
    case B2D_Canberra: { const double s = fabs(a) + fabs(b); if (s > 0.0) acc += fabs(a - b) / s; break; }
    case B2D_LpUnexpanded: acc += pow(fabs(a - b), p); break;
    case B2D_HammingUnexpanded: acc += (a != b) ? 1.0 : 0.0; break;
    case B2D_KLDivergence: {
      const double u = swapped ? b : a, v = swapped ? a : b;  // KL(u || v) = sum u log(u / v), 0 log 0 = 0
      if (u != 0.0) acc += u * (log(u) - log(v));
      break; }
    case B2D_JensenShannon: {
      const double mm = 0.5 * (a + b);
      if (a != 0.0) acc += a * (log(a) - log(mm));
      if (b != 0.0) acc += b * (log(b) - log(mm));
      break; }
    case B2D_BrayCurtis: acc += fabs(a - b); aux += fabs(a + b); break;
    case B2D_HellingerExpanded: acc += sqrt(a) * sqrt(b); break;
    default: acc = fma(a, b, acc); break;  // inner-product family: InnerProduct, Cosine, Correlation, RusselRao, Jaccard, Dice
  }
}

__device__ __forceinline__ double f64_fin(int metric, double acc, double aux, double inv_p, int k, double xs0, double xs1,
                                          double ys0, double ys1)
{
  switch (metric) {
    case B2D_L2SqrtExpanded: case B2D_L2SqrtUnexpanded: return sqrt(acc);
    case B2D_LpUnexpanded: return pow(acc, inv_p);
    case B2D_HammingUnexpanded: return acc / k;
    case B2D_KLDivergence: return 0.5 * acc;
    case B2D_JensenShannon: return sqrt(fmax(0.5 * acc, 0.0));
    case B2D_BrayCurtis: return acc / aux;
    case B2D_HellingerExpanded: return sqrt(fmax(1.0 - acc, 0.0));
    case B2D_RusselRaoExpanded: return (k - acc) / k;
    case B2D_CosineExpanded: return 1.0 - acc / sqrt(xs1 * ys1);
    case B2D_CorrelationExpanded: {
      const double num = k * acc - xs0 * ys0;
      const double den = sqrt((k * xs1 - xs0 * xs0) * (k * ys1 - ys0 * ys0));
      return 1.0 - num / den; }
    case B2D_JaccardExpanded: { const double den = xs1 + ys1 - acc; return den > 0.0 ? fmax(1.0 - acc / den, 0.0) : 0.0; }
    case B2D_DiceExpanded: { const double den = xs1 + ys1; return den > 0.0 ? fmax(1.0 - 2.0 * acc / den, 0.0) : 0.0; }
    default: return acc;  // L1, Linf, Canberra, L2 (squared), InnerProduct, the Gram matrices' base values
  }
}

// the kernel Gram matrices' transform of the base value u (RBF: the squared distance, difference form; POLY / TANH: the
// inner product); every other metric passes through
__device__ __forceinline__ double f64_gram(int metric, double u, const F64Params& p)
{
  switch (metric) {
    case F64_GRAM_RBF: return exp(-(p.gamma * u));
    case F64_GRAM_TANH: return tanh(fma(p.gamma, u, p.coef0));
    case F64_GRAM_POLY: {   // binary exponentiation, as on the tensor path (degree 0: 1)
      const double t = fma(p.gamma, u, p.coef0);
      double r = 1.0, b = t;
      for (unsigned e = static_cast<unsigned>(p.degree); e != 0u; e >>= 1) {
        if (e & 1u) r *= b;
        if (e > 1u) b *= b;
      }
      return r;
    }
    default: return u;
  }
}

constexpr int F64_T = 64, F64_KB = 16;

template <int kMetric>   // (a compile-time metric: the switch in f64_acc / f64_fin folds away)
__global__ void __launch_bounds__(256) f64_pairwise_kernel(const F64Params p)
{
  __shared__ double sx[F64_KB][F64_T + 1], sy[F64_KB][F64_T + 1];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int64_t m0 = (static_cast<int64_t>(blockIdx.x) / p.tiles_n) * F64_T;
  const int64_t n0 = (static_cast<int64_t>(blockIdx.x) % p.tiles_n) * F64_T;
  double acc[4][4], aux[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) { acc[i][j] = 0.0; aux[i][j] = 0.0; }
  for (int k0 = 0; k0 < p.k; k0 += F64_KB) {
    for (int e = tid; e < F64_T * F64_KB; e += 256) {
      const int r = e / F64_KB, t = e % F64_KB;
      const int64_t gi = m0 + r, gj = n0 + r;
      sx[t][r] = (gi < p.m && k0 + t < p.k) ? p.x[gi * p.xrs + static_cast<int64_t>(k0 + t) * p.xcs] : 0.0;
      sy[t][r] = (gj < p.n && k0 + t < p.k) ? p.y[gj * p.yrs + static_cast<int64_t>(k0 + t) * p.ycs] : 0.0;
    }
    __syncthreads();
    const int kend = min(F64_KB, p.k - k0);   // (tails must not enter: log / != would see the zero fill)
    for (int t = 0; t < kend; ++t) {
      double a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = sx[t][ty + 16 * i]; b[i] = sy[t][tx + 16 * i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) f64_acc(kMetric, p.swapped, p.p, a[i], b[j], acc[i][j], aux[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int64_t gi = m0 + ty + 16 * i;
    if (gi >= p.m) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int64_t gj = n0 + tx + 16 * j;
      if (gj >= p.n) continue;
      const double xs0 = p.xs ? p.xs[2 * gi] : 0.0, xs1 = p.xs ? p.xs[2 * gi + 1] : 0.0;
      const double ys0 = p.ys ? p.ys[2 * gj] : 0.0, ys1 = p.ys ? p.ys[2 * gj + 1] : 0.0;
      p.dist[gi * p.ldd + gj] = f64_gram(kMetric, f64_fin(kMetric, acc[i][j], aux[i][j], p.inv_p, p.k, xs0, xs1, ys0, ys1), p);
    }
  }
}

}  // namespace b2d
