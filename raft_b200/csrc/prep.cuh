// Operand preparation for the tensor-core (expanded-metric) path.
//
// Two small kernels over both input matrices, O((m+n)k) work (~1% of the pair loop):
//   prep_max_kernel    per-matrix max |element| (after optional centring / row normalisation),
//                      atomicMax into a device scalar -- no host round trip
//   prep_split_kernel  per row: optionally centre (CorrelationExpanded == cosine of centred rows)
//                      and normalise to unit length (cosine family), scale by the power of two 2^e
//                      that puts the MATRIX maximum in [2^14, 2^15), split into fp16 hi + fp16 lo
//                      (x*2^e = hi + lo + O(2^-22|x*2^e|)) and write the packed layout the MMA
//                      kernel's TMA descriptor expects:
//                          row r, k-block b (32 source columns):  [ hi[0..32) | lo[0..32) ] = 128 bytes
//                      so that one 128-byte SWIZZLE_128B shared-memory row carries both halves of a
//                      k-block and hi*hi, hi*lo, lo*hi are K=16 wgmma steps over the same tile.
// One scale per matrix (not per row): fp16 keeps 11 bits at any normal magnitude, so rows up to
// 2^18 below the matrix maximum still split without loss, and a single scale makes the undo a
// single scalar -- the epilogue is d = acc * c + (t_x[i] + t_y[j]) with
//     L2       c = -2 * 2^-(ex+ey),  t = |row|^2      (fp64 accumulate, rounded once: the reference's
//                                                      row-norm prologue is a compensated fp32 sum,
//                                                      cpp/include/raft/linalg/detail/coalesced_reduction-inl.cuh:34-44)
//     cosine   c = -2^-(ex+ey),      t_x = 1, t_y = 0 (rows pre-normalised; also correlation)
//     inner    c =  2^-(ex+ey),      t = 0
// k need not be a multiple of 32 and the source may have any row/column stride (row- or
// column-major, ld != k): the packed copy is what makes the TMA legal for every input, which is
// the job the reference's tile loader did with zero-fill and Veclen fallback
// (cpp/include/raft/linalg/detail/contractions.cuh:186-193).
#pragma once
#include <cuda_fp16.h>
#include <cstdint>

namespace b2d {

enum PrepMode : int { PREP_L2 = 0, PREP_COSINE = 1, PREP_INNER = 2,
                      PREP_INNER_NORM = 3 };  // inner product with t = |row|^2 (Jaccard / Dice: ratio epilogues)

struct PrepSide {
  const void* src;  // float or half
  int64_t rs, cs;   // element strides: element (r,t) at src[r*rs + t*cs]
  int64_t rows;
  __half* op;       // [rows][nkb][64]
  float* tvec;      // [rows]
  float* svec;      // [rows] 2^(E - e_row): 1 for every row that shares the matrix exponent E (see prep_split_kernel)
  const float* ext_norm_sq;  // optional caller-provided squared norms (fusedL2NN xn/yn)
  float* lvec;               // optional [rows]: |row - hi part| in the units of the (normalised) row: what the 1-product
                             // coarse pass of the screened NN search leaves out (screen_tc.cuh)
  const int* gather;         // optional: packed row r is source row gather[r] (norm-sorted database of the screened NN search)
};

struct PrepParams {
  PrepSide side[2];  // 0 = x (output rows), 1 = y (output columns)
  int k, nkb;
  int mode;          // PrepMode
  int center;        // subtract the row mean first (correlation)
  int xform;         // 1: take sqrt of every element first (HellingerExpanded)
  float coef_mul;    // extra factor on the epilogue scalar (RusselRao: -1/k, Hellinger: -1)
  float tx_const;    // PREP_INNER: row term of x (Hellinger / RusselRao: 1 -> d = 1 - ...)
  unsigned* gmax;    // [2] float bits of the per-matrix maximum (zeroed before prep_max_kernel)
  float* coef;       // [1] the epilogue scalar c
  unsigned* has_lo;  // [1] set to 1 when any lo half is non-zero (zeroed before the kernels run)
  unsigned* nonuni;  // [2] set to 1 when some row of x / y took its own exponent (zeroed before the kernels run)
  // Re-preparing y alone (the centroids of every k-means iteration): first_side = 1 skips the rows of x, whose packed
  // rows, terms and exponent gmax[0] stay as an earlier launch left them; gmax[1] and nonuni[1] must be zeroed first.
  // coef is written by the first prepared row either way.
  int first_side;
  const unsigned* run_flag;  // non-null: the launch is a no-op unless *run_flag != 0
};

template <typename T>
__device__ __forceinline__ float ld_as_float(const T* p);
template <>
__device__ __forceinline__ float ld_as_float<float>(const float* p) { return __ldg(p); }
template <>
__device__ __forceinline__ float ld_as_float<__half>(const __half* p) { return __half2float(__ldg(p)); }
template <typename T>
__device__ __forceinline__ float ld_elem(const T* p, int xform)
{
  const float v = ld_as_float(p);
  return xform ? sqrtf(v) : v;
}

__device__ __forceinline__ int scale_exponent(float amax)
{
  int e = 0;
  if (amax > 0.f && amax < 3.0e38f) {
    int q;
    frexpf(amax, &q);  // amax = f * 2^q, f in [0.5,1)
    e = 15 - q;        // amax * 2^e in [2^14, 2^15)
    e = max(-100, min(100, e));
  }
  return e;
}

// mean (if centring) and sum of squares of a row, warp-cooperative
template <typename T>
__device__ __forceinline__ void row_stats(const T* row, int64_t cs, int k, int center, int xform, int lane,
                                          float& mean, double& ss, float& amax)
{
  mean = 0.f;
  if (center) {
    double s = 0.0;
    for (int t = lane; t < k; t += 32) s += static_cast<double>(ld_elem(row + t * cs, xform));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    mean = static_cast<float>(s / static_cast<double>(k));
  }
  amax = 0.f;
  ss   = 0.0;
  for (int t = lane; t < k; t += 32) {
    const float v = ld_elem(row + t * cs, xform) - mean;
    amax          = fmaxf(amax, fabsf(v));
    ss += static_cast<double>(v) * static_cast<double>(v);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    ss += __shfl_xor_sync(0xffffffffu, ss, o);
  }
}

template <typename T>
__global__ void __launch_bounds__(256) prep_max_kernel(PrepParams p)
{
  if (p.run_flag != nullptr && __ldg(p.run_flag) == 0u) return;
  const int lane  = threadIdx.x & 31;
  int64_t r       = static_cast<int64_t>(blockIdx.x) * 8 + (threadIdx.x >> 5) + (p.first_side ? p.side[0].rows : 0);
  const int which = r >= p.side[0].rows ? 1 : 0;
  if (which) r -= p.side[0].rows;
  const PrepSide& sd = p.side[which];
  if (r >= sd.rows) return;
  const T* row = static_cast<const T*>(sd.src) + r * sd.rs;
  float mean, amax;
  double ss;
  row_stats(row, sd.cs, p.k, p.center, p.xform, lane, mean, ss, amax);
  if (p.mode == PREP_COSINE) amax = ss > 0.0 ? static_cast<float>(static_cast<double>(amax) / sqrt(ss)) : 0.f;
  // atomics only when the value can raise the maximum (200k same-address atomics cost ~140 us;
  // with the read-first test they become O(log rows))
  if (lane == 0 && amax > 0.f && amax < 3.0e38f &&
      __float_as_uint(amax) > *reinterpret_cast<volatile unsigned*>(&p.gmax[which]))
    atomicMax(&p.gmax[which], __float_as_uint(amax));
}

template <typename T>
__global__ void __launch_bounds__(256) prep_split_kernel(PrepParams p)
{
  if (p.run_flag != nullptr && __ldg(p.run_flag) == 0u) return;
  const int lane  = threadIdx.x & 31;
  int64_t r       = static_cast<int64_t>(blockIdx.x) * 8 + (threadIdx.x >> 5) + (p.first_side ? p.side[0].rows : 0);
  const int which = r >= p.side[0].rows ? 1 : 0;
  if (which) r -= p.side[0].rows;
  const PrepSide& sd = p.side[which];
  if (r >= sd.rows) return;
  const int64_t rsrc = sd.gather ? static_cast<int64_t>(__ldg(&sd.gather[r])) : r;  // packed row r <- source row rsrc
  const T* row = static_cast<const T*>(sd.src) + rsrc * sd.rs;

  const int ex = scale_exponent(__uint_as_float(p.gmax[0]));
  const int ey = scale_exponent(__uint_as_float(p.gmax[1]));
  if (which == p.first_side && r == 0 && lane == 0) {
    const float c = p.mode == PREP_L2 ? -2.f : (p.mode == PREP_COSINE ? -1.f : 1.f);  // (PREP_INNER / PREP_INNER_NORM: +1)
    *p.coef       = c * p.coef_mul * ldexpf(1.f, -ex) * ldexpf(1.f, -ey);
  }
  float mean, amax;
  double ss;
  row_stats(row, sd.cs, p.k, p.center, p.xform, lane, mean, ss, amax);
  // One exponent E per matrix puts the matrix maximum in [2^14, 2^15).  A row whose own maximum lands more than
  // 2^12 below that (a single outlier / sentinel element elsewhere in the matrix: ADVICE r1) would slide towards the
  // fp16 subnormals and lose the 22 bits the split promises -- such a row takes its OWN exponent e_row, and the
  // epilogue multiplies its products by 2^(E - e_row) (exact: a power of two).  Ordinary data never takes this
  // branch: svec == 1 everywhere and the results are bit-identical to the single-scale scheme.
  const int E      = which ? ey : ex;
  const double nrm = p.mode == PREP_COSINE ? (sd.ext_norm_sq ? sqrt(static_cast<double>(sd.ext_norm_sq[rsrc])) : sqrt(ss)) : 1.0;
  const float aeff = p.mode == PREP_COSINE ? (nrm > 0.0 ? static_cast<float>(static_cast<double>(amax) / nrm) : 0.f) : amax;
  int e_row        = E;
  if (aeff > 0.f && aeff < 3.0e38f && ldexpf(aeff, E) < 8.0f) {
    e_row = max(E, min(scale_exponent(aeff), E + 120));
    if (lane == 0 && *reinterpret_cast<volatile unsigned*>(&p.nonuni[which]) == 0u) atomicExch(&p.nonuni[which], 1u);
  }
  float scale = ldexpf(1.f, e_row);
  if (p.mode == PREP_COSINE) scale = static_cast<float>(static_cast<double>(scale) / nrm);  // 1/0 -> inf -> NaN distances, like 0/0 in the definition
  if (lane == 0) sd.svec[r] = ldexpf(1.f, E - e_row);

  __half* orow   = sd.op + r * static_cast<int64_t>(p.nkb) * 64;
  const int kpad = p.nkb * 32;
  bool any_lo    = false;
  float res2     = 0.f;   // sum of (xs - hi)^2: the part of the row the hi half does not carry
  for (int t = lane; t < kpad; t += 32) {
    float xs = 0.f;
    if (t < p.k) xs = (ld_elem(row + t * sd.cs, p.xform) - mean) * scale;
    const __half h = __float2half_rn(xs);
    const float rs = xs - __half2float(h);   // exact in fp32
    const __half l = __float2half_rn(rs);
    res2 = fmaf(rs, rs, res2);
    any_lo |= (__half2float(l) != 0.f);
    const int b = t >> 5, j = t & 31;
    orow[b * 64 + j]      = h;
    orow[b * 64 + 32 + j] = l;
  }
  // operands that are exact in fp16 (fp16 inputs, small integers, ...) need no cross terms: the MMA
  // kernel then runs one product instead of three
  if (__any_sync(0xffffffffu, any_lo) && lane == 0 && *reinterpret_cast<volatile unsigned*>(p.has_lo) == 0u)
    atomicExch(p.has_lo, 1u);
  if (sd.lvec != nullptr) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) res2 += __shfl_xor_sync(0xffffffffu, res2, o);
    // back to the units of the row (2^-e_row; the cosine scale already holds 1 / |row|), rounded up
    if (lane == 0) sd.lvec[r] = ldexpf(sqrtf(res2) * (1.f + 1.f / 65536.f), -e_row);
  }
  if (lane == 0) {
    float t;
    if (p.mode == PREP_L2 || p.mode == PREP_INNER_NORM) t = sd.ext_norm_sq ? sd.ext_norm_sq[rsrc] : static_cast<float>(ss);
    else if (p.mode == PREP_COSINE) t = which == 0 ? 1.f : 0.f;
    else t = which == 0 ? p.tx_const : 0.f;
    sd.tvec[r] = t;
  }
}

}  // namespace b2d
