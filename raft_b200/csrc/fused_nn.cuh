// Helper kernels of the fused L2 / cosine 1-NN around the arg-min launches of expanded_tc.cuh: key initialisation and
// finalisation, and the screened search's sort keys, seeds, decisions and exact re-evaluation (with screen_tc.cuh).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include "nn_key.cuh"

namespace b2d {

// ---------------------------------------------------------------------------------------------
// small helper kernels for the NN path

__global__ void minloc_init_kernel(long long* keys, int64_t m)
{
  int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < m) keys[i] = KEY_EMPTY;
}


// packed key -> raft::KeyValuePair<int,float>{argmin, min distance}: clamp at 0, optional sqrt.
__global__ void minloc_finalize_kernel(KvpIF* out, const long long* keys, int64_t m, int do_sqrt,
                                       int merge_existing)
{
  int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const long long key = keys[i];
  const float v       = key_dist(key);
  float d             = v < 0.f ? 0.f : v;  // clamp at 0; NaN (zero-norm rows under cosine / NaN inputs) stays NaN
  if (do_sqrt) d = sqrtf(d);
  KvpIF o;
  o.key   = static_cast<int>(key_index(key));
  o.value = d;
  if (key == KEY_EMPTY) {  // no candidate (n == 0)
    o.key   = 0x7fffffff;
    o.value = __int_as_float(0x7f7fffff);
  }
  if (merge_existing) {
    // initOutBuffer == false: reduce into what the caller already has (argmin_op)
    KvpIF e = out[i];
    if ((e.value < o.value) || (e.value == o.value && e.key < o.key)) o = e;
  }
  out[i] = o;
}

// ---------------------------------------------------------------------------------------------
// Screened fusedL2NN (64 < k <= 128, large n; orchestration: fused_nn_keys_chunk in nearest.cu).  The chunk of y is packed
// in the order of its squared row norms; an exact pass over every 32nd block gives each row an upper bound of its
// minimum; the coarse pass of screen_tc.cuh (1 tensor product instead of 3) over ALL blocks keeps only the columns
// whose rigorous LOWER bound reaches that upper bound; those few are re-evaluated exactly, straight from the fp32
// inputs (sum (x-y)^2), together with the incumbent, so every finalist is measured with the same arithmetic.

// sort key of a database row: the bits of its squared norm (fp32, non-negative: the unsigned order is the float order)
__global__ void __launch_bounds__(256) nn_sortkey_kernel(const float* y, int64_t ldy, int64_t n, int k, const float* yn,
                                                         unsigned* key, int* val)
{
  const int lane  = threadIdx.x & 31;
  const int64_t r = static_cast<int64_t>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (r >= n) return;
  float ss = 0.f;
  if (yn != nullptr) {
    ss = __ldg(&yn[r]);
  } else {
    const float* row = y + r * ldy;
    for (int t = lane; t < k; t += 32) { const float v = __ldg(row + t); ss = fmaf(v, v, ss); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  }
  if (lane == 0) {
    key[r] = (ss >= 0.f) ? __float_as_uint(ss) : 0xffffffffu;   // NaN / negative caller norms: last
    val[r] = static_cast<int>(r);
  }
}

// after the exact sub-sampled pass: thr = incumbent distance, incumbent -> candidate, keys reset
__global__ void nn_seed_kernel(long long* keys, float4* aux, const float* xt, const float* xlo, int2* cand, unsigned* flags,
                               int64_t m, int64_t n, int64_t idx_offset)
{
  int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i == 0) {  // [0] list slots in use [1] overflow [2] go_screen [3] go_exact [4] redo_trial [5] candidates after the trial
    flags[0] = static_cast<unsigned>(m);   // [6] candidates found by the screen (slots are reserved in blocks)
    flags[1] = flags[2] = flags[3] = flags[4] = flags[5] = flags[6] = 0u;
  }
  if (i >= m) return;
  const long long key = keys[i];
  float t             = __int_as_float(0x7f800000);   // no incumbent: no bound
  int2 c              = make_int2(-1, -1);
  if (key != KEY_EMPTY) {
    t                 = key_dist(key);
    const long long j = key_index(key) - idx_offset;
    if (j >= 0 && j < n) {  // incumbent of THIS shard: re-measured with the exact arithmetic below
      c       = make_int2(static_cast<int>(i), static_cast<int>(j));
      keys[i] = KEY_EMPTY;
    }                        // else: a key merged in from another shard stays as it is
  }
  // screening compares v = d - |x|^2 with (bound - |x|^2), rounded up so that it stays an upper bound
  const float xn = xt[i];
  aux[i]  = make_float4((t - xn) + (t + xn) * (1.f / 2097152.f), sqrtf(xn) * (1.f + 1.f / 4194304.f), xlo[i], 0.f);
  cand[i] = c;
}

// device-side control of the screened search (fused_nn_keys in nearest.cu)
//   stage 1, after the trial screen: candidates per row above tau (or a full list) -> exact for the rest
//   stage 2, after the main screen : a full list -> exact for the blocks it covered
__global__ void nn_decide_kernel(unsigned* flags, unsigned m, float tau, int stage, const unsigned* nonuni)
{
  if (stage == 1) {
    flags[5]            = flags[6];
    // per-column scales (rows of y with their own exponent): the screen's single coefficient does not hold ->
    // everything it covered is redone by the exact kernel
    const unsigned redo = (flags[1] != 0u || nonuni[1] != 0u) ? 1u : 0u;
    const bool many     = static_cast<float>(flags[6]) > tau * static_cast<float>(m);
    flags[4]            = redo;
    flags[3]            = (redo || many) ? 1u : 0u;
    flags[2]            = flags[3] ? 0u : 1u;
  } else if (flags[2] != 0u && flags[1] != 0u) {
    flags[3] = 1u;
  }
}

// one warp per candidate, straight from the original fp32 inputs:
//   family 0  d = sum (x_i - y_j)^2
//   family 1  d = 1 - <x', y'> / (|x'| |y'|), x' = x - mean(x) when centred (correlation), else x (cosine)
// (k <= 128 on this path: a lane holds at most 4 elements of each row in registers)
__global__ void __launch_bounds__(256) nn_exact_kernel(long long* keys, const int2* cand, const unsigned* cnt,
                                                       unsigned cap, const float* x, int64_t ldx, const float* y,
                                                       int64_t ldy, int k, int64_t idx_offset, int family, int center,
                                                       unsigned n_seed, const int* col_map)
{
  const int lane       = threadIdx.x & 31;
  const unsigned total = min(*cnt, cap);
  const unsigned nwarp = gridDim.x * (blockDim.x >> 5);
  for (unsigned c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); c < total; c += nwarp) {
    int2 ij = cand[c];
    if (ij.x < 0) continue;
    // the first n_seed entries (nn_seed_kernel: the incumbents) hold source rows of y, the screen's entries packed
    // positions of the norm-sorted chunk
    if (c >= n_seed && col_map != nullptr) ij.y = __ldg(&col_map[ij.y]);
    const float* xr = x + static_cast<int64_t>(ij.x) * ldx;
    const float* yr = y + static_cast<int64_t>(ij.y) * ldy;
    float xv[4], yv[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int t = lane + 32 * u;
      xv[u]       = t < k ? __ldg(xr + t) : 0.f;
      yv[u]       = t < k ? __ldg(yr + t) : 0.f;
    }
    float res;
    if (family == 0) {
      float acc = 0.f;
#pragma unroll
      for (int u = 0; u < 4; ++u) { const float d = xv[u] - yv[u]; acc = fmaf(d, d, acc); }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      res = acc;
    } else {
      // fp64 throughout, rounded once: like prep (which normalises in fp64), the result does not depend on the scale
      // of the rows.  In fp32, nx * ny overflows for rows of norm ~2^32 and underflows for ~2^-32 (a distance of 1, or
      // below 0, for every candidate of such a row); in fp64 every power-of-two scale of an fp32 row stays in range.
      double mx = 0.0, my = 0.0;
      if (center) {
        double sx = (static_cast<double>(xv[0]) + xv[1]) + (static_cast<double>(xv[2]) + xv[3]);
        double sy = (static_cast<double>(yv[0]) + yv[1]) + (static_cast<double>(yv[2]) + yv[3]);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { sx += __shfl_xor_sync(0xffffffffu, sx, o); sy += __shfl_xor_sync(0xffffffffu, sy, o); }
        mx = sx / k;
        my = sy / k;
      }
      double dot = 0.0, nx = 0.0, ny = 0.0;
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const bool in  = lane + 32 * u < k;
        const double a = in ? xv[u] - mx : 0.0, b = in ? yv[u] - my : 0.0;
        dot = fma(a, b, dot); nx = fma(a, a, nx); ny = fma(b, b, ny);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        dot += __shfl_xor_sync(0xffffffffu, dot, o);
        nx += __shfl_xor_sync(0xffffffffu, nx, o);
        ny += __shfl_xor_sync(0xffffffffu, ny, o);
      }
      res = static_cast<float>(1.0 - dot / sqrt(nx * ny));
    }
    if (lane == 0) atomicMin(&keys[ij.x], key_pack(res, static_cast<long long>(ij.y) + idx_offset));
  }
}

}  // namespace b2d
