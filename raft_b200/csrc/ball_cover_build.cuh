// Build kernels of the random ball cover (ball_cover.cu, the one file that includes this header: the non-template
// kernels below are defined once).  The rounding helpers and the queries are in ball_cover.cuh.
#pragma once
#include "ball_cover.cuh"

namespace b2d {

// ------------------------------------------------------------------------------------------
// build

// sampling keys: (31-bit hash of (seed, row)) << 32 | row, rows with a non-finite coordinate last
template <int D>
__global__ void bc_sample_kernel(const float* x, int64_t ldx, int n, unsigned long long seed, unsigned long long* keys)
{
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    bool fin = true;
    for (int c = 0; c < D; ++c) fin = fin && isfinite(x[i * ldx + c]);
    unsigned long long z = seed + 0x9E3779B97F4A7C15ull * (static_cast<unsigned long long>(i) + 1);   // splitmix64
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z ^= z >> 31;
    const unsigned long long h = fin ? (z >> 33) : 0xFFFFFFFFull;
    keys[i] = (h << 32) | static_cast<unsigned>(i);
  }
}

// landmark j = the row of sorted key j
template <int D>
__global__ void bc_landmark_kernel(const float* x, int64_t ldx, const unsigned long long* keys, int nl, float* lm)
{
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < nl; j += gridDim.x * blockDim.x) {
    const int64_t row = static_cast<unsigned>(keys[j]);
    for (int c = 0; c < D; ++c) lm[j * D + c] = x[row * ldx + c];
  }
}

// Every finite row to its nearest finite landmark by (s, landmark): key (landmark << 32) | bits of s, value the row.
// Rows with a non-finite coordinate get landmark nl.  Landmarks are staged in shared memory, kBcTile at a time.
constexpr int kBcTile = 1024;
template <int D>
__global__ void __launch_bounds__(256) bc_assign_kernel(const float* x, int64_t ldx, int n, const float* lm, int nl,
                                                        unsigned long long* keys, int* vals)
{
  __shared__ float tile[kBcTile * D];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  float p[D];
  bool fin = i < n;
  for (int c = 0; c < D; ++c) {
    p[c] = i < n ? x[static_cast<int64_t>(i) * ldx + c] : 0.f;
    fin  = fin && isfinite(p[c]);
  }
  long long best = KEY_EMPTY;
  for (int t0 = 0; t0 < nl; t0 += kBcTile) {
    const int cnt = min(kBcTile, nl - t0);
    __syncthreads();
    for (int e = threadIdx.x; e < cnt * D; e += blockDim.x) tile[e] = lm[t0 * D + e];
    __syncthreads();
    if (fin)
      for (int j = 0; j < cnt; ++j) {
        const float* L = tile + j * D;
        bool lf = true;
        for (int c = 0; c < D; ++c) lf = lf && isfinite(L[c]);
        if (lf) best = min(best, key_pack(bc_s<D>(p, L), t0 + j));
      }
  }
  if (i < n) {
    const unsigned long long lab = fin ? static_cast<unsigned long long>(key_index(best)) : static_cast<unsigned long long>(nl);
    const unsigned sb            = fin ? static_cast<unsigned>(best >> 32) : 0u;   // s >= 0: its ordered bits are its bits
    keys[i] = (lab << 32) | sb;
    vals[i] = i;
  }
}

// ball offsets from the sorted keys: off[l] = first position whose landmark is >= l, l in [0, nl + 1]
__global__ void bc_offsets_kernel(const unsigned long long* keys, int n, int nl, int* off)
{
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t <= n; t += gridDim.x * blockDim.x) {
    const int prev = t > 0 ? static_cast<int>(keys[t - 1] >> 32) : -1;
    const int cur  = t < n ? static_cast<int>(keys[t] >> 32) : nl + 1;
    for (int l = prev + 1; l <= cur; ++l) off[l] = t;
  }
}

// the rows in position order: coordinates, caller's row, s to the landmark
template <int D>
__global__ void bc_permute_kernel(const float* x, int64_t ldx, const unsigned long long* keys, const int* perm, int n,
                                  float* pts, int* ids, float* rl)
{
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += gridDim.x * blockDim.x) {
    const int row = perm[t];
    for (int c = 0; c < D; ++c) pts[static_cast<int64_t>(t) * D + c] = x[static_cast<int64_t>(row) * ldx + c];
    ids[t] = row;
    rl[t]  = __uint_as_float(static_cast<unsigned>(keys[t]));
  }
}

__global__ void bc_radius_kernel(const int* off, const float* rl, int nl, float* rhi)
{
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < nl; j += gridDim.x * blockDim.x)
    rhi[j] = off[j + 1] > off[j] ? bc_dhi(rl[off[j + 1] - 1]) : -1.f;
}

}  // namespace b2d
