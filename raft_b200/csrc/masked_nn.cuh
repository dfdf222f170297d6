// Masked fusedL2NN (b2d_masked_l2_nn in nearest.cu; raft::distance::masked_l2_nn, the 1-NN step of connect_components):
// for every row i of x the nearest row j of y among the rows whose group g has adj[i, g] != 0.  Group g holds the rows
// [group_idxs[g-1], group_idxs[g]) of y (group_idxs[-1] = 0); rows at or after group_idxs[G-1] are in no group.
//
// Pre-pass kernels (after launch_prep, into the workspace), then the exact arg-min kernel of expanded_tc.cuh in its
// EPI_MINLOC_MASKED instantiation, which reads the tile classes to skip dead tiles:
//   masked_validate_kernel   group_idxs non-decreasing and inside [0, n]?  (no host round trip: a device flag; the
//                            finalisation then writes NaN / 0x7fffffff to every row, masked_poison_kernel)
//   masked_group_map_kernel  [n] group of every row of y (-1: none)
//   masked_adj_bits_kernel   the caller's byte matrix adj [m][G] as bits [ceil(m/32)][G]
//   masked_classify_kernel   per (x tile, y block) one byte of four tile classes (tc_params.cuh MaskClass)
#pragma once
#include <cstdint>
#include "nn_key.cuh"
#include "tc_params.cuh"

namespace b2d {

constexpr int MASK_SLAB_ROWS = 64;    // rows of x one consumer warpgroup owns in a tile
constexpr int MASK_HALF_COLS = TC_HN; // columns of y one wgmma covers

// group of row c of y: the first g with group_idxs[g] > c, -1 if there is none (for a valid group_idxs)
__host__ __device__ inline int masked_group_of(const int* group_idxs, int64_t G, int64_t c)
{
  int64_t lo = 0, hi = G;
  while (lo < hi) {
    const int64_t mid = (lo + hi) / 2;
    if (group_idxs[mid] > c) hi = mid;
    else lo = mid + 1;
  }
  return lo < G ? static_cast<int>(lo) : -1;
}

// Class of the tile (64-row slab `slab` of x, 128-column half `half` of y), from the adjacency bits
// ([ceil(m/32)][G], masked_adj_bits_kernel) and a valid group_idxs:
//   MASK_NONE     no (row, column) pair of the tile is adjacent (also: a tile outside the matrices)
//   MASK_ALL      every pair inside the matrices is adjacent
//   MASK_PARTIAL  otherwise
// A column in no group is never adjacent; an empty group holds no column and does not count.
__host__ __device__ inline int masked_tile_class(const unsigned* bits, const int* group_idxs, int64_t G, int64_t m, int64_t n,
                                                 int64_t slab, int64_t half)
{
  const int64_t r0 = slab * MASK_SLAB_ROWS, c0 = half * MASK_HALF_COLS;
  if (r0 >= m || c0 >= n || G <= 0) return MASK_NONE;
  const int64_t c1   = c0 + MASK_HALF_COLS < n ? c0 + MASK_HALF_COLS : n;   // columns [c0, c1)
  const int64_t rows = m - r0 < MASK_SLAB_ROWS ? m - r0 : MASK_SLAB_ROWS;
  const unsigned need0 = rows >= 32 ? ~0u : (1u << rows) - 1u;            // rows of the slab inside x, per bit word
  const unsigned need1 = rows >= 64 ? ~0u : rows <= 32 ? 0u : (1u << (rows - 32)) - 1u;
  const int64_t end    = group_idxs[G - 1];                                  // rows of y at or after it: no group
  bool any = false, all = c1 <= end;
  const int g0 = masked_group_of(group_idxs, G, c0);
  if (g0 >= 0) {
    const int g1 = masked_group_of(group_idxs, G, (c1 < end ? c1 : end) - 1);
    for (int g = g0; g <= g1; ++g) {
      if (group_idxs[g] <= (g > 0 ? group_idxs[g - 1] : 0)) continue;       // empty group
      const unsigned w0 = bits[(2 * slab) * G + g] & need0;
      const unsigned w1 = need1 ? bits[(2 * slab + 1) * G + g] & need1 : 0u;
      any |= (w0 | w1) != 0u;
      all &= w0 == need0 && w1 == need1;
    }
  }
  return !any ? MASK_NONE : all ? MASK_ALL : MASK_PARTIAL;
}

// one block: *bad = 1 unless 0 <= group_idxs[0] <= group_idxs[1] <= ... <= n
__global__ void __launch_bounds__(1024) masked_validate_kernel(unsigned* bad, const int* group_idxs, int64_t G, int64_t n)
{
  int b = 0;
  for (int64_t g = threadIdx.x; g < G; g += blockDim.x) {
    const int v = group_idxs[g];
    if (v < 0 || v > n || (g > 0 && v < group_idxs[g - 1])) b = 1;
  }
  b = __syncthreads_or(b);
  if (threadIdx.x == 0) *bad = b ? 1u : 0u;
}

__global__ void masked_group_map_kernel(int* grp, const int* group_idxs, int64_t G, int64_t n)
{
  const int64_t c = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (c < n) grp[c] = masked_group_of(group_idxs, G, c);
}

// one block per 32-row word of x: thread t builds the words of groups t, t + 256, ... (reads of adj coalesce along g)
__global__ void __launch_bounds__(256) masked_adj_bits_kernel(unsigned* bits, const uint8_t* adj, int64_t ld_adj, int64_t m,
                                                              int64_t G)
{
  const int64_t w  = blockIdx.x;
  const int rows   = static_cast<int>(m - 32 * w < 32 ? m - 32 * w : 32);
  const uint8_t* a = adj + 32 * w * ld_adj;
  for (int64_t g = threadIdx.x; g < G; g += blockDim.x) {
    unsigned word = 0u;
    for (int r = 0; r < rows; ++r) word |= (a[r * ld_adj + g] != 0 ? 1u : 0u) << r;
    bits[w * G + g] = word;
  }
}

// one thread per (x tile mt, y block nb): cls[nb][mt] = the four classes of (slab s, half h) at bits 2 (2 h + s);
// all NONE when group_idxs is invalid (*bad), so the arg-min kernel does no work
__global__ void masked_classify_kernel(uint8_t* cls, const unsigned* bits, const int* group_idxs, int64_t G, int64_t m,
                                       int64_t n, int tiles_m, int tiles_n, const unsigned* bad)
{
  const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= static_cast<int64_t>(tiles_m) * tiles_n) return;
  const int64_t nb = t / tiles_m, mt = t % tiles_m;
  unsigned b = 0u;
  if (*bad == 0u)
    for (int h = 0; h < 2; ++h)
      for (int s = 0; s < 2; ++s)
        b |= static_cast<unsigned>(masked_tile_class(bits, group_idxs, G, m, n, 2 * mt + s, 2 * nb + h)) << (2 * (2 * h + s));
  cls[t] = static_cast<uint8_t>(b);
}

// invalid group_idxs: every row becomes {0x7fffffff, NaN} (a value no valid call produces: a row without a candidate
// gets FLT_MAX)
__global__ void masked_poison_kernel(KvpIF* out, const unsigned* bad, int64_t m)
{
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= m || *bad == 0u) return;
  KvpIF o;
  o.key   = 0x7fffffff;
  o.value = __int_as_float(0x7fffffff);
  out[i]  = o;
}

}  // namespace b2d
