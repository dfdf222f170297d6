// Mean shift (DESIGN.md K18, mean_shift.cu) on the epsilon neighbourhood of the tensor kernel (EPI_EPS).  Seeds are the x
// side (rows) of each EPI_EPS launch and the data the y side, so a batch of b seeds gets its adjacency as bytes
// adj [b][ld] (seed i, data row j at adj[i * ld + j]).  The neighbour sums A . X run on the tensor cores:
//   ms_sum_kernel      persistent, TMA-fed: per (128-seed tile, chunk of kMsChunk data rows, group of <= 4 k-blocks)
//                      the fp32 partial sums of the prepared data rows the tile's seeds reach, and their counts
//   ms_update_kernel   per seed: the partials folded in fp64 in ascending chunk order, the new mean, the stop rule
//   ms_step_end_kernel the run word of the next iteration
//   ms_bin_*           bin seeding (sklearn's get_bin_seeds): bins hashed, sorted, counted per first row of each bin
//   ms_survive / ms_unique / ms_compact kernels and two merge sorts: the surviving seeds merged and ordered
//   ms_walk_kernel     the greedy suppression walk over the ordered candidates
//   ms_label_kernel    labels from the arg-min keys of the data against the kept centres
// Only integer atomics; every floating-point sum runs in a fixed order.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <cstdint>

#include "nn_key.cuh"
#include "prep.cuh"
#include "ptx.cuh"

namespace b2d {

constexpr int kMsChunk     = 2048;   // data rows per fp32 partial of the neighbour sums (fixed: the sum order depends on n only)
constexpr int kMsKs        = 128;    // data rows per stage (one 128-byte adjacency row, one TMA box of prepared rows)
constexpr int kMsTileM     = 128;    // seeds per work item: two consumer warpgroups of 64
constexpr int kMsThreads   = 384;    // consumer warpgroups 0 and 1, then the producer warpgroup (one thread loads)
constexpr int kMsTileBytes = kMsTileM * kMsKs;   // 16 KB: the adjacency tile, and one prepared k-block of a stage
constexpr int kMsMaxStages = 4;

enum MsState : unsigned { MS_ACTIVE = 0, MS_STOPPED = 1, MS_DROPPED = 2 };

// control words of a fit
struct MsCtrl {
  unsigned run;      // 1 while some seed is active (the run word of every launch of an iteration)
  unsigned active;   // seeds still active after the current iteration (counted by ms_update_kernel)
  int n_iter;        // largest completed iteration count
  unsigned n_kept;   // centres kept by the walk
};

struct MsSumParams {
  int64_t m, n;          // seeds of the batch, data rows
  int d, nkb;            // columns, k-blocks of 32
  int gsz, ngroups;      // k-blocks per group, groups
  int tiles_m, nchunks;  // ceil(m / 128), ceil(n / kMsChunk)
  int64_t n_items;       // tiles_m * nchunks * ngroups
  int stages;
  const float* ysc;      // [n] per-row scale of the prepared data (prep.cuh svec)
  const unsigned* nonuni;  // [2]: nonuni[1], some data row took its own exponent
  float* part;           // [nchunks][m][d]
  unsigned* cnt;         // [nchunks][m]
  const unsigned* run_flag;
};

template <int G>
struct MsCarve {
  static constexpr int stages      = G >= 4 ? 2 : kMsMaxStages;
  static constexpr int stage_bytes = kMsTileBytes * (1 + G);
  static constexpr size_t bytes    = 1024 + static_cast<size_t>(stages) * stage_bytes + 2 * kMsMaxStages * 8;
  static_assert(bytes <= 232448, "exceeds the 227 KB per-CTA limit");
};

// D[64 x 64] += A[64 x 16] B[16 x 64]: A (fp16) from registers, B (fp16) from shared memory, MN-major (transposed):
// the 16 rows of a k-step are 16 rows of 128 bytes under SWIZZLE_128B, so one 128-byte packed row [hi | lo] of prepared
// data is one k of B and the 64 columns are hi (0..31) and lo (32..63) of the k-block.
__device__ __forceinline__ void ms_wgmma(float (&d)[32], const uint32_t (&a)[4], uint64_t desc_b)
{
  asm volatile(
    "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
    "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
    "%24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, 1, 1, 1, 1;\n"
    : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
      "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
      "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
      "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
    : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b)
    : "memory");
}
__device__ __forceinline__ void ms_fence_regs(float (&d)[32])
{
#pragma unroll
  for (int i = 0; i < 32; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// MN-major SWIZZLE_128B descriptor: 8-row groups of 128-byte rows 1024 B apart.  With N = 64 the tile is one swizzle
// atom wide, so the offset between atoms along N is never used; both offsets hold 1024.
__device__ __forceinline__ uint64_t ms_desc_mn(uint32_t smem_addr)
{
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(1024 >> 4) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// Two adjacency bytes (k, k + 1) of word w (pair h: bytes 2h, 2h + 1) as fp16x2 {1.0 or 0}: the bytes spread to the low
// byte of each half, then one integer multiply by 0x3C00 (fp16 1.0).  popc of the spread word counts them.
__device__ __forceinline__ uint32_t ms_spread(uint32_t w, int h) { return __byte_perm(w, 0u, h ? 0x4342u : 0x4140u); }

// Work item -> (seed tile, data chunk, k-block group); groups innermost so the items of one adjacency tile run together
__device__ __forceinline__ void ms_item(const MsSumParams& p, int64_t item, int& tile, int& chunk, int& grp)
{
  grp   = static_cast<int>(item % p.ngroups);
  chunk = static_cast<int>((item / p.ngroups) % p.nchunks);
  tile  = static_cast<int>(item / (static_cast<int64_t>(p.ngroups) * p.nchunks));
}

// Neighbour sums of one batch of seeds.  For seed i of the batch, chunk c and column t:
//   part[c][i][t] = 2^E * sum over data rows j of chunk c with adj[i][j] = 1 of x[j][t]   (fp32, hi and lo MMAs added)
//   cnt[c][i]     = #{j in chunk c : adj[i][j] = 1}
// where the prepared data row j is x[j] 2^(e_j) split into fp16 hi + lo (prep.cuh), E the data's matrix exponent.  A row
// that took its own exponent (nonuni) enters with the factor svec[j] = 2^(E - e_j) on its adjacency byte (exact in fp16
// down to 2^-24; a row below that, more than 2^23 under the data's maximum, is left out of the sums but not the counts).
template <int G>
__global__ void __launch_bounds__(kMsThreads, 1) ms_sum_kernel(const __grid_constant__ CUtensorMap adj_map,
                                                               const __grid_constant__ CUtensorMap data_map, MsSumParams p)
{
  if (p.run_flag != nullptr && __ldg(p.run_flag) == 0u) return;
  using C = MsCarve<G>;
  extern __shared__ uint8_t ms_smem_raw[];
  uint8_t* smem  = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(ms_smem_raw) + 1023) & ~uintptr_t{1023});
  uint64_t* full  = reinterpret_cast<uint64_t*>(smem + C::stages * C::stage_bytes);
  uint64_t* empty = full + kMsMaxStages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < C::stages; ++s) {
      ptx::mbar_init(&full[s], 1);
      ptx::mbar_init(&empty[s], 256);
    }
    ptx::fence_mbar_init();
  }
  __syncthreads();

  if (warp >= 8) {   // producer: its registers go to the consumers' accumulators
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp != 8 || lane != 0) return;
    ptx::prefetch_tmap(&adj_map);
    ptx::prefetch_tmap(&data_map);
    const uint64_t pol_adj = ptx::policy_evict_first(), pol_data = ptx::policy_evict_last();
    uint32_t it = 0;
    for (int64_t item = blockIdx.x; item < p.n_items; item += gridDim.x) {
      int tile, chunk, grp;
      ms_item(p, item, tile, chunk, grp);
      const int gn      = min(p.gsz, p.nkb - grp * p.gsz);
      const int64_t j0  = static_cast<int64_t>(chunk) * kMsChunk;
      const int nst     = static_cast<int>((min(static_cast<int64_t>(kMsChunk), p.n - j0) + kMsKs - 1) / kMsKs);
      for (int st = 0; st < nst; ++st, ++it) {
        const int slot = it % C::stages;
        ptx::mbar_wait(&empty[slot], ((it / C::stages) & 1u) ^ 1u);
        uint8_t* base = smem + slot * C::stage_bytes;
        ptx::mbar_expect_tx(&full[slot], static_cast<uint32_t>(kMsTileBytes * (1 + gn)));
        const int32_t jr = static_cast<int32_t>(j0 + st * kMsKs);
        ptx::tma_load_2d(base, &adj_map, &full[slot], jr, tile * kMsTileM, pol_adj);
        for (int q = 0; q < gn; ++q)
          ptx::tma_load_2d(base + kMsTileBytes * (1 + q), &data_map, &full[slot], (grp * p.gsz + q) * 64, jr, pol_data);
      }
    }
    return;
  }

  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  // consumers: warpgroup wg takes seeds [64 wg, 64 wg + 64) of the tile; thread (warp wi, lane g * 4 + t) holds rows
  // r0 = 16 wi + g and r0 + 8 of that slab (the m64 fragment layout, ptx.cuh)
  const int wg = warp >> 2, wi = warp & 3, g = lane >> 2, t = lane & 3;
  const int rl0 = 64 * wg + 16 * wi + g;   // row of the tile
  const bool scaled = __ldg(&p.nonuni[1]) != 0u;
  uint32_t it = 0;
  for (int64_t item = blockIdx.x; item < p.n_items; item += gridDim.x) {
    int tile, chunk, grp;
    ms_item(p, item, tile, chunk, grp);
    const int gn     = min(p.gsz, p.nkb - grp * p.gsz);
    const int64_t j0 = static_cast<int64_t>(chunk) * kMsChunk;
    const int nst    = static_cast<int>((min(static_cast<int64_t>(kMsChunk), p.n - j0) + kMsKs - 1) / kMsKs);
    float acc[G][32];
#pragma unroll
    for (int q = 0; q < G; ++q)
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[q][i] = 0.f;
    unsigned c0 = 0, c1 = 0;
    for (int st = 0; st < nst; ++st, ++it) {
      const int slot = it % C::stages;
      ptx::mbar_wait(&full[slot], (it / C::stages) & 1u);
      const uint8_t* base = smem + slot * C::stage_bytes;
      const uint32_t adj_s = ptx::smem_u32(base);
      uint32_t a[8][4];
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) {
        // 16-byte chunk ks of rows rl0 and rl0 + 8 (SWIZZLE_128B: chunk ks of row r sits at chunk ks ^ (r % 8))
        const uint4 v0 = ptx::ld_shared_v4(adj_s + rl0 * 128 + ((ks ^ (rl0 & 7)) << 4));
        const uint4 v1 = ptx::ld_shared_v4(adj_s + (rl0 + 8) * 128 + ((ks ^ (rl0 & 7)) << 4));
        const uint32_t w00 = t < 2 ? v0.x : v0.y, w01 = t < 2 ? v0.z : v0.w;   // k = 2t, 2t + 1 and 8 + 2t, 9 + 2t
        const uint32_t w10 = t < 2 ? v1.x : v1.y, w11 = t < 2 ? v1.z : v1.w;
        const uint32_t s0 = ms_spread(w00, t & 1), s1 = ms_spread(w10, t & 1);
        const uint32_t s2 = ms_spread(w01, t & 1), s3 = ms_spread(w11, t & 1);
        c0 += __popc(s0) + __popc(s2);
        c1 += __popc(s1) + __popc(s3);
        a[ks][0] = s0 * 0x3C00u; a[ks][1] = s1 * 0x3C00u; a[ks][2] = s2 * 0x3C00u; a[ks][3] = s3 * 0x3C00u;
        if (scaled) {
          const int64_t jb = j0 + st * kMsKs + ks * 16 + 2 * t;
          float sv[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int64_t j = jb + (e & 1) + 8 * (e >> 1);
            sv[e] = j < p.n ? __ldg(&p.ysc[j]) : 0.f;
          }
          const __half2 f01 = __floats2half2_rn(sv[0], sv[1]), f89 = __floats2half2_rn(sv[2], sv[3]);
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            __half2 h = *reinterpret_cast<__half2*>(&a[ks][r]);
            h = __hmul2(h, r < 2 ? f01 : f89);
            a[ks][r] = *reinterpret_cast<uint32_t*>(&h);
          }
        }
      }
      ptx::wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) {
#pragma unroll
        for (int q = 0; q < G; ++q)
          if (q < gn) ms_wgmma(acc[q], a[ks], ms_desc_mn(ptx::smem_u32(base + kMsTileBytes * (1 + q) + ks * 2048)));
      }
      ptx::wgmma_commit();
      ptx::wgmma_wait<0>();
#pragma unroll
      for (int q = 0; q < G; ++q) ms_fence_regs(acc[q]);
      ptx::mbar_arrive(&empty[slot]);
    }
    // epilogue: hi + lo of every column, one fp32 partial per (chunk, seed, column)
    const int64_t row_base = static_cast<int64_t>(tile) * kMsTileM + rl0;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int64_t i = row_base + 8 * j;
      if (i >= p.m) continue;
      float* out = p.part + (static_cast<int64_t>(chunk) * p.m + i) * p.d;
#pragma unroll
      for (int q = 0; q < G; ++q) {
        if (q >= gn) continue;
        const int kb = grp * p.gsz + q;
#pragma unroll
        for (int ii = 0; ii < 4; ++ii)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = kb * 32 + 8 * ii + 2 * t + e;
            if (col < p.d) out[col] = acc[q][4 * ii + 2 * j + e] + acc[q][4 * (ii + 4) + 2 * j + e];
          }
      }
    }
    c0 += __shfl_xor_sync(0xffffffffu, c0, 1);
    c0 += __shfl_xor_sync(0xffffffffu, c0, 2);
    c1 += __shfl_xor_sync(0xffffffffu, c1, 1);
    c1 += __shfl_xor_sync(0xffffffffu, c1, 2);
    if (grp == 0 && t == 0) {
      if (row_base < p.m) p.cnt[static_cast<int64_t>(chunk) * p.m + row_base] = c0;
      if (row_base + 8 < p.m) p.cnt[static_cast<int64_t>(chunk) * p.m + row_base + 8] = c1;
    }
  }
}

// One warp per seed of the batch [r0, r0 + m): the partials folded in fp64 in ascending chunk order (each lane its own
// columns, the squared shift reduced in a fixed xor tree), the mean rounded once to fp32, and sklearn's stop rule:
// no neighbour drops the seed; a shift <= thr or `max_iter` completed iterations stops it; else it goes on.
__global__ void ms_update_kernel(const unsigned* run, const float* part, const unsigned* cnt, int nchunks, int64_t m,
                                 int64_t r0, int d, const unsigned* gmax, double thr, int max_iter, float* mean,
                                 unsigned* state, int* iters, unsigned* inten, MsCtrl* ctrl)
{
  if (*run == 0u) return;
  const int lane = threadIdx.x & 31;
  const int64_t i = static_cast<int64_t>(blockIdx.x) * (blockDim.x / 32) + (threadIdx.x >> 5);
  if (i >= m) return;
  const int64_t gi = r0 + i;
  if (state[gi] != MS_ACTIVE) return;
  unsigned count = 0;
  for (int c = 0; c < nchunks; ++c) count += cnt[static_cast<int64_t>(c) * m + i];
  if (count == 0u) {
    if (lane == 0) state[gi] = MS_DROPPED;
    return;
  }
  const double undo = ldexp(1.0, -scale_exponent(__uint_as_float(gmax[1]))) / static_cast<double>(count);
  double ss = 0.0;
  float* mrow = mean + gi * d;
  for (int col = lane; col < d; col += 32) {
    double s = 0.0;
    for (int c = 0; c < nchunks; ++c) s += static_cast<double>(part[(static_cast<int64_t>(c) * m + i) * d + col]);
    const float nv = static_cast<float>(s * undo);
    const double dv = static_cast<double>(nv) - static_cast<double>(mrow[col]);
    ss += dv * dv;
    mrow[col] = nv;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  if (lane == 0) {
    inten[gi] = count;
    if (sqrt(ss) <= thr || iters[gi] == max_iter) {
      state[gi] = MS_STOPPED;
    } else {
      iters[gi] += 1;
      atomicAdd(&ctrl->active, 1u);
    }
  }
}

// after every batch of an iteration: the next iteration runs when some seed is still active
__global__ void ms_step_end_kernel(MsCtrl* ctrl)
{
  if (ctrl->run == 0u) return;
  ctrl->run    = ctrl->active != 0u ? 1u : 0u;
  ctrl->active = 0u;
}

// ------------------------------------------------------------------------------------------ bin seeding
__device__ __forceinline__ double ms_bin(float x, double h)
{
  return rint(static_cast<double>(x) / h) + 0.0;   // ties to even as np.round; + 0.0 makes -0 the bin of +0
}

// bin of each row, hashed (splitmix64 over the fp64 bits of its coordinates)
__global__ void ms_bin_hash_kernel(const float* x, int64_t ldx, int64_t n, int d, double h, unsigned long long* key, int* val)
{
  const int64_t r = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (r >= n) return;
  unsigned long long hsh = 0x9E3779B97F4A7C15ull;
  for (int k = 0; k < d; ++k) {
    unsigned long long z = static_cast<unsigned long long>(__double_as_longlong(ms_bin(x[r * ldx + k], h))) + hsh;
    z   = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z   = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    hsh = z ^ (z >> 31);
  }
  key[r] = hsh;
  val[r] = static_cast<int>(r);
}

__device__ __forceinline__ bool ms_same_bin(const float* x, int64_t ldx, int d, double h, int a, int b)
{
  for (int k = 0; k < d; ++k)
    if (ms_bin(x[static_cast<int64_t>(a) * ldx + k], h) != ms_bin(x[static_cast<int64_t>(b) * ldx + k], h)) return false;
  return true;
}

// Over the rows sorted stably by hash: the first row (smallest index) of each row's bin is its leader; freq[leader] counts
// the bin.  The leader is the first row of the hash run unless two bins share the hash, then the first equal row of it.
__global__ void ms_bin_count_kernel(const float* x, int64_t ldx, int64_t n, int d, double h, const unsigned long long* key,
                                    const int* val, unsigned* leader_of, unsigned* freq)
{
  const int64_t p = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const unsigned long long kp = key[p];
  int64_t lo = 0, hi = p;   // first position of the run of kp
  while (lo < hi) {
    const int64_t mid = (lo + hi) / 2;
    if (key[mid] < kp) lo = mid + 1;
    else hi = mid;
  }
  const int r = val[p];
  int64_t q = lo;
  while (q < p && !ms_same_bin(x, ldx, d, h, val[q], r)) ++q;
  leader_of[r] = static_cast<unsigned>(val[q]);
  atomicAdd(&freq[val[q]], 1u);
}

// flag[r] = 1 for a leader whose bin holds at least min_freq rows
__global__ void ms_bin_flag_kernel(const unsigned* leader_of, const unsigned* freq, int64_t n, unsigned min_freq, unsigned* flag)
{
  const int64_t r = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (r >= n) return;
  flag[r] = (leader_of[r] == static_cast<unsigned>(r) && freq[r] >= min_freq) ? 1u : 0u;
}

// seeds at fp32(bin) * fp32(h) in ascending order of their leaders (flag scanned into positions); when every row is a
// seed the seeds are the rows themselves (sklearn)
__global__ void ms_bin_seed_kernel(const float* x, int64_t ldx, int64_t n, int d, double h, const unsigned* leader_of,
                                   const unsigned* freq, unsigned min_freq, const unsigned* pos, const unsigned* total,
                                   float* seeds)
{
  const int64_t r = static_cast<int64_t>(blockIdx.x) * (blockDim.x / 32) + (threadIdx.x >> 5);
  if (r >= n) return;
  const int lane = threadIdx.x & 31;
  const bool all = static_cast<int64_t>(*total) == n;
  if (!all && !(leader_of[r] == static_cast<unsigned>(r) && freq[r] >= min_freq)) return;
  float* out = seeds + static_cast<int64_t>(all ? r : pos[r]) * d;
  const float hf = static_cast<float>(h);
  for (int k = lane; k < d; k += 32) {
    const float v = x[r * ldx + k];
    out[k] = all ? v : __fmul_rn(static_cast<float>(ms_bin(v, h)), hf);
  }
}

// ------------------------------------------------------------------------------------------ centres
__global__ void ms_init_kernel(int64_t s, unsigned* state, int* iters, unsigned* inten)
{
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= s) return;
  state[i] = MS_ACTIVE;
  iters[i] = 0;
  inten[i] = 0;
}

// survivors flagged; n_iter = the largest completed count over all seeds
__global__ void ms_survive_kernel(int64_t s, const unsigned* state, const int* iters, unsigned* flag, MsCtrl* ctrl)
{
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= s) return;
  flag[i] = state[i] == MS_STOPPED ? 1u : 0u;
  atomicMax(&ctrl->n_iter, iters[i]);
}

__global__ void ms_iota_kernel(int* out, int64_t n)
{
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) out[i] = static_cast<int>(i);
}

// out[pos[p]] = src[p] for the flagged p of [0, N), with the flags already scanned in place into pos (p is flagged when
// the next position differs) and *total the count
__global__ void ms_compact_kernel(int64_t N, const int* src, const unsigned* pos, const unsigned* total, int* out)
{
  const int64_t p = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (p >= N) return;
  if ((p + 1 < N ? pos[p + 1] : *total) != pos[p]) out[pos[p]] = src[p];
}

// Comparators of the candidate sorts (descending): by the mean's coordinates (ordered bits, lexicographic) then the
// intensity, with the seeds that did not survive last; and by the intensity then the coordinates.
struct MsByMean {
  const float* mean;
  const unsigned* inten;
  const unsigned* state;
  int d;
  __device__ bool operator()(int a, int b) const
  {
    const bool la = state[a] != MS_STOPPED, lb = state[b] != MS_STOPPED;
    if (la || lb) return !la && lb;
    for (int k = 0; k < d; ++k) {
      const int oa = ordered_bits(mean[static_cast<int64_t>(a) * d + k]), ob = ordered_bits(mean[static_cast<int64_t>(b) * d + k]);
      if (oa != ob) return oa > ob;
    }
    return inten[a] > inten[b];
  }
};
struct MsByIntensity {
  const float* mean;
  const unsigned* inten;
  int d;
  __device__ bool operator()(int a, int b) const
  {
    if (inten[a] != inten[b]) return inten[a] > inten[b];
    for (int k = 0; k < d; ++k) {
      const int oa = ordered_bits(mean[static_cast<int64_t>(a) * d + k]), ob = ordered_bits(mean[static_cast<int64_t>(b) * d + k]);
      if (oa != ob) return oa > ob;
    }
    return false;
  }
};

// flag[p] = 1 for the first of each run of bitwise-equal means in the mean order (it has the largest intensity)
__global__ void ms_unique_kernel(const int* order, const unsigned* n_sorted, const float* mean, int d, unsigned* flag,
                                 int64_t cap)
{
  const int64_t p = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (p >= cap) return;
  if (p >= static_cast<int64_t>(*n_sorted)) { flag[p] = 0u; return; }
  bool first = p == 0;
  if (!first) {
    const float* a = mean + static_cast<int64_t>(order[p]) * d;
    const float* b = mean + static_cast<int64_t>(order[p - 1]) * d;
    for (int k = 0; k < d && !first; ++k) first = __float_as_uint(a[k]) != __float_as_uint(b[k]);
  }
  flag[p] = first ? 1u : 0u;
}

// rows idx[0, n) of src [.][d] into dst [n][d], one warp per row
__global__ void ms_gather_kernel(const float* src, int d, const int* idx, int64_t n, float* dst)
{
  const int64_t r = static_cast<int64_t>(blockIdx.x) * (blockDim.x / 32) + (threadIdx.x >> 5);
  if (r >= n) return;
  const float* a = src + static_cast<int64_t>(idx[r]) * d;
  for (int k = threadIdx.x & 31; k < d; k += 32) dst[r * d + k] = a[k];
}

// The greedy walk over the candidates [r0, r0 + b) in order, with adj [b][ld] their EPI_EPS rows against all C
// candidates.  Candidate j is suppressed when a kept i < j has adj(i, j) (marked forward when i was kept) or adj(j, i)
// (checked on row j against the kept list): the symmetric relation.  status: 0 open, 1 kept, 2 suppressed.  One block.
__global__ void __launch_bounds__(1024) ms_walk_kernel(const uint8_t* adj, int64_t ld, int64_t r0, int64_t b, int64_t C,
                                                       uint8_t* status, int* kept, MsCtrl* ctrl)
{
  __shared__ unsigned nk;
  if (threadIdx.x == 0) nk = ctrl->n_kept;
  __syncthreads();
  for (int64_t jl = 0; jl < b; ++jl) {
    const int64_t j = r0 + jl;
    if (*reinterpret_cast<volatile uint8_t*>(&status[j]) == 2) continue;
    const uint8_t* row = adj + jl * ld;
    int hit = 0;
    for (unsigned q = threadIdx.x; q < nk; q += blockDim.x) hit |= row[kept[q]];
    if (__syncthreads_or(hit)) {
      if (threadIdx.x == 0) status[j] = 2;
      __syncthreads();
      continue;
    }
    for (int64_t c = j + 1 + threadIdx.x; c < C; c += blockDim.x)
      if (row[c]) status[c] = 2;
    if (threadIdx.x == 0) {
      status[j] = 1;
      kept[nk]  = static_cast<int>(j);
      nk += 1;
    }
    __threadfence_block();
    __syncthreads();
  }
  if (threadIdx.x == 0) ctrl->n_kept = nk;
}

// labels from the arg-min keys; with !cluster_all, a row farther than h2 from its centre (or with no finite one) is -1
__global__ void ms_label_kernel(const long long* keys, int64_t n, int cluster_all, float h2, int* labels)
{
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long k = keys[i];
  const bool none = k == KEY_EMPTY || !(cluster_all || key_dist(k) <= h2);
  labels[i] = none ? -1 : static_cast<int>(key_index(k));
}

}  // namespace b2d
