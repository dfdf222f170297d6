// Store-pattern probe for the EPI_STORE output stream of expanded_tc_kernel (scripts/store_probe.py builds and drives it).
// It writes a [m][ldd] fp32 matrix the way tc_stage_store does, with no MMAs and no operand loads: a persistent grid of one
// CTA per SM walking the work items of launch_tc's schedule (y block inner, `chunk` x tiles per item), two writer
// warpgroups per CTA that each own 64 rows of every 128 x 128 half tile, the same swizzled st.shared.v2 pattern into 8 KB
// staging boxes, fence.proxy.async and the pair protocol on a named barrier, and one issuing thread per warpgroup.  An idle
// spin per half stands in for the MMA turn.  What varies (one binary; everything but the box shape and the ring depth is a
// launch argument):
//   policy   L2 hint of the TMA stores: 0 evict_first, 1 evict_normal, 2 none
//   G        bytes per row per TMA store: 128 G.  G = 1 is a 2-D box of 64 rows x 32 columns (the kernel's earlier box);
//            G = 2 / 4 go through a 3-D view of the matrix, dims {32 columns, n / 32 column groups, m rows}, box
//            {32, G, 64 / G} (8 KB either way; G = 2 is the kernel's box)
//   P        pairs of boxes in the ring (2 P slots), wait_group.read P - 1 before a pair is written
//   chunk    x tiles per work item (1: the CTAs sweep whole rows of tiles together)
//   idle     clock cycles of spin before each half's staging
// Plus a plain row-major st.global.v4 sweep as a reference.  Results are meaningless as distances (each value is a
// function of its row and column only, so a broken store shows up in the check the driver does).
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdint>
#include "../raft_b200/csrc/ptx.cuh"

namespace {

using namespace b2d;

struct ProbeParams {
  int64_t m, n;
  int tiles_m, tiles_n, chunk, chunks_m;
  int64_t n_items;
  int policy;
  long long idle;
};

__device__ __forceinline__ uint64_t probe_policy(int policy)
{
  return policy == 0 ? ptx::policy_evict_first() : ptx::policy_evict_normal();
}

__device__ __forceinline__ void tma_store_3d(const void* tmap, uint32_t src, int32_t c0, int32_t c1, int32_t c2, uint64_t pol,
                                             bool hint)
{
  if (hint)
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group.L2::cache_hint [%0, {%2, %3, %4}], [%1], %5;"
                 :: "l"(reinterpret_cast<uint64_t>(tmap)), "r"(src), "r"(c0), "r"(c1), "r"(c2), "l"(pol) : "memory");
  else
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
                 :: "l"(reinterpret_cast<uint64_t>(tmap)), "r"(src), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_store_2d(const void* tmap, uint32_t src, int32_t c0, int32_t c1, uint64_t pol, bool hint)
{
  if (hint) ptx::tma_store_2d(tmap, src, c0, c1, pol);
  else
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                 :: "l"(reinterpret_cast<uint64_t>(tmap)), "r"(src), "r"(c0), "r"(c1) : "memory");
}
template <int N>
__device__ __forceinline__ void wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }

// Box b of a half tile (4 boxes of 8 KB, pair q = boxes 2 q, 2 q + 1):
//   G = 1: columns [32 b, 32 b + 32), all 64 rows      G = 2: columns [64 q, 64 q + 64), rows [32 s, 32 s + 32)
//   G = 4: all 128 columns, rows [16 b, 16 b + 16)
// Element (r, g, c) of a box (row r, column group g, column c of the group) sits at line L = G r + g, byte
// L * 128 + ((c / 4) ^ (L % 8)) * 16 + (c % 4) * 4 (SWIZZLE_128B over the box's 128-byte lines).
template <int G, int P>
__device__ __forceinline__ void stage_half(const float (&v)[64], const CUtensorMap* tmap, uint32_t stg, bool issuer,
                                           uint32_t& pair_it, int64_t row_w, int64_t col_w, const ProbeParams& p, uint64_t pol)
{
  constexpr int R = 64 / G;
  const int lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
  const int quad = lane >> 2, tq = lane & 3;
  const int wg   = threadIdx.x >> 7;
  const bool hint = p.policy != 2;
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    const uint32_t slot0 = stg + (pair_it % P) * 2 * 8192;
    ++pair_it;
    if (issuer) wait_read<P - 1>();
    ptx::bar_sync(2 + wg, 128);
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      const int b = 2 * q + s;
      const int rb = G == 1 ? 0 : G == 2 ? s : b;       // the box's block of R rows
      if ((16 * w) / R != rb) continue;                 // (warp-uniform) none of this warp's rows are in the box
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const int cb = G == 1 ? b : G == 2 ? q : 0;     // the box's block of 32 G columns
        if (i / (4 * G) != cb) continue;
        const int g = (i % (4 * G)) / 4;
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int r      = (16 * w + quad + 8 * j) % R;
          const uint32_t L = static_cast<uint32_t>(G * r + g);
          const uint32_t o = L * 128 + (((2 * (i % 4) + (tq >> 1)) ^ (L % 8)) * 16) + 8 * (tq & 1);
          ptx::st_shared_v2(slot0 + s * 8192 + o, v[4 * i + 2 * j], v[4 * i + 2 * j + 1]);
        }
      }
    }
    ptx::fence_proxy_async_smem();
    ptx::bar_sync(2 + wg, 128);
    if (issuer) {
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        const int b  = 2 * q + s;
        const int rb = G == 1 ? 0 : G == 2 ? s : b;
        const int cb = G == 1 ? b : G == 2 ? q : 0;
        const int64_t gc = col_w + 32 * G * cb, gr = row_w + R * rb;
        if (gc < p.n && gr < p.m) {
          if (G == 1) tma_store_2d(tmap, slot0 + s * 8192, static_cast<int32_t>(gc), static_cast<int32_t>(gr), pol, hint);
          else tma_store_3d(tmap, slot0 + s * 8192, 0, static_cast<int32_t>(gc / 32), static_cast<int32_t>(gr), pol, hint);
        }
      }
      ptx::tma_store_commit();
    }
  }
}

template <int G, int P>
__global__ void __launch_bounds__(256, 1) probe_kernel(const __grid_constant__ CUtensorMap tmap, const ProbeParams p)
{
  extern __shared__ __align__(1024) uint8_t smem[];
  const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
  const bool issuer = (threadIdx.x & 127) == 0;
  const uint32_t stg = ptx::smem_u32(smem) + wg * 2 * P * 8192;
  const uint64_t pol = probe_policy(p.policy);
  uint32_t pair_it = 0;
  float v[64];
  for (int64_t item = blockIdx.x; item < p.n_items; item += gridDim.x) {
    const int n_blk = static_cast<int>(item % p.tiles_n);
    const int mt0   = static_cast<int>(item / p.tiles_n) * p.chunk;
    const int mt1   = min(mt0 + p.chunk, p.tiles_m);
    const int nh    = static_cast<int64_t>(n_blk) * 256 + 128 < p.n ? 2 : 1;
    for (int mt = mt0; mt < mt1; ++mt)
      for (int h = 0; h < nh; ++h) {
        if (p.idle > 0) {
          const long long t0 = clock64();
          while (clock64() - t0 < p.idle) {}
        }
        const int64_t row_w = static_cast<int64_t>(mt) * 128 + 64 * wg;
        const int64_t col_w = static_cast<int64_t>(n_blk) * 256 + 128 * h;
        const float r0 = static_cast<float>(row_w + 16 * w + (lane >> 2));
        const float c0 = static_cast<float>(col_w + 2 * (lane & 3));
#pragma unroll
        for (int i = 0; i < 16; ++i)
#pragma unroll
          for (int j = 0; j < 2; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) v[4 * i + 2 * j + e] = fmaf(r0 + 8 * j, 1.0f / 1024.f, c0 + 8 * i + e);
        stage_half<G, P>(v, &tmap, stg, issuer, pair_it, row_w, col_w, p, pol);
      }
  }
  if (issuer) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

__global__ void sweep_kernel(float4* d, int64_t n4)
{
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4; i += stride)
    asm volatile("st.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(d + i), "f"(1.f), "f"(2.f), "f"(3.f), "f"(4.f) : "memory");
}

using EncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                              const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                              CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int encode(CUtensorMap* map, float* d, int64_t m, int64_t n, int64_t ldd, int G)
{
  static EncodeFn enc = nullptr;
  if (!enc) {
    void* fp = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      return 1;
    enc = reinterpret_cast<EncodeFn>(fp);
  }
  const cuuint32_t estr[3] = {1, 1, 1};
  CUresult r;
  if (G == 1) {
    const cuuint64_t dims[2] = {static_cast<cuuint64_t>(n), static_cast<cuuint64_t>(m)};
    const cuuint64_t str[1]  = {static_cast<cuuint64_t>(ldd * 4)};
    const cuuint32_t box[2]  = {32, 64};
    r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, d, dims, str, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  } else {
    const cuuint64_t dims[3] = {32, static_cast<cuuint64_t>(n / 32), static_cast<cuuint64_t>(m)};
    const cuuint64_t str[2]  = {128, static_cast<cuuint64_t>(ldd * 4)};
    const cuuint32_t box[3]  = {32, static_cast<cuuint32_t>(G), static_cast<cuuint32_t>(64 / G)};
    r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, d, dims, str, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  }
  return r == CUDA_SUCCESS ? 0 : 2;
}

template <int G, int P>
int launch(const CUtensorMap& map, const ProbeParams& p, int grid, cudaStream_t s)
{
  const int smem = 2 * 2 * P * 8192;
  if (cudaFuncSetAttribute(probe_kernel<G, P>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) return 3;
  probe_kernel<G, P><<<grid, 256, smem, s>>>(map, p);
  return cudaGetLastError() == cudaSuccess ? 0 : 4;
}

}  // namespace

// One probe launch (G = 0: the st.global.v4 sweep).  The schedule is launch_tc's: plan_tc_items(p, 6, max_chunk).
extern "C" int probe_launch(float* d, int64_t m, int64_t n, int64_t ldd, int G, int P, int policy, int max_chunk,
                            long long idle, void* stream)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (G == 0) {
    sweep_kernel<<<4 * sms, 1024, 0, s>>>(reinterpret_cast<float4*>(d), m * ldd / 4);
    return cudaGetLastError() == cudaSuccess ? 0 : 4;
  }
  if (n % 32 != 0 || (G > 1 && ldd % 32 != 0)) return 5;
  ProbeParams p{};
  p.m = m; p.n = n; p.policy = policy; p.idle = idle;
  p.tiles_m = static_cast<int>((m + 127) / 128);
  p.tiles_n = static_cast<int>((n + 255) / 256);
  int64_t chunk = static_cast<int64_t>(p.tiles_m) * p.tiles_n / (static_cast<int64_t>(sms) * 6);
  chunk = chunk < 1 ? 1 : chunk > max_chunk ? max_chunk : chunk;
  p.chunk    = static_cast<int>(chunk < p.tiles_m ? chunk : p.tiles_m);
  p.chunks_m = (p.tiles_m + p.chunk - 1) / p.chunk;
  p.n_items  = static_cast<int64_t>(p.tiles_n) * p.chunks_m;
  const int grid = static_cast<int>(p.n_items < sms ? p.n_items : sms);
  CUtensorMap map;
  if (int rc = encode(&map, d, m, n, ldd, G)) return rc;
  const int key = 10 * G + P;
  switch (key) {
    case 11: return launch<1, 1>(map, p, grid, s);
    case 12: return launch<1, 2>(map, p, grid, s);
    case 13: return launch<1, 3>(map, p, grid, s);
    case 21: return launch<2, 1>(map, p, grid, s);
    case 22: return launch<2, 2>(map, p, grid, s);
    case 41: return launch<4, 1>(map, p, grid, s);
    default: return 6;
  }
}
