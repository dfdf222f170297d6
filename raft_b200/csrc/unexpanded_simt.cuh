// K2: unexpanded metrics (L1, L2Unexpanded, L2SqrtUnexpanded, Linf, Canberra, LpUnexpanded) --
// not bilinear, so no tensor-core form: a register-tiled FP32 kernel (SURVEY.md 8(a4)).
//
// 128x128 output tile per CTA, 256 threads, 8x8 outputs per thread, k-blocks of 32 floats staged
// in shared memory as 128-byte rows whose 16-byte chunks are XOR-swizzled by (row & 7) -- the
// same pattern TMA's SWIZZLE_128B produces -- so both the cooperative 16-byte loads into smem
// and the LDS.128 reads along k are bank-conflict free.  Global reads are 128-byte coalesced
// float4 loads when the rows are 16-byte aligned and k % 4 == 0, scalar otherwise (any row /
// column stride, zero-filled tails: what the reference's Contractions_NT loader guaranteed,
// cpp/include/raft/linalg/detail/contractions.cuh:186-193).  The next k-block is fetched into
// registers while the current one is consumed (software pipelining, double-buffered smem).
// Bound: FP32 pipe (>= 2 lane-ops per pair-element), not HBM -- see DESIGN.md.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdint>
#include "ptx.cuh"

namespace b2d {

constexpr int UX_BM = 128, UX_BN = 128, UX_KB = 32, UX_THREADS = 256;
constexpr int UX_SMEM_BYTES = 2 * (UX_BM + UX_BN) * UX_KB * 4;
constexpr int UX_TMA_STAGES = 3;
constexpr int UX_TMA_SMEM_BYTES = UX_TMA_STAGES * (UX_BM + UX_BN) * UX_KB * 4 + 64;

enum UxMetric : int { UX_L1 = 0, UX_L2 = 1, UX_L2SQRT = 2, UX_LINF = 3, UX_CANBERRA = 4, UX_LP = 5,
                      UX_HAMMING = 6, UX_KL = 7, UX_JS = 8,
                      UX_KL_REV = 9,
                      UX_BRAYCURTIS = 10 };  // sum |a - b| / sum |a + b|: the denominator rides in a second accumulator  // KL with the operand roles swapped: sum b log(b/a) (Fortran-order inputs)

struct UxParams {
  const float* x;
  const float* y;
  float* dist;
  int64_t xrs, xcs, yrs, ycs;  // element strides
  int64_t ldd;
  int64_t m, n;
  int k;
  int vec_x, vec_y;  // float4 path legal
  float p, inv_p;
  int tiles_n;
};

template <int kMetric>
__device__ __forceinline__ void ux_acc(float& acc, float a, float b, float p)
{
  if (kMetric == UX_L1) {
    acc += fabsf(a - b);
  } else if (kMetric == UX_L2 || kMetric == UX_L2SQRT) {
    const float d = a - b;
    acc           = fmaf(d, d, acc);
  } else if (kMetric == UX_LINF) {
    acc = fmaxf(acc, fabsf(a - b));
  } else if (kMetric == UX_CANBERRA) {
    // |a-b| / (|a|+|b|), 0/0 -> 0 (scipy / reference convention).  s == 0 implies d == 0, so
    // clamping s away from zero turns the special case into 0 * finite = 0 without a select;
    // one MUFU.RCP per element makes this metric MUFU-bound (16 lanes/clk/SM).
    const float d = fabsf(a - b);
    const float s = fmaxf(fabsf(a) + fabsf(b), 1e-30f);
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(s));
    acc = fmaf(d, r, acc);
  } else if (kMetric == UX_HAMMING) {
    acc += (a != b) ? 1.f : 0.f;  // final: / k
  } else if (kMetric == UX_KL) {
    // sum x log(x/y), terms with x == 0 contribute 0 ([RECALLED] reference epilogue halves the sum;
    // see ux_fin).  log2 domain, scaled by ln 2 at the end; a zero-padded k tail adds 0.
    const float t = a * (__log2f(a) - __log2f(b));
    acc += (a == 0.f) ? 0.f : t;
  } else if (kMetric == UX_KL_REV) {
    // the column-major entry point computes D^T with x and y exchanged (pairwise.cu); KL is not symmetric,
    // so the kernel accumulates KL(b || a) there -- the reference's !is_row_major branch did the same swap
    const float t = b * (__log2f(b) - __log2f(a));
    acc += (b == 0.f) ? 0.f : t;
  } else if (kMetric == UX_BRAYCURTIS) {
    acc += fabsf(a - b);  // numerator; the denominator sum |a + b| accumulates next to it (ux_den)
  } else if (kMetric == UX_JS) {
    // sum x log(x/m) + y log(y/m), m = (x+y)/2; 0 log 0 = 0
    const float lm = __log2f(0.5f * (a + b));
    const float ta = a * (__log2f(a) - lm);
    const float tb = b * (__log2f(b) - lm);
    acc += ((a == 0.f) ? 0.f : ta) + ((b == 0.f) ? 0.f : tb);
  } else {
    const float d = fabsf(a - b);
    acc += exp2f(p * __log2f(d));  // d == 0 -> log2 = -inf -> exp2 = 0
  }
}

template <int kMetric>
__device__ __forceinline__ void ux_den(float& den, float a, float b)
{
  if (kMetric == UX_BRAYCURTIS) den += fabsf(a + b);
}

template <int kMetric>
__device__ __forceinline__ float ux_fin(float acc, float inv_p)
{
  if (kMetric == UX_L2SQRT) return sqrtf(acc);
  if (kMetric == UX_LP) return exp2f(inv_p * __log2f(acc));
  if (kMetric == UX_HAMMING) return acc * inv_p;                          // inv_p carries 1/k
  if (kMetric == UX_KL || kMetric == UX_KL_REV) return 0.5f * 0.69314718056f * acc;  // 0.5 * sum x ln(x/y)
  if (kMetric == UX_JS) return sqrtf(fmaxf(0.5f * 0.69314718056f * acc, 0.f));  // sqrt(JS divergence), natural log
  return acc;
}

__device__ __forceinline__ float4 ux_load4(const float* base, int64_t rs, int64_t cs, int64_t row,
                                           int64_t nrows, int kcol, int k, int vec)
{
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (row < nrows) {
    const float* p = base + row * rs;
    if (vec && kcol + 3 < k) {
      v = __ldg(reinterpret_cast<const float4*>(p + kcol));
    } else {
      if (kcol < k) v.x = __ldg(p + (int64_t)kcol * cs);
      if (kcol + 1 < k) v.y = __ldg(p + (int64_t)(kcol + 1) * cs);
      if (kcol + 2 < k) v.z = __ldg(p + (int64_t)(kcol + 2) * cs);
      if (kcol + 3 < k) v.w = __ldg(p + (int64_t)(kcol + 3) * cs);
    }
  }
  return v;
}

template <int kMetric>
__global__ void __launch_bounds__(UX_THREADS, 1) unexpanded_simt_kernel(const UxParams p)
{
  extern __shared__ __align__(128) float ux_smem[];
  float(*sx)[UX_BM * UX_KB] = reinterpret_cast<float(*)[UX_BM * UX_KB]>(ux_smem);
  float(*sy)[UX_BN * UX_KB] = reinterpret_cast<float(*)[UX_BN * UX_KB]>(ux_smem + 2 * UX_BM * UX_KB);

  const int tid = threadIdx.x;
  const int tx  = tid & 15;  // column group
  const int ty  = tid >> 4;  // row group
  const int64_t tile = blockIdx.x;
  const int64_t m0   = (tile / p.tiles_n) * UX_BM;
  const int64_t n0   = (tile % p.tiles_n) * UX_BN;

  constexpr int kD = kMetric == UX_BRAYCURTIS ? 8 : 1;  // second accumulator only where a metric needs one
  float acc[8][8], den[kD][kD];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) { acc[i][j] = 0.f; den[i % kD][j % kD] = 0.f; }

  const int nkb = (p.k + UX_KB - 1) / UX_KB;
  float4 gx[4], gy[4];

  auto gload = [&](int kb) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int f = tid + UX_THREADS * i, row = f >> 3, c4 = f & 7;
      gx[i] = ux_load4(p.x, p.xrs, p.xcs, m0 + row, p.m, kb * UX_KB + c4 * 4, p.k, p.vec_x);
      gy[i] = ux_load4(p.y, p.yrs, p.ycs, n0 + row, p.n, kb * UX_KB + c4 * 4, p.k, p.vec_y);
    }
  };
  auto sstore = [&](int buf) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int f = tid + UX_THREADS * i, row = f >> 3, c4 = f & 7;
      const int off = row * UX_KB + ((c4 ^ (row & 7)) << 2);
      *reinterpret_cast<float4*>(&sx[buf][off]) = gx[i];
      *reinterpret_cast<float4*>(&sy[buf][off]) = gy[i];
    }
  };

  gload(0);
  sstore(0);
  __syncthreads();

  for (int kb = 0; kb < nkb; ++kb) {
    const int buf = kb & 1;
    if (kb + 1 < nkb) gload(kb + 1);
#pragma unroll 2
    for (int c4 = 0; c4 < 8; ++c4) {
      float4 a[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int row = ty + 16 * i;
        a[i] = *reinterpret_cast<const float4*>(&sx[buf][row * UX_KB + ((c4 ^ (row & 7)) << 2)]);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int row  = tx + 16 * j;
        const float4 b = *reinterpret_cast<const float4*>(&sy[buf][row * UX_KB + ((c4 ^ (row & 7)) << 2)]);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          ux_acc<kMetric>(acc[i][j], a[i].x, b.x, p.p);
          ux_acc<kMetric>(acc[i][j], a[i].y, b.y, p.p);
          ux_acc<kMetric>(acc[i][j], a[i].z, b.z, p.p);
          ux_acc<kMetric>(acc[i][j], a[i].w, b.w, p.p);
          ux_den<kMetric>(den[i % kD][j % kD], a[i].x, b.x);
          ux_den<kMetric>(den[i % kD][j % kD], a[i].y, b.y);
          ux_den<kMetric>(den[i % kD][j % kD], a[i].z, b.z);
          ux_den<kMetric>(den[i % kD][j % kD], a[i].w, b.w);
        }
      }
    }
    if (kb + 1 < nkb) {
      sstore(buf ^ 1);
      __syncthreads();
    }
  }

#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int64_t gi = m0 + ty + 16 * i;
    if (gi >= p.m) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int64_t gj = n0 + tx + 16 * j;
      if (gj < p.n)
        __stcs(p.dist + gi * p.ldd + gj,
               kMetric == UX_BRAYCURTIS ? acc[i][j] / den[i % kD][j % kD] : ux_fin<kMetric>(acc[i][j], p.inv_p));
    }
  }
}

__device__ __forceinline__ uint64_t ux_pk(float lo, float hi)
{
  uint64_t r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
  return r;
}
__device__ __forceinline__ void ux_unpk(uint64_t v, float& lo, float& hi)
{
  asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
// (Hopper has no packed f32x2 pipe: two scalar operations on the halves of the pair)
__device__ __forceinline__ uint64_t ux_add2(uint64_t a, uint64_t b)
{
  float a0, a1, b0, b1;
  ux_unpk(a, a0, a1);
  ux_unpk(b, b0, b1);
  return ux_pk(a0 + b0, a1 + b1);
}
__device__ __forceinline__ uint64_t ux_fma2(uint64_t a, uint64_t b, uint64_t c)
{
  float a0, a1, b0, b1, c0, c1;
  ux_unpk(a, a0, a1);
  ux_unpk(b, b0, b1);
  ux_unpk(c, c0, c1);
  return ux_pk(fmaf(a0, b0, c0), fmaf(a1, b1, c1));
}
__device__ __forceinline__ float ux_max3(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }

// TMA-fed variant (rows 16-byte aligned, k % 4 == 0, row-major): the same 128x128x32 tiles arrive
// by cp.async.bulk.tensor with SWIZZLE_128B -- the XOR pattern the manual loader writes -- through
// a 3-stage mbarrier ring, so no thread spends registers or issue slots on staging and OOB rows /
// k tails are zero-filled by the hardware.  One elected thread issues; all 256 threads compute.
template <int kMetric>
__global__ void __launch_bounds__(UX_THREADS, 1)
unexpanded_tma_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_y,
                      const UxParams p)
{
  extern __shared__ __align__(1024) uint8_t ux_raw[];
  if ((ptx::smem_u32(ux_raw) & 1023u) != 0u) __trap();
  constexpr int kTile = UX_BM * UX_KB;  // floats per operand tile
  float* sx       = reinterpret_cast<float*>(ux_raw);
  float* sy       = sx + UX_TMA_STAGES * kTile;
  uint64_t* full  = reinterpret_cast<uint64_t*>(sy + UX_TMA_STAGES * kTile);

  const int tid = threadIdx.x;
  const int tx  = tid & 15;
  const int ty  = tid >> 4;
  const int64_t tile = blockIdx.x;
  const int m0       = static_cast<int>(tile / p.tiles_n) * UX_BM;
  const int n0       = static_cast<int>(tile % p.tiles_n) * UX_BN;
  const int nkb      = (p.k + UX_KB - 1) / UX_KB;

  if (tid == 0) {
    for (int i = 0; i < UX_TMA_STAGES; ++i) ptx::mbar_init(&full[i], 1);
    ptx::fence_mbar_init();
  }
  __syncthreads();
  const uint64_t pol = ptx::policy_evict_last();
  auto issue = [&](int kb) {
    const int s = kb % UX_TMA_STAGES;
    ptx::mbar_expect_tx(&full[s], 2 * kTile * 4);
    ptx::tma_load_2d(sx + s * kTile, &tmap_x, &full[s], kb * UX_KB, m0, pol);
    ptx::tma_load_2d(sy + s * kTile, &tmap_y, &full[s], kb * UX_KB, n0, pol);
  };
  if (tid == 0)
    for (int kb = 0; kb < UX_TMA_STAGES - 1 && kb < nkb; ++kb) issue(kb);

  // L2 / L2Sqrt: (even-k, odd-k) pair math;
  // every output keeps an (even-k, odd-k) pair of partial sums that is folded at the end.
  constexpr bool kPackedL2 = (kMetric == UX_L2 || kMetric == UX_L2SQRT);
  constexpr int kD = kMetric == UX_BRAYCURTIS ? 8 : 1;
  float acc[8][8], den[kD][kD];
  uint64_t acc2[kPackedL2 ? 8 : 1][kPackedL2 ? 8 : 1];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      acc[i][j] = 0.f;
      den[i % kD][j % kD] = 0.f;
      if (kPackedL2) acc2[i % (kPackedL2 ? 8 : 1)][j % (kPackedL2 ? 8 : 1)] = 0ull;
    }

  for (int kb = 0; kb < nkb; ++kb) {
    const int s = kb % UX_TMA_STAGES;
    ptx::mbar_wait(&full[s], (kb / UX_TMA_STAGES) & 1);
    const float* bx = sx + s * kTile;
    const float* by = sy + s * kTile;
#pragma unroll 2
    for (int c4 = 0; c4 < 8; ++c4) {
      float4 a[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int row = ty + 16 * i;
        a[i] = *reinterpret_cast<const float4*>(&bx[row * UX_KB + ((c4 ^ (row & 7)) << 2)]);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int row  = tx + 16 * j;
        const float4 b = *reinterpret_cast<const float4*>(&by[row * UX_KB + ((c4 ^ (row & 7)) << 2)]);
        if (kPackedL2) {
          const uint64_t nb0 = ux_pk(-b.x, -b.y), nb1 = ux_pk(-b.z, -b.w);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const uint64_t d0 = ux_add2(ux_pk(a[i].x, a[i].y), nb0);
            const uint64_t d1 = ux_add2(ux_pk(a[i].z, a[i].w), nb1);
            uint64_t& t       = acc2[i % (kPackedL2 ? 8 : 1)][j % (kPackedL2 ? 8 : 1)];
            t                 = ux_fma2(d0, d0, t);
            t                 = ux_fma2(d1, d1, t);
          }
        } else if (kMetric == UX_LINF) {
          const uint64_t nb0 = ux_pk(-b.x, -b.y), nb1 = ux_pk(-b.z, -b.w);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            float d0, d1, d2, d3;
            ux_unpk(ux_add2(ux_pk(a[i].x, a[i].y), nb0), d0, d1);
            ux_unpk(ux_add2(ux_pk(a[i].z, a[i].w), nb1), d2, d3);
            acc[i][j] = ux_max3(acc[i][j], fabsf(d0), fabsf(d1));
            acc[i][j] = ux_max3(acc[i][j], fabsf(d2), fabsf(d3));
          }
        } else {
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            ux_acc<kMetric>(acc[i][j], a[i].x, b.x, p.p);
            ux_acc<kMetric>(acc[i][j], a[i].y, b.y, p.p);
            ux_acc<kMetric>(acc[i][j], a[i].z, b.z, p.p);
            ux_acc<kMetric>(acc[i][j], a[i].w, b.w, p.p);
            ux_den<kMetric>(den[i % kD][j % kD], a[i].x, b.x);
            ux_den<kMetric>(den[i % kD][j % kD], a[i].y, b.y);
            ux_den<kMetric>(den[i % kD][j % kD], a[i].z, b.z);
            ux_den<kMetric>(den[i % kD][j % kD], a[i].w, b.w);
          }
        }
      }
    }
    // every thread is done with the stage that block kb-1 used: refill it with block kb+STAGES-1
    __syncthreads();
    if (tid == 0 && kb + UX_TMA_STAGES - 1 < nkb) issue(kb + UX_TMA_STAGES - 1);
  }
  if (kPackedL2) {
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float lo, hi;
        ux_unpk(acc2[i % (kPackedL2 ? 8 : 1)][j % (kPackedL2 ? 8 : 1)], lo, hi);
        acc[i][j] = lo + hi;
      }
  }

#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int64_t gi = m0 + ty + 16 * i;
    if (gi >= p.m) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int64_t gj = n0 + tx + 16 * j;
      if (gj < p.n)
        __stcs(p.dist + gi * p.ldd + gj,
               kMetric == UX_BRAYCURTIS ? acc[i][j] / den[i % kD][j % kD] : ux_fin<kMetric>(acc[i][j], p.inv_p));
    }
  }
}

}  // namespace b2d
