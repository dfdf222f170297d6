// Thin inline-PTX wrappers for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA
// with shared-memory operand descriptors), fences.  No CUTLASS dependency: the bit layout of the
// wgmma shared-memory matrix descriptor is restated here from the PTX ISA.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace b2d {
namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p)
{
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one()
{
  uint32_t pred = 0;
  asm volatile(
    "{\n\t.reg .pred P;\n\t"
    "elect.sync _|P, 0xffffffff;\n\t"
    "selp.b32 %0, 1, 0, P;\n\t}\n"
    : "=r"(pred));
  return pred != 0;
}

// ------------------------------------------------------------------ mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count)
{
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init()
{
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes)
{
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar)
{
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity)
{
  uint32_t ok;
  asm volatile(
    "{\n\t.reg .pred P;\n\t"
    "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
    "selp.b32 %0, 1, 0, P;\n\t}\n"
    : "=r"(ok)
    : "r"(smem_u32(bar)), "r"(parity)
    : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug traps (context error, process fails loudly) instead of hanging
// the GPU.  The bound is ~seconds of spinning, far above any legitimate wait.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity)
{
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 26)) { __trap(); }
  }
}

// ------------------------------------------------------------------ fences
__device__ __forceinline__ void fence_proxy_async_smem()
{
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

__device__ __forceinline__ void bar_sync(uint32_t id, uint32_t nthreads)
{
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ void bar_arrive(uint32_t id, uint32_t nthreads)
{
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ------------------------------------------------------------------ TMA
__device__ __forceinline__ void prefetch_tmap(const void* tmap)
{
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
// 2-D tiled load global -> shared, completion on an mbarrier (complete_tx::bytes), with an L2
// cache-policy hint.
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const void* tmap, uint64_t* bar,
                                            int32_t c0, int32_t c1, uint64_t policy)
{
  asm volatile(
    "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
    " [%0], [%1, {%3, %4}], [%2], %5;"
    :
    : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0),
      "r"(c1), "l"(policy)
    : "memory");
}
// 2-D tiled store shared -> global (bulk async-group completion); OOB parts of the box are clipped.
// smem_src is a shared-window address (smem_u32).
__device__ __forceinline__ void tma_store_2d(const void* tmap, uint32_t smem_src, int32_t c0, int32_t c1, uint64_t policy)
{
  asm volatile(
    "cp.async.bulk.tensor.2d.global.shared::cta.bulk_group.L2::cache_hint [%0, {%2, %3}], [%1], %4;"
    :
    : "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_src), "r"(c0), "r"(c1), "l"(policy)
    : "memory");
}
// the same through a 3-D tensor map (coordinates innermost first)
__device__ __forceinline__ void tma_store_3d(const void* tmap, uint32_t smem_src, int32_t c0, int32_t c1, int32_t c2,
                                             uint64_t policy)
{
  asm volatile(
    "cp.async.bulk.tensor.3d.global.shared::cta.bulk_group.L2::cache_hint [%0, {%2, %3, %4}], [%1], %5;"
    :
    : "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_src), "r"(c0), "r"(c1), "r"(c2), "l"(policy)
    : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// all but the N most recent committed bulk-store groups of this thread have finished READING shared memory
template <int N>
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
// every committed bulk-store group of this thread has completed (writes included)
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

__device__ __forceinline__ uint64_t policy_evict_last()
{
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t policy_evict_normal()
{
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t policy_evict_first()
{
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}

// ------------------------------------------------------------------ wgmma
// A warpgroup (4 consecutive warps, 128 threads) issues one wgmma together; the accumulator lives in
// the registers of its threads.  Fragment of an m64nN accumulator (the m16n8 layout per warp,
// repeated along columns): warp w of the warpgroup, lane l, for i in [0, N/8):
//   d[4i+0], d[4i+1] = row 16w + l/4,     columns 8i + 2(l%4) + {0,1}
//   d[4i+2], d[4i+3] = row 16w + l/4 + 8, same columns
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of the accumulator registers across wgmma issue / wait
__device__ __forceinline__ void fence_regs(float (&d)[64])
{
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x 128] (+)= A[64 x 16] * B[128 x 16]^T, fp16 operands from shared memory (both K-major), fp32
// accumulate in registers.  accumulate == 0: D = A * B.
__device__ __forceinline__ void wgmma_m64n128k16_f16(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate)
{
  asm volatile(
    "{\n\t.reg .pred p;\n\t"
    "setp.ne.b32 p, %66, 0;\n\t"
    "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
    "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}\n"
    : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
      "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
      "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
      "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
      "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
      "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
      "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
      "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
    : "l"(desc_a), "l"(desc_b), "r"(accumulate)
    : "memory");
}

// ------------------------------------------------------------------ descriptors
// wgmma shared-memory matrix descriptor, K-major operand, rows of 128 bytes, SWIZZLE_128B:
//   bits [0,14)  start address >> 4
//   bits [16,30) leading byte offset >> 4 (unused for swizzled K-major; 1)
//   bits [32,46) stride byte offset >> 4 (distance between 8-row groups = 1024 B -> 64)
//   bits [62,64) layout type = 1 (SWIZZLE_128B)
// A k-step of 16 fp16 inside the swizzled row advances the start address by 32 bytes (+2).
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr)
{
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// Same, SWIZZLE_64B with rows of 64 bytes (8-row groups of 512 B; layout type 2): used where only
// half of a packed k-block is staged.
__device__ __forceinline__ uint64_t gmma_desc_sw64(uint32_t smem_addr)
{
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(512 >> 4) << 32;
  d |= static_cast<uint64_t>(2) << 62;
  return d;
}

// ------------------------------------------------------------------ misc
__device__ __forceinline__ void st_shared_v2(uint32_t addr, float a, float b)
{
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ uint4 ld_shared_v4(uint32_t addr)
{
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void st_shared_u16(uint32_t addr, uint32_t v)
{
  asm volatile("st.shared.u16 [%0], %1;" ::"r"(addr), "h"(static_cast<unsigned short>(v)) : "memory");
}
__device__ __forceinline__ void st_global_cs_v2(float* p, float a, float b)
{
  asm volatile("st.global.cs.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ void st_global_cs(float* p, float v)
{
  asm volatile("st.global.cs.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}

}  // namespace ptx
}  // namespace b2d
