// K3b: coarse screening pass of the screened fusedL2NN (sm_90a, wgmma).
//
// fused_nn_keys (nearest.cu) first runs the exact arg-min kernel on every S-th 256-row block of y, which
// leaves each x row with an upper bound U_i of its minimum.  This kernel visits the other blocks with
// ONE tensor product per k-block (hi*hi only: a third of the exact kernel's MMA work, half of its
// operand bytes) and computes, per pair, a rigorous LOWER bound of the fp32-grade distance
//     L_ij = acc_ij * c + |y_j|^2 (1 - 2^-21) - margin_i,
//     margin_i = f (|x_i| YL + |xl_i| Y + 3 |xl_i| YL) + f 0.05 * 2^-10 |x_i| Y      (Y, YL: block maxima of |y_j|, |yl_j|)
// where xl = x - (its hi part) is MEASURED per row by prep.cuh and f = 2 (L2) or 1 (cosine / correlation: rows are
// unit vectors after prep, d = 1 + acc * c): Cauchy-Schwarz on the three dropped products; the last term and the
// 2^-21 |y|^2 cover the fp32 rounding of the accumulation and of the epilogue.  Only pairs with L_ij <= U_i can hold
// the minimum: they go to a candidate list that nn_exact_kernel re-measures straight from the fp32 inputs.  The margin
// is a per-row constant inside a y block, so it moves into the row's threshold.  The element loop does not even form
// L_ij: it bounds the thread's 8 values of a 32-column group G by  c max acc_ij + min_{j in G} |y_j|^2 (1 - 2^-21)
// (c < 0), and only a group that reaches the threshold is looked at column by column.  The database chunk is packed
// in the order of |y_j|^2 (nearest.cu), which makes the group bound as good as the per-column one and the per-block
// margin (max_j' |y_j'|) local; `col_map` translates a packed position back to the caller's row where an index
// leaves the kernel.
//
// Every coarse value is also an UPPER bound of a real pair's distance (value + margin), so a row's
// bound tightens (atomic min on aux[i].x) whenever one of its candidates is found, which is what lets
// the exact pass sample only every 32nd block.
//
//   operands   hi halves only: TMA boxes of 32 fp16 (64 B, SWIZZLE_64B) out of the packed [hi32|lo32] k-blocks;
//              a stage is one whole x tile (nkb x 8 KB), one mbarrier round trip per TILE; the y block
//              (nkb x 16 KB) is resident per item
//   warpgroup 0      TMA producer (warp 0)
//   warpgroups 1-2   consumers: warpgroup c owns rows [64c, 64c+64) of every x tile and all 256 columns (two
//                    wgmma.m64n128k16 accumulators), releases the x stage as soon as its MMAs have finished and
//                    screens from the registers; a warp with a hit takes the atomics (list append, bound update)
#pragma once
#include "expanded_tc.cuh"

namespace b2d {

constexpr int SC_A_KB_BYTES   = TC_BM * 64;  // one k-block of an x tile, hi halves: 128 rows x 64 B
constexpr int SC_B_KB_BYTES   = TC_BN * 64;  // one k-block of the y block:          256 rows x 64 B
constexpr int SC_MAX_KB       = 4;           // k <= 128
constexpr int SC_MAX_STAGES   = 8;
constexpr int SC_BLK          = 64;          // candidate-list slots a warp reserves at a time
constexpr int SC_THREADS      = 384;
constexpr size_t SC_A_RING    = 128 * 1024;
constexpr size_t SC_SMEM_OPERANDS = (size_t)SC_MAX_KB * SC_B_KB_BYTES + SC_A_RING;  // 192 KB
constexpr size_t SC_SMEM_BYTES    = SC_SMEM_OPERANDS + TC_BN * 4 + 96 + 256;
static_assert(SC_SMEM_BYTES <= 232448, "exceeds the 227 KB per-CTA limit");

struct ScreenParams {
  int64_t m, n;
  int nkb;                // k-blocks of 32 source columns (<= SC_MAX_KB)
  int n_stages;           // x-tile stages in the ring (host: min(SC_MAX_STAGES, SC_A_RING / (nkb * 8 KB)))
  int tiles_m, tiles_sel; // ceil(m/128); y blocks this launch visits
  int sel_s, sel_lo, sel_hi;  // as TcParams
  int chunk, chunks_m;    // m-tiles per work item
  int64_t n_items;
  const float* yt;        // [n] |y_j|^2
  const float* coef;      // [1] -2 * 2^-(ex+ey)
  const float* xsc;       // [m] per-row scale of x (prep.cuh; 1 unless the row took its own exponent)
  const unsigned* nonuni; // [2] some row of x / y has its own exponent (y: fused_nn_keys sends everything to the exact kernel)
  const float* ylo;       // [n] |y_j - hi part| (prep.cuh lvec)
  float4* aux;            // [m] (U_i - |x_i|^2 rounded up, |x_i|, |x_i - hi part|, -); the bound tightens as candidates are found
  int2* cand;             // candidate (row, packed column position) list; (-1, -1) = unused slot ...
  unsigned* cand_cnt;     // ... its slot counter ([0]; [6] counts the candidates themselves) ...
  unsigned cand_cap;      // ... capacity ...
  unsigned* overflow;     // ... and overflow flag (then the exact pass re-runs)
  const unsigned* run_flag;  // non-null: the whole launch is a no-op unless *run_flag != 0
  const int* col_map;     // non-null: packed column j is source row col_map[j] (norm-sorted chunk)
  int unit_norm;          // cosine family: rows are unit vectors, d = 1 + acc * c (c without the factor 2)
};

__global__ void __launch_bounds__(SC_THREADS, 1)
screen_tc_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                 const ScreenParams p)
{
  if (p.run_flag != nullptr && __ldg(p.run_flag) == 0u) return;  // conditional launch (no host round trip)
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((ptx::smem_u32(smem) & 1023u) != 0u) __trap();
  uint8_t* b_base  = smem;
  uint8_t* a_base  = smem + SC_MAX_KB * SC_B_KB_BYTES;
  float* col_tb    = reinterpret_cast<float*>(smem + SC_SMEM_OPERANDS);  // [256] |y_j|^2 (1 - 2^-21), +inf beyond n
  float* col_ny    = col_tb + TC_BN;                                     // [8] per-warp maxima of |y_j|
  float* col_gm    = col_ny + 8;                                         // [8] per 32-column group: min of col_tb
  float* col_nl    = col_gm + 8;                                         // [8] per-warp maxima of |y_j - hi part|
  uint64_t* bars   = reinterpret_cast<uint64_t*>(col_nl + 8);
  uint64_t* afull  = bars;                      // [SC_MAX_STAGES]
  uint64_t* aempty = bars + SC_MAX_STAGES;      // [SC_MAX_STAGES]
  uint64_t* bfull  = bars + 2 * SC_MAX_STAGES;  // [1]
  uint64_t* bempty = bfull + 1;                 // [1]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    // empty barriers: one arrival per consumer warpgroup
    for (int i = 0; i < SC_MAX_STAGES; ++i) { ptx::mbar_init(&afull[i], 1); ptx::mbar_init(&aempty[i], 2); }
    ptx::mbar_init(bfull, 1);
    ptx::mbar_init(bempty, 2);
    ptx::fence_mbar_init();
    ptx::prefetch_tmap(&tmap_a);
    ptx::prefetch_tmap(&tmap_b);
  }
  __syncthreads();

  const int nkb              = p.nkb;
  const uint32_t stage_bytes = static_cast<uint32_t>(nkb) * SC_A_KB_BYTES;
  const uint32_t n_stages    = static_cast<uint32_t>(p.n_stages);

  if (warp < 4) {
    // ================================ TMA producer =================================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp != 0) return;
    const uint64_t pol = ptx::policy_evict_last();
    uint32_t t_it = 0, it_local = 0;
    for (int64_t item = blockIdx.x; item < p.n_items; item += gridDim.x, ++it_local) {
      const auto [n_blk, mt0, mt1, nh] = tc_item(p, item);
      ptx::mbar_wait(bempty, (it_local & 1) ^ 1);
      if (ptx::elect_one()) {
        ptx::mbar_expect_tx(bfull, static_cast<uint32_t>(nkb) * SC_B_KB_BYTES);
        for (int kb = 0; kb < nkb; ++kb)
          ptx::tma_load_2d(b_base + kb * SC_B_KB_BYTES, &tmap_b, bfull, kb * 64, n_blk * TC_BN, pol);
      }
      __syncwarp();
      for (int mt = mt0; mt < mt1; ++mt, ++t_it) {
        const uint32_t s = t_it % n_stages, ph = (t_it / n_stages) & 1;
        ptx::mbar_wait(&aempty[s], ph ^ 1);
        if (ptx::elect_one()) {
          ptx::mbar_expect_tx(&afull[s], stage_bytes);
          for (int kb = 0; kb < nkb; ++kb)
            ptx::tma_load_2d(a_base + s * stage_bytes + kb * SC_A_KB_BYTES, &tmap_a, &afull[s], kb * 64, mt * TC_BM,
                             pol);
        }
        __syncwarp();
      }
    }
    return;
  }

  // ================================ consumer warpgroups ================================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int wg    = (threadIdx.x >> 7) - 1;  // rows [64 wg, 64 wg + 64) of every x tile
  const int et    = threadIdx.x - 128;       // 0..255
  const bool lead = (threadIdx.x & 127) == 0;
  const int quad  = lane >> 2, tq = lane & 3;
  const float cf0 = __ldg(p.coef);
  const bool xnu  = __ldg(&p.nonuni[0]) != 0u;
  const float4 aux_none = make_float4(__int_as_float(0xff800000), 0.f, 0.f, 0.f);  // rows beyond m: threshold -inf, never taken
  unsigned blk_base = 0;      // this warp's block of candidate-list slots ...
  int blk_used      = SC_BLK; // ... and how many of them are taken (SC_BLK: none reserved yet)
  bool list_full    = false;  // a reservation of this warp came back beyond the list's capacity (sticky, warp-uniform)
  uint32_t t_it = 0, it_local = 0;
  float acc[2][64];           // columns [0, 128) and [128, 256) of the y block
  for (int64_t item = blockIdx.x; item < p.n_items; item += gridDim.x, ++it_local) {
    const auto [n_blk, mt0, mt1, nh] = tc_item(p, item);
    // per-column terms of this y block (shared by every tile of the item)
    ptx::bar_sync(1, 256);
    {
      const int64_t gj = static_cast<int64_t>(n_blk) * TC_BN + et;
      float tv = __int_as_float(0x7f800000), nyv = 0.f, nlv = 0.f;  // +inf: never a candidate
      if (gj < p.n) {
        nlv = __ldg(&p.ylo[gj]);
        if (p.unit_norm) {  // |y_j| = 1, column term 0
          tv  = 0.f;
          nyv = 1.f;
        } else {
          tv  = __ldg(&p.yt[gj]);
          nyv = sqrtf(tv) * (1.f + 1.f / 4194304.f);
          tv  = tv - tv * (1.f / 2097152.f);
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        nyv = fmaxf(nyv, __shfl_xor_sync(0xffffffffu, nyv, o));
        nlv = fmaxf(nlv, __shfl_xor_sync(0xffffffffu, nlv, o));
      }
      float gm = tv;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) gm = fminf(gm, __shfl_xor_sync(0xffffffffu, gm, o));
      if (lane == 0) { col_ny[et >> 5] = nyv; col_nl[et >> 5] = nlv; col_gm[et >> 5] = gm; }
      col_tb[et] = tv;
    }
    ptx::bar_sync(1, 256);
    // What the coarse product leaves out of <x, y>:  xh.yl + xl.yh + xl.yl  with x = xh + xl (hi part + the rest), so by
    // Cauchy-Schwarz at most |x| |yl| + |xl| |y| + 3 |xl| |yl|; the residual norms are MEASURED per row by prep.cuh
    // (about 0.2 * 2^-10 of the row norm for fp16 rounding, against the worst case 2^-11 per element).
    // With Y = max |y_j|, YL = max |yl_j| over the block and f = 2 (L2: d = .. - 2 <x, y>) or 1 (cosine family):
    //   margin_i = |x_i| P + |xl_i| Q,   P = f (YL + 0.05 * 2^-10 Y),   Q = f (Y + 3 YL)
    // (the 0.05 * 2^-10 |x| |y| term covers the fp32 rounding of the accumulation and of the epilogue).
    float y_max = 0.f, yl_max = 0.f;
#pragma unroll
    for (int i = 0; i < TC_BN / 32; ++i) { y_max = fmaxf(y_max, col_ny[i]); yl_max = fmaxf(yl_max, col_nl[i]); }
    const float ff     = p.unit_norm ? 1.f : 2.f;
    const float marg_p = ff * fmaf(y_max, 0.05f / 1024.f, yl_max) * (1.f + 1.f / 1048576.f);
    const float marg_q = ff * fmaf(3.f, yl_max, y_max) * (1.f + 1.f / 1048576.f);
    const float yn_max = y_max * y_max;  // max |y_j|^2 of the block

    ptx::mbar_wait(bfull, it_local & 1);
    for (int mt = mt0; mt < mt1; ++mt, ++t_it) {
      // the two rows this thread owns: row[0] and row[0] + 8
      int64_t row[2];
      float4 aux_c[2];
      float cf[2], margin[2], thr[2];
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        row[j]   = static_cast<int64_t>(mt) * TC_BM + 64 * wg + 16 * (warp & 3) + quad + 8 * j;
        aux_c[j] = row[j] < p.m ? __ldg(&p.aux[row[j]]) : aux_none;
        cf[j]    = (xnu && row[j] < p.m) ? cf0 * __ldg(&p.xsc[row[j]]) : cf0;  // a row with its own exponent
        // U_i - |x_i|^2 + margin_i, nudged up so that it stays an upper bound
        margin[j] = fmaf(aux_c[j].y, marg_p, aux_c[j].z * marg_q);
        thr[j]    = aux_c[j].x + margin[j];
        thr[j]    = thr[j] + fabsf(thr[j]) * (1.f / 4194304.f);
      }

      const uint32_t s = t_it % n_stages, ph = (t_it / n_stages) & 1;
      ptx::mbar_wait(&afull[s], ph);
      ptx::fence_regs(acc[0]);
      ptx::fence_regs(acc[1]);
      ptx::wgmma_fence();
#pragma unroll
      for (int kb = 0; kb < SC_MAX_KB; ++kb) {
        if (kb < nkb) {
          // descriptor address units are 16 B: k[0,16) of the 64-byte row at +0, k[16,32) at +2
          const uint64_t da = ptx::gmma_desc_sw64(ptx::smem_u32(a_base + s * stage_bytes + kb * SC_A_KB_BYTES) + wg * 64 * 64);
          const uint64_t db = ptx::gmma_desc_sw64(ptx::smem_u32(b_base + kb * SC_B_KB_BYTES));
          const uint64_t db1 = db + ((TC_HN * 64) >> 4);   // rows [128, 256) of the y block
          ptx::wgmma_m64n128k16_f16(acc[0], da, db, kb > 0 ? 1u : 0u);
          ptx::wgmma_m64n128k16_f16(acc[1], da, db1, kb > 0 ? 1u : 0u);
          ptx::wgmma_m64n128k16_f16(acc[0], da + 2, db + 2, 1u);
          ptx::wgmma_m64n128k16_f16(acc[1], da + 2, db1 + 2, 1u);
        }
      }
      ptx::wgmma_commit();
      ptx::wgmma_wait<0>();
      ptx::fence_regs(acc[0]);
      ptx::fence_regs(acc[1]);
      if (lead) {   // the x stage (and, after the item's last tile, the y block) is free again
        ptx::mbar_arrive(&aempty[s]);
        if (mt == mt1 - 1) ptx::mbar_arrive(bempty);
      }

      // per row and 32-column group gp: this thread holds 8 of the group's values, acc[gp >> 2][4i + 2j + e] with
      // i in [4 (gp & 3), 4 (gp & 3) + 4).  c < 0, so  c max acc + min_{j in G} t_j  bounds all 8 from below, and a
      // group holds a value at or below the threshold only if the bound of some thread's 8 values reaches it.
      unsigned hitmask[2] = {0u, 0u};
#pragma unroll
      for (int gp = 0; gp < 8; ++gp) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const float* a = &acc[gp >> 2][16 * (gp & 3) + 2 * j];
          const float mx = fmaxf(max3(max3(a[0], a[1], a[4]), max3(a[5], a[8], a[9]), a[12]), a[13]);
          hitmask[j] |= (fmaf(mx, cf[j], col_gm[gp]) <= thr[j]) ? (1u << gp) : 0u;
        }
      }
      unsigned long long cmask[2] = {0ull, 0ull};  // bit 2i + e: column 8i + 2tq + e of the block goes to the exact pass
      float vmin[2] = {__int_as_float(0x7f800000), __int_as_float(0x7f800000)};
      if (__any_sync(0xffffffffu, (hitmask[0] | hitmask[1]) != 0u)) {
        // rare after the first y blocks: some column of some row of this warp can still hold the minimum
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const float thr_f = fminf(thr[j], 3.0e38f);   // +inf columns (beyond n) never pass, even against an infinite bound
#pragma unroll
          for (int gp = 0; gp < 8; ++gp) {
            if ((hitmask[j] >> gp) & 1u) {
#pragma unroll
              for (int ii = 0; ii < 4; ++ii) {
                const int i = 4 * gp + ii;   // 8-column group of the block, 0..31
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  const float lv = fmaf(acc[i >> 4][4 * (i & 15) + 2 * j + e], cf[j], col_tb[8 * i + 2 * tq + e]);
                  if (lv <= thr_f) {
                    cmask[j] |= 1ull << (2 * i + e);
                    vmin[j] = fminf(vmin[j], lv);
                  }
                }
              }
            }
          }
        }
      }
      // The bound is lowered with a fire-and-forget reduction (no return value), and list slots come out of a private
      // block of SC_BLK entries per warp, reserved with ONE atomicAdd when the previous block is used up (unused entries
      // of a block are marked invalid, nn_exact_kernel skips them); the entry holds the packed POSITION, which
      // nn_exact_kernel translates.
      const int ncand = __popcll(cmask[0]) + __popcll(cmask[1]);
      if (__any_sync(0xffffffffu, ncand != 0)) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          if (cmask[j] != 0ull) {
            // every coarse value is also an UPPER bound of a real pair's distance (value + margin): later
            // tiles of this row, here and on the other SMs, screen against the tighter bound
            float nb = vmin[j] + margin[j];
            nb += (fabsf(nb) + 2.f * (aux_c[j].y * aux_c[j].y + yn_max)) * (1.f / 2097152.f);
            if (nb < aux_c[j].x) {   // float min as integer reductions: non-negative -> signed min, negative -> unsigned max
              if (nb >= 0.f) atomicMin(reinterpret_cast<int*>(&p.aux[row[j]].x), __float_as_int(nb));
              else atomicMax(reinterpret_cast<unsigned*>(&p.aux[row[j]].x), __float_as_uint(nb));
            }
          }
        }
        if (list_full) {
          // (warp-uniform) a reservation of this warp already came back beyond the end of the list: the overflow flag
          // is up, the exact pass will redo these blocks, and the slot counter must not keep growing -- data on which
          // everything is a candidate would otherwise wrap it around and overwrite the incumbents' entries
          if (lane == 0) *p.overflow = 1u;
        } else {
          int incl = ncand;
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
          }
          const int total = __shfl_sync(0xffffffffu, incl, 31);
          if (lane == 0) atomicAdd(p.cand_cnt + 6, static_cast<unsigned>(total));   // real candidates (slots include unused ones)
          unsigned slot;
          if (total > SC_BLK) {  // (more candidates in one warp-tile than a block holds: a reservation of its own)
            unsigned base = 0;
            if (lane == 0) base = atomicAdd(p.cand_cnt, static_cast<unsigned>(total));
            base = __shfl_sync(0xffffffffu, base, 0);
            if (base >= p.cand_cap) list_full = true;
            slot = base + static_cast<unsigned>(incl - ncand);
          } else {
            if (blk_used + total > SC_BLK) {
#pragma unroll 1
              for (int i = blk_used + lane; i < SC_BLK; i += 32)
                if (blk_base + i < p.cand_cap) p.cand[blk_base + i] = make_int2(-1, -1);
              unsigned base = 0;
              if (lane == 0) base = atomicAdd(p.cand_cnt, static_cast<unsigned>(SC_BLK));
              blk_base = __shfl_sync(0xffffffffu, base, 0);
              blk_used = 0;
              if (blk_base >= p.cand_cap) list_full = true;
            }
            slot = blk_base + static_cast<unsigned>(blk_used + incl - ncand);
            blk_used += total;
          }
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            unsigned long long cm = cmask[j];
#pragma unroll 1
            while (cm != 0ull) {
              const int b = __ffsll(static_cast<long long>(cm)) - 1;
              cm &= cm - 1ull;
              const int col = 8 * (b >> 1) + 2 * tq + (b & 1);
              if (slot < p.cand_cap) p.cand[slot] = make_int2(static_cast<int>(row[j]), n_blk * TC_BN + col);
              else *p.overflow = 1u;
              ++slot;
            }
          }
        }
      }
    }
  }
#pragma unroll 1
  for (int i = blk_used + lane; i < SC_BLK; i += 32)   // the unused rest of this warp's last block
    if (blk_base + i < p.cand_cap) p.cand[blk_base + i] = make_int2(-1, -1);
}

}  // namespace b2d
