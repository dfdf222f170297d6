// Which kernels a dense pairwise call runs, as host arithmetic on the shape, the pitches and the pointer alignments.
// The launch code (tc_store and b2d_pairwise_distance in pairwise.cu, launch_tc in tensor_launch.cu) follows these functions and
// b2d_debug_pairwise_plan reports them, so a test can name the path a shape takes without a device.
#pragma once
#include <cstdint>
#include "tc_params.cuh"

namespace b2d {

// k-blocks (32 columns) of the packed operands
inline int tc_k_blocks(int64_t k) { return static_cast<int>((k + 31) / 32); }

// the tensor kernel's instantiation: the y block stays resident in shared memory, or both operands stream
inline bool tc_resident(int nkb) { return nkb <= TC_MAX_RES_KB; }

constexpr int TC_MAX_SINGLE_KB = 10;   // k <= 320: one pass over K
constexpr int TC_CHUNK_KB      = 8;    // k > 320: K chunks of 256 columns, accumulated in dist

// One EPI_STORE result [ma][na] with pitch ldd at address dist.
struct TcStorePlan {
  int nkb_total;
  int chunked;     // K-chunked accumulation: one launch per TC_CHUNK_KB k-blocks, read-modify-write of dist
  int launches;
  int tma_store;   // the tiles leave through shared-memory staging and TMA stores, else from registers ...
  int vec2;        // ... as 8-byte vectors on the tiles that lie wholly inside dist (tc_dist_vec2), else scalars
};

// One launch of the plan: k-blocks [kb0, kb0 + nkb) in TcParams::acc_mode, on the resident or the streaming kernel.
struct TcStoreLaunch {
  int kb0, nkb, acc_mode, resident;
};

inline TcStorePlan tc_store_plan(int post, int64_t ma, int64_t na, int64_t k, uintptr_t dist, int64_t ldd)
{
  TcStorePlan pl;
  pl.nkb_total = tc_k_blocks(k);
  // k > 320: accumulate K in chunks, each added to dist with a round-to-nearest fp32 add -- bounds the truncation
  // bias of long MMA chains (DESIGN.md, numerics).  The ratio metrics need the whole inner product at once.
  pl.chunked  = (pl.nkb_total > TC_MAX_SINGLE_KB && !tc_post_ratio(post)) ? 1 : 0;
  pl.launches = pl.chunked ? (pl.nkb_total + TC_CHUNK_KB - 1) / TC_CHUNK_KB : 1;
  // The result leaves through shared-memory staging and TMA stores wherever TMA can address dist: 16-byte aligned
  // base and pitch, row and column coordinates within int32 (the store takes 32-bit coordinates), and rows that end
  // on a 16-byte boundary.  The last condition is from observation: on an H100, with n = 150 and ldd = 160, the
  // box stores also wrote columns 150 and 151, i.e. the partial 16 bytes at the end of each row, into the caller's
  // padding (tests/test_pairwise_gpu.py::test_padded_leading_dimensions_and_out_param).  Otherwise, and for the
  // read-modify-write K chunks, the epilogue stores from registers.
  pl.tma_store = (!pl.chunked && dist % 16 == 0 && ldd % 4 == 0 && na % 4 == 0 && ma <= 0x7fffffffll &&
                  na <= 0x7fffffffll) ? 1 : 0;
  pl.vec2 = (!pl.tma_store && tc_dist_vec2(dist, ldd)) ? 1 : 0;
  return pl;
}

inline TcStoreLaunch tc_store_launch(const TcStorePlan& pl, int i)
{
  TcStoreLaunch l;
  if (!pl.chunked) {
    l.kb0 = 0; l.nkb = pl.nkb_total; l.acc_mode = 0;
  } else {
    l.kb0      = i * TC_CHUNK_KB;
    l.nkb      = pl.nkb_total - l.kb0 < TC_CHUNK_KB ? pl.nkb_total - l.kb0 : TC_CHUNK_KB;
    l.acc_mode = i == 0 ? 1 : (i == pl.launches - 1 ? 3 : 2);   // raw store, +=, += and the post-processing
  }
  l.resident = tc_resident(l.nkb) ? 1 : 0;
  return l;
}

// unexpanded fp32 kernels: 16-byte loads of an operand with element strides (rs, cs) at address base need a unit
// column stride, k % 4 == 0 and 16-byte aligned rows.  Both operands vectorisable: the TMA-fed kernel; otherwise the
// SIMT kernel loads each operand its own way.
struct UxPlan {
  int vec_x, vec_y, tma;
};
inline UxPlan ux_plan(int64_t xrs, int64_t xcs, uintptr_t x, int64_t yrs, int64_t ycs, uintptr_t y, int64_t k)
{
  UxPlan pl;
  pl.vec_x = (xcs == 1 && xrs % 4 == 0 && k % 4 == 0 && x % 16 == 0) ? 1 : 0;
  pl.vec_y = (ycs == 1 && yrs % 4 == 0 && k % 4 == 0 && y % 16 == 0) ? 1 : 0;
  pl.tma   = pl.vec_x && pl.vec_y;
  return pl;
}

}  // namespace b2d
