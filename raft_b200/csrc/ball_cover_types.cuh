// The ball cover's index and the walks' block shape, which its kernels (ball_cover.cuh) and the host code of the files
// that build an index (host.cuh) share.
#pragma once

namespace b2d {

constexpr int kBcWarps = 8;   // items (queries or index positions) per block of the walks, one warp each

// The index, one caller-owned buffer (its regions: bc_layout in ball_cover.cu).  Positions are the rows sorted by
// (ball, s to the ball's landmark, row); rows with a non-finite coordinate follow the last ball.
struct BcIndex {
  float* lm;    // [nl][d] landmark coordinates
  float* rhi;   // [nl] bc_dhi of the ball's largest member s: an upper bound of its true radius; -1: empty ball
  int* off;     // [nl + 2] ball b holds positions [off[b], off[b + 1]); [off[nl], off[nl + 1] = n) the non-finite rows
  float* pts;   // [n][d] coordinates by position
  int* ids;     // [n] the caller's row at each position
  float* rl;    // [n] s(landmark, row), ascending inside each ball (0 for the non-finite rows)
};

}  // namespace b2d
