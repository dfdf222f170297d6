// Exact single linkage for 2-D and 3-D points (single_linkage.cu, the one file that includes this header next to
// single_linkage.cuh): the Euclidean minimum spanning tree by Borůvka over the random ball cover (DESIGN.md K21).
//
// The vertices are the index positions (ball_cover_types.cuh): colour, parent and the per-component slots are indexed
// by position, so the walk reads the colours of a ball's members coalesced.  Pair (i, j) of caller rows weighs
// s(i, j) = bc_s (bitwise symmetric), and edges are ordered by (s, min(i, j), max(i, j)): a strict total order, so the
// tree is unique.  Its 91 bits do not fit one word, so a component's minimum takes two atomics:
//   best1[c] = min of key1 = key_pack(s, min row) over the candidates of c's rows (one 64-bit atomicMin per row), then
//   best2[c] = min of the max row over the rows whose candidate has key1 == best1[c].
// (best1, best2) names the chosen edge itself: its weight and both rows.
// One Borůvka round (every kernel returns at once when the run word is 0):
//   sl_round_begin_kernel   best1 <- KEY_EMPTY, jump flags <- 0
//   slr_ball_kernel         per ball: its single colour, or -1 when its members have several
//   slr_walk_kernel         per position: the nearest row of another colour; best2 <- INT_MAX
//   slr_tie_kernel          the rows whose candidate holds best1 of their colour: atomicMin of the max row
//   slr_hook_kernel         every component hooks to the other side of its edge (a mutual pair: the smaller id stays
//                           root) and appends the edge once
//   sl_jump_kernel, sl_relabel_kernel, sl_round_end_kernel   as in the edge-list rounds (single_linkage.cuh)
#pragma once
#include <climits>

#include "ball_cover.cuh"
#include "single_linkage.cuh"

namespace b2d {

// pos[ids[t]] = t: the position of every caller row
__global__ void slr_pos_kernel(const int* ids, int64_t n, int* pos)
{
  const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t < n) pos[ids[t]] = static_cast<int>(t);
}

// bcol[b] = the colour of every member of ball b, or -1 (several colours, or an empty ball); one warp per ball
__global__ void slr_ball_kernel(const SlCtrl* ctrl, const int* off, const int* colour, int nl, int* bcol)
{
  if (!sl_running(ctrl)) return;
  const int lane = threadIdx.x & 31;
  const int b    = blockIdx.x * kBcWarps + (threadIdx.x >> 5);
  if (b >= nl) return;
  const int lo = off[b], hi = off[b + 1];
  int mn = INT_MAX, mx = INT_MIN;
  for (int p = lo + lane; p < hi; p += 32) {
    const int c = colour[p];
    mn          = min(mn, c);
    mx          = max(mx, c);
  }
  mn = __reduce_min_sync(0xffffffffu, mn);
  mx = __reduce_max_sync(0xffffffffu, mx);
  if (lane == 0) bcol[b] = hi > lo && mn == mx ? mn : -1;
}

// (a1, a2) before (b1, b2) in the edge order
__device__ __forceinline__ bool slr_before(long long a1, int a2, long long b1, int b2) { return a1 < b1 || (a1 == b1 && a2 < b2); }

// The cross-component 1-NN walker of one query row of a warp: its best edge (b1, b2) so far, the component slot's value
// as last read (seen) and the distance bound dmax they give.  A ball of the query's colour is not admitted.
// Mr (HDBSCAN, hdbscan_rbc.cuh): pair (i, j) weighs w = max(core_i, core_j, s) instead of s, and the walk prunes by the
// core distances too (core: by position, cmin: the smallest core of every ball, cq: the query's).  Each prune is strict
// against the bound wb, so a pair at the bound's weight is still compared.  Since w >= s, the window and ball tests on s
// stay valid at bc_dhi(wb).
// Pred (HDBSCAN's approximate_predict, hdbscan_rbc.cuh; with Mr): the query is not a row of the index, so there is no
// colour and no component slot; row j is keyed (w, s, j), b1 = key_pack(w, bits of s) and b2 = j.
template <int D, bool Mr = false, bool Pred = false>
struct SlrWalk {
  const BcIndex& ix;
  const int* colour;
  const int* bcol;
  long long* slot;   // best1 of the query's colour
  float q[D];
  int row, col, lane;
  long long b1 = KEY_EMPTY, seen = KEY_EMPTY;
  int b2     = INT_MAX;
  float dmax = BC_INF;
  const float* core = nullptr;
  const float* cmin = nullptr;
  float cq = 0.f;
  float wb = BC_INF;   // Mr: the bound itself

  __device__ __forceinline__ SlrWalk(const BcIndex& i, const int* c, const int* bc, long long* s)
      : ix(i), colour(c), bcol(bc), slot(s) {}

  // Mr: a ball whose every pair weighs more than the bound (max(cq, cmin) > wb) is not admitted either
  __device__ __forceinline__ bool admit(int j) const
  {
    if constexpr (Pred) return !(fmaxf(cq, cmin[j]) > wb);
    if constexpr (Mr) return bcol[j] != col && !(fmaxf(cq, cmin[j]) > wb);
    return bcol[j] != col;
  }

  // the bound is the smaller of the two weights: a pair proven farther than bc_dhi(bound) has s > bound, so w > bound
  __device__ __forceinline__ void bound()
  {
    const float b = fminf(key_bound(b1), key_bound(seen));
    if constexpr (Mr) wb = b;
    dmax = bc_dhi(b);
  }

  // the positions [lo, hi) of one ball at s = sq from the query, members of the query's colour skipped.  Mr: true (the
  // walk ends) once the query's own core distance exceeds the bound on some lane, whose read of the slot bounds the
  // component's minimum: every pair of the row then orders after it
  __device__ __forceinline__ bool scan(int lo, int hi, float sq)
  {
    if constexpr (!Pred) seen = min(seen, *reinterpret_cast<volatile long long*>(slot));
    bound();
    if constexpr (Mr)
      if (__any_sync(0xffffffffu, cq > wb)) return true;
    float wlo, whi;
    bc_window(sq, dmax, &wlo, &whi);
    for (int p = bc_search(ix.rl, lo, hi, wlo, false); p < hi; p += 32) {
      const int i    = p + lane;
      const float r  = i < hi ? ix.rl[i] : BC_INF;
      const bool out = i < hi && r > whi;
      long long k1   = KEY_EMPTY;
      int k2         = INT_MAX;
      if (i < hi && !out && r >= wlo && (Pred || colour[i] != col)) {
        if constexpr (Pred) {
          const float cp = core[i];
          if (!(cp > wb)) {
            const float s = bc_s<D>(q, ix.pts + static_cast<int64_t>(i) * D);
            k1            = key_pack(fmaxf(fmaxf(cq, cp), s), __float_as_int(s));
            k2            = ix.ids[i];
          }
        } else if constexpr (Mr) {
          const float cp = core[i];   // a member above the bound is not measured
          if (!(cp > wb)) {
            const float s = bc_s<D>(q, ix.pts + static_cast<int64_t>(i) * D);
            if (s == s) {
              const int j = ix.ids[i];
              k1          = key_pack(fmaxf(fmaxf(cq, cp), s), min(row, j));
              k2          = max(row, j);
            }
          }
        } else {
          const float s = bc_s<D>(q, ix.pts + static_cast<int64_t>(i) * D);
          if (s == s) {
            const int j = ix.ids[i];
            k1          = key_pack(s, min(row, j));
            k2          = max(row, j);
          }
        }
      }
      if (__any_sync(0xffffffffu, slr_before(k1, k2, b1, b2))) {
        for (int o = 16; o > 0; o >>= 1) {
          const long long o1 = __shfl_xor_sync(0xffffffffu, k1, o);
          const int o2       = __shfl_xor_sync(0xffffffffu, k2, o);
          if (slr_before(o1, o2, k1, k2)) { k1 = o1; k2 = o2; }
        }
        b1 = k1;
        b2 = k2;
        bound();
        bc_window(sq, dmax, &wlo, &whi);
      }
      if (__any_sync(0xffffffffu, out)) break;
    }
    // an improvement is published at once, so that the component's other rows prune with it
    if constexpr (!Pred) {
      if (lane == 0 && b1 < seen) atomicMin(slot, b1);
      seen = min(seen, b1);
    }
    return false;
  }
};

// One warp per position t: the first edge in the order from t's row to a row of another colour, into cand1[t] /
// cand2[t] and (atomicMin) best1[colour].  bc_walk with the nearest ball first and SlrWalk: bc_knn_kernel's walk with
// k = 1 and a colour filter.  The bound also comes from the component's best1, read while the walk runs: it only
// decreases, so every value read bounds the component's minimum.  Only the K19 margin helpers prune, and only what is
// proven farther than bc_dhi(bound): such a pair has s > bound and orders strictly after it, so every pair at the
// bound's s (the ties the rows break) is still compared.
template <int D>
__global__ void __launch_bounds__(kBcWarps * 32) slr_walk_kernel(const SlCtrl* ctrl, BcIndex ix, int n, int nl,
                                                                 const int* colour, const int* bcol, long long* best1,
                                                                 int* best2, long long* cand1, int* cand2, int smem)
{
  if (!sl_running(ctrl)) return;
  const float *lm, *rhi;
  bc_stage<D>(ix, nl, smem, &lm, &rhi);
  const int t = blockIdx.x * kBcWarps + (threadIdx.x >> 5);
  if (t >= n) return;
  const int col = colour[t];
  SlrWalk<D> w(ix, colour, bcol, best1 + col);
  w.lane = threadIdx.x & 31;
  w.row  = ix.ids[t];
  w.col  = col;
  if (bc_query<D>(ix.pts + static_cast<int64_t>(t) * D, w.q)) bc_walk<D, true>(ix, n, nl, lm, rhi, w.q, w.lane, w);
  if (w.lane == 0) {
    cand1[t] = w.b1;
    cand2[t] = w.b2;
    best2[t] = INT_MAX;
  }
}

// the second half of the component minimum: among the rows whose candidate holds best1 of their colour, the smallest
// max row
__global__ void slr_tie_kernel(const SlCtrl* ctrl, const int* colour, const long long* cand1, const int* cand2,
                               const long long* best1, int* best2, int64_t n)
{
  if (!sl_running(ctrl)) return;
  const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const long long k = cand1[t];
  const int c       = colour[t];
  if (k != KEY_EMPTY && k == best1[c]) atomicMin(&best2[c], cand2[t]);
}

// sl_hook_kernel for edges named by (best1, best2): the rows key_index(best1) and best2, their positions by pos.  The
// edge is appended as its two words.
__global__ void slr_hook_kernel(SlCtrl* ctrl, const int* colour, const int* pos, const long long* best1, const int* best2,
                                int* parent, long long* mst1, int* mst2, int64_t n)
{
  if (!sl_running(ctrl)) return;
  const int64_t v = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (v >= n || colour[v] != v) return;
  const long long b = best1[v];
  if (b == KEY_EMPTY) { parent[v] = static_cast<int>(v); return; }
  const int b2      = best2[v];
  const int ca      = colour[pos[key_index(b)]];
  const int other   = ca == v ? colour[pos[b2]] : ca;
  const bool mutual = best1[other] == b && best2[other] == b2;
  parent[v]         = (mutual && v < other) ? static_cast<int>(v) : other;
  if (!mutual || v < other) {
    const unsigned e = atomicAdd(&ctrl->n_mst, 1u);
    mst1[e]          = b;
    mst2[e]          = b2;
  }
}

// tree edge t of the sorted edges (key1, max row): (min row, max row, s or its correctly rounded root); a slot the
// rounds did not fill (a non-finite x) gets (-1, -1, NaN)
__global__ void slr_emit_kernel(const SlCtrl* ctrl, const long long* key1, const int* maxrow, int64_t cap, int root,
                                int* out_src, int* out_dst, float* out_w)
{
  const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= cap) return;
  if (t >= static_cast<int64_t>(ctrl->n_mst)) {
    out_src[t] = -1;
    out_dst[t] = -1;
    out_w[t]   = __int_as_float(0x7fc00000);
    return;
  }
  const long long k = key1[t];
  const float s     = key_dist(k);
  out_src[t]        = static_cast<int>(key_index(k));
  out_dst[t]        = maxrow[t];
  out_w[t]          = root ? __fsqrt_rn(s) : s;
}

}  // namespace b2d
