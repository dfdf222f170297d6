// Parameters, constants and tile schedule of the tensor-core kernels (expanded_tc.cuh, screen_tc.cuh), without kernels:
// the host launch code and the host replays of the schedule (tests/cpp) read them too.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace b2d {

constexpr int TC_BM          = 128;
constexpr int TC_BN          = 256;
constexpr int TC_HN          = 128;          // columns of one wgmma (half of a y block)
constexpr int TC_A_BYTES     = TC_BM * 128;  // one k-block of A: 128 rows x 128 B
constexpr int TC_B_BYTES     = TC_BN * 128;  // one k-block of the resident y block: 256 rows x 128 B
constexpr int TC_BH_BYTES    = TC_HN * 128;  // one k-block of a streamed y half: 128 rows x 128 B
constexpr int TC_MAX_RES_KB  = 4;            // resident-B variant: k <= 128
constexpr int TC_STAGES_RES  = 5;            // A-only stages (16 KB) next to the resident y block
constexpr int TC_STAGES_STR  = 6;            // A + B-half stages (32 KB) when both operands stream
constexpr int TC_STAGES_RES_ST = 4;          // the same with the output staging of EPI_STORE beside them
constexpr int TC_STAGES_STR_ST = 6;
constexpr int TC_MAX_STAGES  = 6;
constexpr int TC_THREADS     = 384;
// EPI_STORE output staging: TMA boxes of 32 rows x 64 fp32 columns, stored through a 3-D view of dist (32 columns x
// column group x row, box {32, TC_D_BOX_GROUPS, TC_D_BOX_ROWS}, SWIZZLE_128B over its 128-byte lines), so that each
// store writes 256 contiguous bytes of every row it touches; a ring of TC_STG_BOXES per consumer warpgroup (DESIGN.md
// section 2 K1: the box shape and the carve against the x stages, measured).  The ring logic of tc_stage_store is
// written for exactly two boxes of this shape.  EPI_EPS stages its 64 x 128-byte adjacency tiles in the same 8 KB slots.
constexpr int TC_D_BOX_GROUPS = 2;
constexpr int TC_D_BOX_COLS   = 32 * TC_D_BOX_GROUPS;
constexpr int TC_D_BOX_ROWS   = 32;
constexpr int TC_D_BOX_BYTES  = TC_D_BOX_COLS * TC_D_BOX_ROWS * 4;
constexpr int TC_STG_BOXES    = 2;

enum TcEpilogue : int { EPI_STORE = 0, EPI_MINLOC = 1, EPI_TOPK = 2, EPI_MINLOC_MASKED = 3, EPI_EPS = 4, EPI_RADIUS = 5,
                         EPI_KDE = 6 };
constexpr int64_t TC_NO_DIAG = INT64_MIN;   // TcParams::diag_off: y is not a row window of x

// EPI_MINLOC_MASKED (masked_nn.cuh): class of one (64-row slab of x, 128-column half of a y block) tile.  Byte
// TcParams::mask_cls[n_blk][mt] holds the four classes of an (x tile, y block) pair, 2 bits each at bit 2 (2 h + s)
// for slab s (= consumer warpgroup) and half h.  A byte of 0 is a tile with nothing to do.
enum MaskClass : int { MASK_NONE = 0, MASK_ALL = 1, MASK_PARTIAL = 2 };
__host__ __device__ __forceinline__ int mask_class_of(unsigned cls_byte, int h, int s) { return (cls_byte >> (2 * (2 * h + s))) & 3; }
// some slab of half h is live: the streaming variant loads the half's stages
__host__ __device__ __forceinline__ bool mask_half_live(unsigned cls_byte, int h) { return ((cls_byte >> (4 * h)) & 15u) != 0u; }

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

enum TcPost : int { POST_NONE = 0, POST_CLAMP = 1, POST_CLAMP_SQRT = 2,
                    POST_JACCARD = 3,  // d = 1 - a / (s - a), a = <x,y>, s = |x|^2 + |y|^2 (0/0 -> 0)
                    POST_DICE    = 4,  // d = 1 - 2 a / s
                    // kernel Gram matrices (gram_post; TcParams::gamma / coef0 / degree):
                    POST_RBF     = 5,  // exp(-gamma d), d the POST_CLAMP distance
                    POST_POLY    = 6,  // (gamma <x,y> + coef0)^degree
                    POST_TANH    = 7 };  // tanh(gamma <x,y> + coef0)

// the ratio metrics: computed from the inner product and the squared norms at once (never K-chunked)
__host__ __device__ constexpr bool tc_post_ratio(int post) { return post == POST_JACCARD || post == POST_DICE; }
// the squared L2 distance, clamped at 0 (with d(i, i) = 0 when x and y alias) before anything else is done with it
__host__ __device__ constexpr bool tc_post_clamps(int post)
{
  return post == POST_CLAMP || post == POST_CLAMP_SQRT || post == POST_RBF;
}
__host__ __device__ constexpr bool tc_post_gram(int post) { return post == POST_RBF || post == POST_POLY || post == POST_TANH; }
// EPI_STORE from registers: dist [.][ldd] takes 8-byte vector accesses at every even column of every row
__host__ __device__ __forceinline__ bool tc_dist_vec2(uintptr_t dist, int64_t ldd) { return ((dist | static_cast<uintptr_t>(ldd * 4)) & 7u) == 0; }

// Construct as TcParams p{}: every member 0 / null except diag_off, so a launch has no self pairs unless it asks for them.
struct TcParams {
  int64_t m, n;
  int nkb;                // k-blocks of 32 source columns
  int tiles_m, tiles_n;   // ceil(m/128), ceil(n/256)
  int tiles_sel;          // y blocks this launch visits (all of them unless sel_s > 1)
  int sel_s, sel_lo, sel_hi;  // sel_s > 1: only the y blocks with sel_lo <= index % sel_s < sel_hi
  int chunk;              // m-tiles per work item
  int chunks_m;           // ceil(tiles_m/chunk)
  int64_t n_items;        // tiles_n * chunks_m
  const float* xt;        // [m] row term t_x[i]
  const float* yt;        // [n] column term t_y[j]
  const float* coef;      // [1] scalar c: d = acc * c + (t_x[i] + t_y[j])  (prep.cuh)
  const unsigned* has_lo; // [1] 0: every operand is exact in fp16 -> the cross-term MMAs are skipped
  const float* xsc;       // [m] per-row scale of x: d = acc * c * xsc[i] * ysc[j] + ...  (1 unless the row took its own
  const float* ysc;       // [n]   exponent in prep.cuh -- rows far below the matrix maximum)
  const unsigned* nonuni; // [2] some row of x / of y has a scale != 1 (y: the per-column factor is applied)
  // EPI_STORE
  float* dist;
  int64_t ldd;
  int tma_store;         // dist goes out through the staging boxes and the dist tensor map (tc_store_plan: aligned, single pass)
  int acc_mode;           // K-chunked accumulation: 0 single pass, 1 first chunk (raw store), 2 middle (+=), 3 last (+=, post)
  // EPI_MINLOC
  long long* keys;        // [m] packed (ordered bits of the distance << 32 | index)
  int64_t idx_offset;
  const int* col_map;     // non-null: column j of the packed y is source row col_map[j] (norm-sorted chunk, nearest.cu)
  const unsigned* run_flag;  // non-null: the whole launch is a no-op unless *run_flag != 0
  // EPI_TOPK (fused brute-force kNN): every pair at or below the row's current k-th best joins the row's list
  const float* knn_thr;   // [m] current k-th best squared distance of the row (+inf until k are known)
  unsigned* knn_cnt;      // [m] fill counter of the row's candidate list
  long long* knn_cand;    // [m][knn_cap] packed (ordered bits of the distance << 32 | index)
  unsigned knn_cap;
  long long* knn_dropmin; // [m] smallest key that did not fit into the row's list this pass (knn_merge_kernel decides whether
                          //     anything that matters was lost; rows where it was are redone by knn_fix_kernel)
  // EPI_MINLOC_MASKED (masked_nn.cuh): only pairs whose row of x is adjacent to the group of the row of y are candidates
  const uint8_t* mask_cls;    // [tiles_n][tiles_m] tile classes (MaskClass, see mask_class_of)
  const int* mask_grp;        // [n] group of every row of y (-1: in no group)
  const unsigned* mask_bits;  // [ceil(m/32)][mask_groups] bit i % 32 of word (i / 32, g): row i of x is adjacent to group g
  int64_t mask_groups;
  // EPI_EPS (epsilon neighbourhood): adj[i][j] = (d(i, j) <= eps) with d the EPI_STORE / POST_CLAMP distance; vd[j] += the
  // number of adjacent rows of column j, vd[n] += the total.  tma_store: adj leaves through the staging boxes
  uint8_t* adj;           // [m][ld_adj] 0 / 1 bytes (null: count only)
  int64_t ld_adj;
  void* vd;               // [n + 1] uint32 counts, or uint64 when vd64 (null: adjacency only)
  int vd64;
  float eps;              // the squared radius
  // EPI_STORE, EPI_EPS, EPI_RADIUS with a clamping post (tc_finish): row j of y is row j + diag_off of x (the same memory),
  // and d = 0 there exactly, which the expanded form alone does not give (reference: CHANGELOG.md:1057,1213).  0: x is y
  int64_t diag_off = TC_NO_DIAG;
  // EPI_STORE with POST_RBF / POST_POLY / POST_TANH (gram_post): the kernel parameters, applied to the final value only
  float gamma;
  float coef0;
  int degree;
  // EPI_RADIUS (radius_neighbors, radius.cu): the pairs with d(i, j) <= eps, d the EPI_STORE distance of post kPost (diag_off
  // as there).  Count mode: knn_cnt[i] += the row's pairs.  Fill mode: knn_cnt[i] is the row's fill counter and every pair
  // is written as key_pack(d, j) to knn_cand[rad_indptr[i] + slot], a slot at or past min(rad_indptr[i + 1], rad_nnz) dropped
  const long long* rad_indptr;   // [m + 1] (fill mode)
  long long rad_nnz;
  int rad_fill;                  // 0: count, 1: fill
  // EPI_KDE (kernel_density, kde.cu): per row i and 128-column half g of the launch, kde_part[g * kde_ld + i] = (M, S)
  // over the half's columns j < n, with d the EPI_STORE / POST_CLAMP distance (diag_off as there) and c_j = kde_colw[j]:
  //   gaussian, exponential (log-sum-exp, base 2): u_j = c_j - s d^2 resp. c_j - s sqrt(d^2), c_j = log2 w_j; M = max u_j,
  //     S = sum 2^(u_j - M) (M = -inf: S = sum 2^u_j)
  //   tophat, epanechnikov, linear, cosine (the pairs with d^2 < kde_h2 only): M = 0, S = sum c_j K_j, c_j = w_j
  int kde_kernel;                // B2D_KDE_*
  float kde_s;                   // the kernel's fp32 scale factor (kde_row32)
  float kde_h2;                  // fp32(h^2): the support d^2 < kde_h2 of the compact kernels
  float kde_pad;                 // c_j of the columns at or past n: -inf (log-sum-exp) or 0
  const float* kde_colw;         // [n]
  float2* kde_part;              // [halves][kde_ld]
  int64_t kde_ld;
};

constexpr size_t TC_SMEM_OPERANDS = (size_t)TC_MAX_RES_KB * TC_B_BYTES + (size_t)TC_STAGES_RES * TC_A_BYTES;  // 208 KB
static_assert((size_t)TC_STAGES_STR * (TC_A_BYTES + TC_BH_BYTES) <= TC_SMEM_OPERANDS, "streaming carve fits");

// Shared-memory carve of one instantiation: [resident y block][x (+ y half) stages][output staging][t_y][barriers].
// The arg-min / top-k epilogues store nothing and keep 208 KB of operands; EPI_STORE trades one x stage for 32 KB of
// output staging (the streaming variant fits it beside all of its stages).
// x rings: streaming, one ring of `stages` stages that both consumer warpgroups read.  Resident, one ring of `stages`
// 64-row k-blocks (8 KB) per consumer warpgroup, laid out in the same bytes: slot s of ring w is the 8 KB at w * 8 KB of
// the 16 KB stage s, and every ring has full / empty mbarriers of its own.
// mbarriers (after t_y): afull[rings * TC_MAX_STAGES], aempty[rings * TC_MAX_STAGES] (slot s of ring w at rings * s + w),
// bfull[TC_MAX_RES_KB], bempty[TC_MAX_RES_KB].
// EPI_EPS has the carve of EPI_STORE (its adjacency boxes are the same 8 KB) plus the [256] column counts in the slot of the
// masked kernel's groups.  EPI_RADIUS stores nothing through shared memory: the carve of the arg-min epilogues.  EPI_KDE:
// the carve of the arg-min epilogues plus the [256] column weights of the y block in that slot.
template <bool kResident, int kEpi>
struct TcCarve {
  static constexpr bool staged = kEpi == EPI_STORE || kEpi == EPI_EPS;
  static constexpr int stages = staged ? (kResident ? TC_STAGES_RES_ST : TC_STAGES_STR_ST)
                                       : (kResident ? TC_STAGES_RES : TC_STAGES_STR);
  static constexpr int rings  = kResident ? 2 : 1;
  static constexpr uint32_t stage_bytes = kResident ? TC_A_BYTES : TC_A_BYTES + TC_BH_BYTES;
  static constexpr size_t a_off   = kResident ? (size_t)TC_MAX_RES_KB * TC_B_BYTES : 0;
  static constexpr size_t stg_off = a_off + (size_t)stages * stage_bytes;
  static constexpr size_t tb_off  = staged ? stg_off + 2 * (size_t)TC_STG_BOXES * TC_D_BOX_BYTES : TC_SMEM_OPERANDS;
  static constexpr size_t grp_off = tb_off + TC_BN * 4 + 256;   // EPI_MINLOC_MASKED: [256] group, EPI_EPS: count of every column,
                                                                // EPI_KDE: weight of every column
  static constexpr size_t bytes   = grp_off + (kEpi == EPI_MINLOC_MASKED || kEpi == EPI_EPS || kEpi == EPI_KDE ? TC_BN * 4 : 0);
  static_assert(stages <= TC_MAX_STAGES, "barrier arrays hold TC_MAX_STAGES stages");
  static_assert((2 * rings * TC_MAX_STAGES + 2 * TC_MAX_RES_KB) * 8 <= grp_off - tb_off - TC_BN * 4,
                "the mbarriers of every ring fit in the 256 bytes after t_y");
  static_assert(!kResident || stages >= TC_MAX_RES_KB, "resident: the ring holds every x k-block of a tile (both halves read them)");
  static_assert(stg_off % 1024 == 0, "SWIZZLE_128B staging boxes need 1024-byte alignment");
  static_assert(staged || stg_off <= TC_SMEM_OPERANDS, "operands fit");
  static_assert(bytes <= 232448, "exceeds the 227 KB per-CTA limit");
};

// index of the s-th selected y block (see TcParams::sel_s)
__host__ __device__ __forceinline__ int sel_to_blk(int s, int S, int lo, int hi)
{
  if (S <= 1) return s;
  const int w = hi - lo;
  return (s / w) * S + lo + (s % w);
}
// how many of the blocks [0, tiles_n) are selected
__host__ __device__ __forceinline__ int sel_count(int tiles_n, int S, int lo, int hi)
{
  if (S <= 1) return tiles_n;
  const int rem = tiles_n % S;
  return (tiles_n / S) * (hi - lo) + max(0, min(rem, hi) - lo);
}

// Work item `item` of a persistent tensor-core launch (TcParams or ScreenParams): y block n_blk, x tiles [mt0, mt1), and
// the nh halves of the y block that lie inside the matrix.
struct TcItem {
  int n_blk, mt0, mt1, nh;
};
template <class P>
__host__ __device__ __forceinline__ TcItem tc_item(const P& p, int64_t item)
{
  TcItem t;
  t.n_blk = sel_to_blk(static_cast<int>(item % p.tiles_sel), p.sel_s, p.sel_lo, p.sel_hi);
  t.mt0   = static_cast<int>(item / p.tiles_sel) * p.chunk;
  t.mt1   = min(t.mt0 + p.chunk, p.tiles_m);
  t.nh    = static_cast<int64_t>(t.n_blk) * TC_BN + TC_HN < p.n ? 2 : 1;
  return t;
}

// EPI_MINLOC_MASKED skip decisions (DESIGN.md section 2 K3m), shared by the producer, the consumers and the host replay of
// the schedule (tests/cpp/masked_schedule_test.cu).  Class bytes are read through mask_cls_at.
__host__ __device__ __forceinline__ unsigned mask_cls_at(const uint8_t* cls, int mt)
{
#ifdef __CUDA_ARCH__
  return __ldg(&cls[mt]);
#else
  return cls[mt];
#endif
}
// the item's last loaded tile (its y block is handed back after it); -1: no tile is loaded, the item is skipped
__host__ __device__ __forceinline__ int mask_mt_last(const uint8_t* cls, int mt0, int mt1)
{
  int mt_last = -1;
  for (int mt = mt0; mt < mt1; ++mt)
    if (mask_cls_at(cls, mt) != 0u) mt_last = mt;
  return mt_last;
}
// half h of a tile with class byte tcls != 0 has stages in the ring: resident, the tile's stages serve both halves;
// streaming, a half no slab needs is not loaded
__host__ __device__ __forceinline__ bool mask_half_loaded(bool resident, unsigned tcls, int h)
{
  return resident || mask_half_live(tcls, h);
}
// half h of nh hands its stages back (resident: the tile's last half, after both have read them)
__host__ __device__ __forceinline__ bool tc_half_releases(bool resident, int h, int nh) { return !resident || h == nh - 1; }

// The producer's load order, one definition for every instantiation and for the host replay of the masked schedule:
// load_b(kb, it_local, t) for each k-block of a resident y block, load_a(a_it, t, mt, h, kb) for each stage (t: the
// work item, tc_item).
// kMasked skips the loads of dead tiles: a tile whose class byte is 0 loads nothing; in the streaming variant a half no
// slab needs loads nothing; an item without a live tile loads no y block and does not count in it_local (the bfull /
// bempty parity).
#pragma nv_exec_check_disable
template <bool kResident, bool kMasked, class P, class LoadB, class LoadA>
__host__ __device__ __forceinline__ void tc_producer_walk(const P& p, int nkb, int64_t first_item, int64_t stride,
                                                          LoadB&& load_b, LoadA&& load_a)
{
  uint32_t a_it = 0, it_local = 0;
  for (int64_t item = first_item; item < p.n_items; item += stride) {
    const TcItem t     = tc_item(p, item);
    const uint8_t* cls = kMasked ? p.mask_cls + static_cast<int64_t>(t.n_blk) * p.tiles_m : nullptr;
    bool b_loaded      = false;
    for (int mt = t.mt0; mt < t.mt1; ++mt) {
      unsigned tcls = 0u;
      if constexpr (kMasked) {
        tcls = mask_cls_at(cls, mt);
        if (tcls == 0u) continue;
      }
      // resident: one load of an x k-block serves both halves of the tile; streaming: every stage carries its y half
      for (int h = 0; h < (kResident ? 1 : t.nh); ++h) {
        if constexpr (kMasked)
          if (!mask_half_loaded(kResident, tcls, h)) continue;
        for (int kb = 0; kb < nkb; ++kb, ++a_it) {
          // the item's first loaded tile brings its y block (unmasked, every tile is loaded)
          if (kResident && (kMasked ? !b_loaded : mt == t.mt0)) load_b(kb, it_local, t);
          load_a(a_it, t, mt, h, kb);
        }
        b_loaded = true;
      }
    }
    if (!kMasked || b_loaded) ++it_local;
  }
}

// EPI_TOPK candidate lists of the fused brute-force kNN (knn.cuh)
constexpr int KNN_MAX_K = 64;
constexpr int KNN_CAP   = 128;   // list entries per row and pass
constexpr int KNN_SORT  = 256;   // KNN_MAX_K + KNN_CAP padded to a power of two

}  // namespace b2d
