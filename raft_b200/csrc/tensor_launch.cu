// Launch code of the tensor-core path: workspace layout, operand preparation (prep.cuh), the persistent schedule and
// every instantiation of expanded_tc_kernel, and the coarse screening pass (screen_tc.cuh).
#include <cuda.h>
#include <cuda_runtime.h>
#include <algorithm>
#include <cstring>

#include "host.cuh"
#include "dispatch_plan.cuh"
#include "expanded_tc.cuh"
#include "prep.cuh"
#include "screen_tc.cuh"

namespace b2d {

// packed operand [rows][nkb*64] fp16, box = 64 x box_rows, SWIZZLE_128B
// (hi_only: boxes of the 32 hi halves of a k-block, 64 B rows, SWIZZLE_64B -- the coarse screening pass)
static int make_operand_map(CUtensorMap* map, const void* base, int64_t rows, int nkb, int box_rows,
                            int kb0 = 0, int nkb_total = 0, bool hi_only = false)
{
  if (nkb_total == 0) nkb_total = nkb;
  base = static_cast<const char*>(base) + static_cast<size_t>(kb0) * 128;  // K chunk [kb0, kb0 + nkb) of every row
  return encode_2d(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, base, static_cast<int64_t>(nkb) * 64, rows,
                   static_cast<int64_t>(nkb_total) * 128, hi_only ? 32u : 64u, static_cast<unsigned>(box_rows),
                   hi_only ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "");
}

TcWorkspace tc_layout(Carve& c, int64_t m, int64_t n, int64_t k, bool with_keys)
{
  const int nkb = static_cast<int>((k + 31) / 32);
  TcWorkspace w{};
  w.gmax = c.take<unsigned>(8);   // gmax[2], coef, has_lo, nonuni[2]
  if (w.gmax) {
    w.coef   = reinterpret_cast<float*>(w.gmax + 2);
    w.has_lo = w.gmax + 3;
    w.nonuni = w.gmax + 4;
  }
  w.xt   = c.take<float>(m);
  w.xsc  = c.take<float>(m);
  w.keys = c.take<long long>(with_keys ? m : 0);
  // screened fusedL2NN scratch: thresholds, counters, candidate list (128 per row and 1M-row chunk of y;
  // ~54 measured on far-from-origin clusters; overflow falls back to the exact pass on the device,
  // never to a wrong answer)
  // (+2^19: the coarse kernel's warps take list slots in blocks of 64 -- 132 x 8 warps x 2 launches leave up to
  // ~135k slots unused, which must not look like an overflow when m is small)
  w.cand_cap = with_keys ? static_cast<unsigned>(std::min<int64_t>(128 * m + (1 << 19), 0x7fffffff)) : 0u;
  w.aux      = c.take<float4>(with_keys ? m : 0);
  w.cand_cnt = c.take<unsigned>(with_keys ? 8 : 0);
  w.cand     = c.take<int2>(w.cand_cap);
  w.yt   = c.take<float>(n);
  w.ysc  = c.take<float>(n);
  w.xop  = c.take<__half>(static_cast<size_t>(m) * nkb * 64);
  w.yop  = c.take<__half>(static_cast<size_t>(n) * nkb * 64);
  const size_t ns = with_keys ? static_cast<size_t>(std::min<int64_t>(n, kNnChunkRows)) : 0;
  for (int i = 0; i < 2; ++i) {
    w.sort_key[i] = c.take<unsigned>(ns);
    w.sort_val[i] = c.take<int>(ns);
  }
  w.sort_tmp = c.take<char>(with_keys ? kSortTmpBytes : 0);
  if (with_keys) {
    w.xlo = c.take<float>(m);
    w.ylo = c.take<float>(n);
  }
  w.bytes = c.bytes;
  return w;
}

TcWorkspace tc_layout(void* base, int64_t m, int64_t n, int64_t k, bool with_keys)
{
  Carve c(base, 1024);
  return tc_layout(c, m, n, k, with_keys);
}

TcWorkspace tc_rows(TcWorkspace w, int side, int64_t r0, int64_t k)
{
  const int64_t nkb = (k + 31) / 32;
  (side ? w.yop : w.xop) += static_cast<size_t>(r0) * nkb * 64;
  (side ? w.yt : w.xt) += r0;
  (side ? w.ysc : w.xsc) += r0;
  return w;
}

bool tc_metric(int metric, int64_t k, TcMetric* out)
{
  switch (metric) {  // {mode, center, post, xform, coef_mul, tx_const}
    case B2D_L2Expanded:         *out = TC_L2; return true;
    case B2D_L2SqrtExpanded:      *out = TcMetric{PREP_L2,         0, POST_CLAMP_SQRT, 0,  1.f, 0.f}; return true;
    case B2D_CosineExpanded:      *out = TcMetric{PREP_COSINE,     0, POST_NONE,       0,  1.f, 0.f}; return true;
    case B2D_CorrelationExpanded: *out = TcMetric{PREP_COSINE,     1, POST_NONE,       0,  1.f, 0.f}; return true;
    case B2D_InnerProduct:        *out = TcMetric{PREP_INNER,      0, POST_NONE,       0,  1.f, 0.f}; return true;
    case B2D_HellingerExpanded:   *out = TcMetric{PREP_INNER,      0, POST_CLAMP_SQRT, 1, -1.f, 1.f}; return true;
    case B2D_RusselRaoExpanded:   *out = TcMetric{PREP_INNER,      0, POST_NONE,       0, -1.f / static_cast<float>(k), 1.f}; return true;
    case B2D_JaccardExpanded:     *out = TcMetric{PREP_INNER_NORM, 0, POST_JACCARD,    0,  1.f, 0.f}; return true;
    case B2D_DiceExpanded:        *out = TcMetric{PREP_INNER_NORM, 0, POST_DICE,       0,  1.f, 0.f}; return true;
    default: return false;
  }
}

int64_t tc_self_diag(const TcMetric& tm, const void* x, int64_t xrs, int64_t xcs, int64_t m, const void* y, int64_t yrs,
                     int64_t ycs, int64_t n)
{
  const bool same = x == y && m == n && xrs == yrs && xcs == ycs;
  return same && tm.mode == PREP_L2 && tc_post_clamps(tm.post) ? 0 : TC_NO_DIAG;
}

template <typename T>
int launch_prep(cudaStream_t s, const TcWorkspace& w, const void* x, int64_t xrs, int64_t xcs, int64_t m,
                const void* y, int64_t yrs, int64_t ycs, int64_t n, int64_t k, const float* xn, const float* yn,
                const TcMetric& tm, const int* y_gather, bool y_only, const unsigned* run_flag)
{
  PrepParams p;
  p.side[0] = PrepSide{x, xrs, xcs, m, w.xop, w.xt, w.xsc, xn, w.xlo, nullptr};
  p.side[1] = PrepSide{y, yrs, ycs, n, w.yop, w.yt, w.ysc, yn, w.ylo, y_gather};
  p.k = static_cast<int>(k); p.nkb = static_cast<int>((k + 31) / 32); p.mode = tm.mode; p.center = tm.center;
  p.gmax = w.gmax; p.coef = w.coef; p.has_lo = w.has_lo; p.nonuni = w.nonuni;
  p.xform = tm.xform; p.coef_mul = tm.coef_mul; p.tx_const = tm.tx_const;
  p.first_side = y_only ? 1 : 0; p.run_flag = run_flag;
  // (y_only: the caller has zeroed gmax[1] and nonuni[1] on the stream -- km_begin_kernel)
  if (!y_only) B2D_CUDA(cudaMemsetAsync(w.gmax, 0, 32, s));
  const int64_t blocks = ((y_only ? 0 : m) + n + 7) / 8;
  prep_max_kernel<T><<<static_cast<unsigned>(blocks), 256, 0, s>>>(p);
  B2D_CUDA(cudaGetLastError());
  prep_split_kernel<T><<<static_cast<unsigned>(blocks), 256, 0, s>>>(p);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}
template int launch_prep<float>(cudaStream_t, const TcWorkspace&, const void*, int64_t, int64_t, int64_t, const void*,
                                int64_t, int64_t, int64_t, int64_t, const float*, const float*, const TcMetric&,
                                const int*, bool, const unsigned*);
template int launch_prep<__half>(cudaStream_t, const TcWorkspace&, const void*, int64_t, int64_t, int64_t, const void*,
                                 int64_t, int64_t, int64_t, int64_t, const float*, const float*, const TcMetric&,
                                 const int*, bool, const unsigned*);

template <bool kRes, int kEpi, int kPost>
static int launch_tc_inst(cudaStream_t s, const CUtensorMap& ma, const CUtensorMap& mb, const CUtensorMap (&md)[2],
                          const TcParams& p, int grid)
{
  constexpr size_t smem = TcCarve<kRes, kEpi>::bytes;
  // the attribute is per device and per function: cheap, set on every launch
  B2D_CUDA(cudaFuncSetAttribute(expanded_tc_kernel<kRes, kEpi, kPost>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                static_cast<int>(smem)));
  expanded_tc_kernel<kRes, kEpi, kPost><<<grid, TC_THREADS, smem, s>>>(ma, mb, md[0], md[1], p);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

template <bool kRes>
static int launch_tc_epi(cudaStream_t s, const CUtensorMap& ma, const CUtensorMap& mb, const CUtensorMap (&md)[2],
                         const TcParams& p, int grid, int epi, int post)
{
  if (epi == EPI_MINLOC) return launch_tc_inst<kRes, EPI_MINLOC, POST_NONE>(s, ma, mb, md, p, grid);
  if (epi == EPI_MINLOC_MASKED) return launch_tc_inst<kRes, EPI_MINLOC_MASKED, POST_NONE>(s, ma, mb, md, p, grid);
  if (epi == EPI_TOPK) return launch_tc_inst<kRes, EPI_TOPK, POST_NONE>(s, ma, mb, md, p, grid);
  if (epi == EPI_EPS) return launch_tc_inst<kRes, EPI_EPS, POST_CLAMP>(s, ma, mb, md, p, grid);
  if (epi == EPI_RADIUS) {
    if (post == POST_CLAMP) return launch_tc_inst<kRes, EPI_RADIUS, POST_CLAMP>(s, ma, mb, md, p, grid);
    if (post == POST_CLAMP_SQRT) return launch_tc_inst<kRes, EPI_RADIUS, POST_CLAMP_SQRT>(s, ma, mb, md, p, grid);
    return launch_tc_inst<kRes, EPI_RADIUS, POST_NONE>(s, ma, mb, md, p, grid);
  }
  if (post == POST_NONE) return launch_tc_inst<kRes, EPI_STORE, POST_NONE>(s, ma, mb, md, p, grid);
  if (post == POST_CLAMP) return launch_tc_inst<kRes, EPI_STORE, POST_CLAMP>(s, ma, mb, md, p, grid);
  if (post == POST_JACCARD) return launch_tc_inst<kRes, EPI_STORE, POST_JACCARD>(s, ma, mb, md, p, grid);
  if (post == POST_DICE) return launch_tc_inst<kRes, EPI_STORE, POST_DICE>(s, ma, mb, md, p, grid);
  if (post == POST_RBF) return launch_tc_inst<kRes, EPI_STORE, POST_RBF>(s, ma, mb, md, p, grid);
  if (post == POST_POLY) return launch_tc_inst<kRes, EPI_STORE, POST_POLY>(s, ma, mb, md, p, grid);
  if (post == POST_TANH) return launch_tc_inst<kRes, EPI_STORE, POST_TANH>(s, ma, mb, md, p, grid);
  return launch_tc_inst<kRes, EPI_STORE, POST_CLAMP_SQRT>(s, ma, mb, md, p, grid);
}

// Schedule of a persistent tensor-core launch (TcParams or ScreenParams, tc_item): fills tiles_m, tiles_sel, chunk,
// chunks_m and n_items of p from m, n and the y block selection, and sets *grid to one CTA per SM (fewer if there are
// fewer items).  The x tiles are cut into runs so that each SM gets about items_per_sm items; a run holds at most
// max_chunk tiles.
template <class P>
static int plan_tc_items(P& p, int items_per_sm, int max_chunk, int* grid)
{
  int sms = 0;
  const int rc = device_sms(&sms);
  if (rc) return rc;
  p.tiles_m         = static_cast<int>((p.m + TC_BM - 1) / TC_BM);
  const int tiles_n = static_cast<int>((p.n + TC_BN - 1) / TC_BN);
  p.tiles_sel       = sel_count(tiles_n, p.sel_s, p.sel_lo, p.sel_hi);
  int64_t chunk     = static_cast<int64_t>(p.tiles_m) * p.tiles_sel / (static_cast<int64_t>(sms) * items_per_sm);
  chunk             = std::max<int64_t>(1, std::min<int64_t>(chunk, max_chunk));
  chunk             = std::min<int64_t>(chunk, p.tiles_m);
  p.chunk           = static_cast<int>(chunk);
  p.chunks_m        = (p.tiles_m + p.chunk - 1) / p.chunk;
  p.n_items         = static_cast<int64_t>(p.tiles_sel) * p.chunks_m;
  *grid             = static_cast<int>(p.n_items < sms ? p.n_items : sms);
  return B2D_OK;
}

int launch_tc(cudaStream_t s, const TcWorkspace& w, TcParams p, int64_t k, int epi, int post, int kb0, int nkb_chunk)
{
  const int nkb_total = static_cast<int>((k + 31) / 32);
  p.nkb     = nkb_chunk ? nkb_chunk : nkb_total;
  p.tiles_n = static_cast<int>((p.n + TC_BN - 1) / TC_BN);
  int grid  = 0;
  int rc    = plan_tc_items(p, 6, 32, &grid);
  if (rc) return rc;
  p.xt       = w.xt;
  p.yt       = w.yt;
  p.coef     = w.coef;
  p.has_lo   = w.has_lo;
  p.xsc      = w.xsc;
  p.ysc      = w.ysc;
  p.nonuni   = w.nonuni;
  if (p.n_items == 0) return B2D_OK;
  const bool resident = tc_resident(p.nkb);
  CUtensorMap ma, mb;
  // resident: each consumer warpgroup's ring takes the 64-row slab of an x tile it multiplies; streaming: whole tiles
  rc = make_operand_map(&ma, w.xop, p.m, p.nkb, resident ? TC_BM / 2 : TC_BM, kb0, nkb_total);
  if (rc) return rc;
  // resident: the whole 256-row y block in one box per k-block; streaming: one 128-row half per stage
  rc = make_operand_map(&mb, w.yop, p.n, p.nkb, resident ? TC_BN : TC_HN, kb0, nkb_total);
  if (rc) return rc;
  CUtensorMap md[2];   // only read by the kernel when EPI_STORE or EPI_EPS goes through TMA
  memset(md, 0, sizeof(md));
  // both need a 16-byte aligned base and pitch.  EPI_STORE: dist [m][n] fp32 as {32 columns, column group, row} in boxes
  // of 32 x 2 x 32 (expanded_tc.cuh tc_stage_store): md[0] holds the ng = n / 32 whole column groups; when n % 32 != 0,
  // md[1] holds n % 32 columns of the groups from the box that contains the partial group ng (from group ng rounded down
  // to even) to ng.  With no whole group md[0] is a copy of md[1]: the kernel then never stores through md[0].
  // EPI_EPS: adj [m][n] bytes in boxes of 128 columns x 64 rows (tc_eps_tile)
  if (epi == EPI_STORE && p.tma_store) {
    const int64_t ng = p.n / 32, tail = p.n % 32, gb = ng & ~int64_t{1}, pitch[2] = {128, p.ldd * 4};
    const unsigned box[3] = {32, TC_D_BOX_GROUPS, TC_D_BOX_ROWS};
    if (tail != 0) {
      rc = encode_3d(&md[1], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, p.dist + gb * 32, {tail, ng - gb + 1, p.m}, pitch, box,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, "(dist, last column group)");
      if (rc) return rc;
    }
    if (ng != 0) {
      rc = encode_3d(&md[0], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, p.dist, {32, ng, p.m}, pitch, box,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, "(dist)");
      if (rc) return rc;
    } else {
      md[0] = md[1];
    }
  }
  if (epi == EPI_EPS && p.tma_store) {
    rc = encode_2d(&md[0], CU_TENSOR_MAP_DATA_TYPE_UINT8, p.adj, p.n, p.m, p.ld_adj, TC_HN, TC_BM / 2,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, "(adj)");
    if (rc) return rc;
  }
  return resident ? launch_tc_epi<true>(s, ma, mb, md, p, grid, epi, post)
                  : launch_tc_epi<false>(s, ma, mb, md, p, grid, epi, post);
}

int launch_screen(cudaStream_t s, const TcWorkspace& w, int64_t m, int64_t n, int64_t k, int sel_s, int sel_lo,
                  int sel_hi, unsigned* overflow, const unsigned* run_flag, int unit_norm, const int* col_map)
{
  ScreenParams p;
  memset(&p, 0, sizeof(p));
  p.m = m; p.n = n;
  p.nkb     = static_cast<int>((k + 31) / 32);
  if (p.nkb > SC_MAX_KB) return fail(B2D_ERR_UNSUPPORTED, "internal: screening needs k <= 128");
  p.n_stages = static_cast<int>(std::min<size_t>(SC_MAX_STAGES, SC_A_RING / (static_cast<size_t>(p.nkb) * SC_A_KB_BYTES)));
  p.sel_s = sel_s; p.sel_lo = sel_lo; p.sel_hi = sel_hi;
  // long runs of x tiles per y block: the y block load is not overlapped with the previous item
  int grid = 0;
  int rc   = plan_tc_items(p, 4, 128, &grid);
  if (rc) return rc;
  p.xsc = w.xsc; p.nonuni = w.nonuni;
  p.yt = w.yt; p.ylo = w.ylo; p.coef = w.coef; p.aux = w.aux; p.cand = w.cand; p.cand_cnt = w.cand_cnt; p.cand_cap = w.cand_cap;
  p.overflow = overflow; p.run_flag = run_flag; p.unit_norm = unit_norm; p.col_map = col_map;
  if (p.n_items == 0) return B2D_OK;
  CUtensorMap ma, mb;
  rc = make_operand_map(&ma, w.xop, m, p.nkb, TC_BM, 0, 0, true);
  if (rc) return rc;
  rc = make_operand_map(&mb, w.yop, n, p.nkb, TC_BN, 0, 0, true);
  if (rc) return rc;
  B2D_CUDA(cudaFuncSetAttribute(screen_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                static_cast<int>(SC_SMEM_BYTES)));
  screen_tc_kernel<<<grid, SC_THREADS, SC_SMEM_BYTES, s>>>(ma, mb, p);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

}  // namespace b2d
