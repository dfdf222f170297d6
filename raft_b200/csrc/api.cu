// C-ABI entry points (include/raft_b200.h) and host-side dispatch.
#include <cuda.h>
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <algorithm>
#include <atomic>
#include <mutex>
#include <string>
#include <vector>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_segmented_radix_sort.cuh>

#include "../../include/raft_b200.h"
#include "expanded_tc.cuh"
#include "dispatch_plan.cuh"
#include "masked_nn.cuh"
#include "screen_tc.cuh"
#include "prep.cuh"
#include "unexpanded_simt.cuh"
#include "stats.cuh"
#include "fp64_simt.cuh"
#include "select_k.cuh"
#include "kmeans.cuh"
#include "single_linkage.cuh"
#include "dbscan.cuh"

namespace b2d {

static thread_local std::string g_err;

static int fail(int code, const std::string& msg)
{
  g_err = msg;
  return code;
}
#define B2D_CUDA(call)                                                                       \
  do {                                                                                       \
    cudaError_t e__ = (call);                                                                \
    if (e__ != cudaSuccess)                                                                  \
      return fail(B2D_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e__));        \
  } while (0)

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// Cuts a caller's workspace into consecutive regions, each rounded up to `align` bytes.  With a null base it only
// counts the bytes (the *_workspace_bytes queries): every region is then null, and no pointer is formed from null.
struct Carve {
  char* base;
  size_t align;
  size_t bytes = 0;
  Carve(void* b, size_t a) : base(static_cast<char*>(b)), align(a) {}
  template <typename T>
  T* take(size_t count)
  {
    T* at = base ? reinterpret_cast<T*>(base + bytes) : nullptr;
    bytes += align_up(count * sizeof(T), align);
    return at;
  }
};

// the caller's workspace holds `need` bytes (none needed: anything goes) and starts on an `align`-byte boundary
static int check_workspace(const void* ws, size_t bytes, size_t need, size_t align = 256)
{
  if (need > 0 && (!ws || bytes < need))
    return fail(B2D_ERR_WORKSPACE, "workspace too small: need " + std::to_string(need) + " bytes");
  if (reinterpret_cast<uintptr_t>(ws) % align) return fail(B2D_ERR_INVALID_ARG, "workspace must be 256-byte aligned");
  return B2D_OK;
}

// process-wide tuning / test hooks (b2d_set_option): nothing on the hot path reads the environment
static std::atomic<float> g_nn_tau{6.0f};   // screened fusedL2NN: candidates per row above which the trial calls screening off
static std::atomic<int> g_nn_screen{1};     // 0: always the exact arg-min kernel

// ------------------------------------------------------------------------------------------
// TMA descriptor encode through the driver entry point (no link-time libcuda dependency, so the
// library still loads -- and reports a clean error -- on a machine without a driver).
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode()
{
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

// a row-major matrix [rows][cols] of `dtype` with a row pitch of pitch_bytes, in boxes of box_cols x box_rows;
// `tag` names the map in the error message
static int encode_2d(CUtensorMap* map, CUtensorMapDataType dtype, const void* base, int64_t cols, int64_t rows,
                     int64_t pitch_bytes, unsigned box_cols, unsigned box_rows, CUtensorMapSwizzle swizzle,
                     CUtensorMapL2promotion promotion, const char* tag)
{
  EncodeTiledFn enc = get_encode();
  if (!enc) return fail(B2D_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
  cuuint64_t dims[2]    = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  cuuint64_t strides[1] = {static_cast<cuuint64_t>(pitch_bytes)};
  cuuint32_t box[2]     = {box_cols, box_rows};
  cuuint32_t estr[2]    = {1, 1};
  CUresult r = enc(map, dtype, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                   promotion, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail(B2D_ERR_CUDA, std::string("cuTensorMapEncodeTiled") + tag + " failed: " + std::to_string((int)r));
  return B2D_OK;
}

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

// SM count of the current device; every kernel of the library is built for sm_90a only, so any other device is an error
static int device_sms(int* sms)
{
  int dev = 0, cc = 0;
  B2D_CUDA(cudaGetDevice(&dev));
  B2D_CUDA(cudaDeviceGetAttribute(sms, cudaDevAttrMultiProcessorCount, dev));
  B2D_CUDA(cudaDeviceGetAttribute(&cc, cudaDevAttrComputeCapabilityMajor, dev));
  if (cc != 9) return fail(B2D_ERR_CUDA, "raft_b200 requires an sm_90 (H100) device; found cc major " + std::to_string(cc));
  return B2D_OK;
}

// ------------------------------------------------------------------------------------------
// Optional timing of the dominant kernel (bench.py's roofline): CUDA events on the call's stream around
// the main kernel of every b2d_pairwise_distance call between b2d_profile_begin and b2d_profile_end.
// Nothing is synchronised until b2d_profile_end, so the timed region of the caller is not perturbed.
namespace {
struct ProfileRing {
  std::vector<cudaEvent_t> ev;  // pairs
  int used = 0;
  bool on  = false;
} g_prof;
std::mutex g_prof_mu;
std::atomic<bool> g_prof_armed{false};   // fast path: a call outside a profiling region touches no lock

struct ProfileScope {
  cudaStream_t s;
  int slot = -1;
  explicit ProfileScope(cudaStream_t st) : s(st)
  {
    if (!g_prof_armed.load(std::memory_order_acquire)) return;
    std::lock_guard<std::mutex> lk(g_prof_mu);
    if (g_prof.on && 2 * (g_prof.used + 1) <= static_cast<int>(g_prof.ev.size())) {
      slot = g_prof.used++;
      cudaEventRecord(g_prof.ev[2 * slot], s);
    }
  }
  ~ProfileScope()
  {
    if (slot >= 0) cudaEventRecord(g_prof.ev[2 * slot + 1], s);
  }
};
}  // namespace

// ------------------------------------------------------------------------------------------
// workspace layout of the tensor-core path
struct TcWorkspace {
  __half* xop;
  __half* yop;
  float* xt;
  float* yt;
  float* xsc;        // [m] per-row scale 2^(E - e_row) of x (1 unless the row took its own exponent, prep.cuh)
  float* ysc;        // [n] the same for y
  unsigned* nonuni;  // [2] some row of x / y took its own exponent
  long long* keys;
  unsigned* gmax;  // [2]
  float* coef;     // [1]
  unsigned* has_lo;  // [1]
  float4* aux;       // [m]    screened NN: per-row (bound - |x|^2, |x|, |x - hi part|, -)
  float* xlo;        // [m]    screened NN: |x_i - hi part| (prep.cuh lvec)
  float* ylo;        // [n]
  int2* cand;        // [cap]  screened NN: candidate list
  unsigned* cand_cnt;  // [1] (+ overflow flag right behind it)
  unsigned cand_cap;
  // screened NN: the database chunk is worked through in the order of its squared row norms (screen_tc.cuh)
  unsigned* sort_key[2];  // [min(n, 2^20)] each
  int* sort_val[2];       // [min(n, 2^20)] each: position -> source row
  void* sort_tmp;
  size_t bytes;      // end of these regions in the workspace
};
constexpr int64_t kNnChunkRows  = 1 << 20;   // database rows per screened chunk
constexpr size_t kSortTmpBytes  = 4u << 20;  // cub::DeviceRadixSort scratch for <= 2^20 pairs (checked at run time)

// the tensor-core path's regions at the front of `c` (1024-byte alignment); with_keys: the screened arg-min's too
static TcWorkspace tc_layout(Carve& c, int64_t m, int64_t n, int64_t k, bool with_keys)
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

static TcWorkspace tc_layout(void* base, int64_t m, int64_t n, int64_t k, bool with_keys)
{
  Carve c(base, 1024);
  return tc_layout(c, m, n, k, with_keys);
}

// w with side 0 (x) or side 1 (y) starting at prepared row r0: the operand, t and scale rows the tensor kernels read
static TcWorkspace tc_rows(TcWorkspace w, int side, int64_t r0, int64_t k)
{
  const int64_t nkb = (k + 31) / 32;
  (side ? w.yop : w.xop) += static_cast<size_t>(r0) * nkb * 64;
  (side ? w.yt : w.xt) += r0;
  (side ? w.ysc : w.xsc) += r0;
  return w;
}

static bool is_expanded(int metric)
{
  return metric == B2D_L2Expanded || metric == B2D_L2SqrtExpanded || metric == B2D_CosineExpanded ||
         metric == B2D_CorrelationExpanded || metric == B2D_InnerProduct || metric == B2D_HellingerExpanded ||
         metric == B2D_RusselRaoExpanded || metric == B2D_JaccardExpanded || metric == B2D_DiceExpanded;
}
static bool is_unexpanded(int metric)
{
  return metric == B2D_L1 || metric == B2D_L2Unexpanded || metric == B2D_L2SqrtUnexpanded ||
         metric == B2D_Linf || metric == B2D_Canberra || metric == B2D_LpUnexpanded ||
         metric == B2D_HammingUnexpanded || metric == B2D_KLDivergence || metric == B2D_JensenShannon ||
         metric == B2D_BrayCurtis;
}

template <typename T>
static int launch_prep(cudaStream_t s, const TcWorkspace& w, const void* x, int64_t xrs, int64_t xcs, int64_t m,
                       const void* y, int64_t yrs, int64_t ycs, int64_t n, int64_t k, const float* xn, const float* yn,
                       int mode, int center, int xform = 0, float coef_mul = 1.f, float tx_const = 0.f,
                       const int* y_gather = nullptr, bool y_only = false, const unsigned* run_flag = nullptr)
{
  PrepParams p;
  p.side[0] = PrepSide{x, xrs, xcs, m, w.xop, w.xt, w.xsc, xn, w.xlo, nullptr};
  p.side[1] = PrepSide{y, yrs, ycs, n, w.yop, w.yt, w.ysc, yn, w.ylo, y_gather};
  p.k = static_cast<int>(k); p.nkb = static_cast<int>((k + 31) / 32); p.mode = mode; p.center = center;
  p.gmax = w.gmax; p.coef = w.coef; p.has_lo = w.has_lo; p.nonuni = w.nonuni;
  p.xform = xform; p.coef_mul = coef_mul; p.tx_const = tx_const;
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

template <bool kRes, int kEpi, int kPost>
static int launch_tc_inst(cudaStream_t s, const CUtensorMap& ma, const CUtensorMap& mb, const CUtensorMap& md,
                          const TcParams& p, int grid)
{
  constexpr size_t smem = TcCarve<kRes, kEpi>::bytes;
  // the attribute is per device and per function: cheap, set on every launch
  B2D_CUDA(cudaFuncSetAttribute(expanded_tc_kernel<kRes, kEpi, kPost>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                static_cast<int>(smem)));
  expanded_tc_kernel<kRes, kEpi, kPost><<<grid, TC_THREADS, smem, s>>>(ma, mb, md, p);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

template <bool kRes>
static int launch_tc_epi(cudaStream_t s, const CUtensorMap& ma, const CUtensorMap& mb, const CUtensorMap& md,
                         const TcParams& p, int grid, int epi, int post)
{
  if (epi == EPI_MINLOC) return launch_tc_inst<kRes, EPI_MINLOC, POST_NONE>(s, ma, mb, md, p, grid);
  if (epi == EPI_MINLOC_MASKED) return launch_tc_inst<kRes, EPI_MINLOC_MASKED, POST_NONE>(s, ma, mb, md, p, grid);
  if (epi == EPI_TOPK) return launch_tc_inst<kRes, EPI_TOPK, POST_NONE>(s, ma, mb, md, p, grid);
  if (epi == EPI_EPS) return launch_tc_inst<kRes, EPI_EPS, POST_CLAMP>(s, ma, mb, md, p, grid);
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

static int launch_tc(cudaStream_t s, const TcWorkspace& w, TcParams p, int64_t k, int epi, int post, int kb0 = 0,
                     int nkb_chunk = 0)
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
  CUtensorMap md;   // only read by the kernel when EPI_STORE or EPI_EPS goes through TMA
  memset(&md, 0, sizeof(md));
  // both need a 16-byte aligned base and pitch.  EPI_STORE: dist [m][n] fp32 in boxes of 32 columns x 64 rows
  // (expanded_tc.cuh tc_stage_store); EPI_EPS: adj [m][n] bytes in boxes of 128 columns x 64 rows (tc_eps_tile)
  if (epi == EPI_STORE && p.tma_store) {
    rc = encode_2d(&md, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, p.dist, p.n, p.m, p.ldd * 4, TC_D_BOX_COLS, TC_D_BOX_ROWS,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, "(dist)");
    if (rc) return rc;
  }
  if (epi == EPI_EPS && p.tma_store) {
    rc = encode_2d(&md, CU_TENSOR_MAP_DATA_TYPE_UINT8, p.adj, p.n, p.m, p.ld_adj, TC_HN, TC_D_BOX_ROWS,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, "(adj)");
    if (rc) return rc;
  }
  return resident ? launch_tc_epi<true>(s, ma, mb, md, p, grid, epi, post)
                  : launch_tc_epi<false>(s, ma, mb, md, p, grid, epi, post);
}

// coarse screening pass of the screened fusedL2NN (screen_tc.cuh) over the y blocks with
// sel_lo <= index % sel_s < sel_hi
static int launch_screen(cudaStream_t s, const TcWorkspace& w, int64_t m, int64_t n, int64_t k, int sel_s, int sel_lo,
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

template <int kMetric>
static int launch_ux_inst(cudaStream_t s, const UxParams& p, int64_t tiles, bool tma)
{
  if (tma) {  // TMA-legal operands: hardware-staged tiles of 32 floats x 128 rows, SWIZZLE_128B
    CUtensorMap mx, my;
    int rc = encode_2d(&mx, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, p.x, p.k, p.m, p.xrs * 4, UX_KB, UX_BM,
                       CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "(f32 operand)");
    if (rc) return rc;
    rc = encode_2d(&my, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, p.y, p.k, p.n, p.yrs * 4, UX_KB, UX_BM,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "(f32 operand)");
    if (rc) return rc;
    B2D_CUDA(cudaFuncSetAttribute(unexpanded_tma_kernel<kMetric>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  UX_TMA_SMEM_BYTES));
    unexpanded_tma_kernel<kMetric><<<static_cast<unsigned>(tiles), UX_THREADS, UX_TMA_SMEM_BYTES, s>>>(mx, my, p);
    B2D_CUDA(cudaGetLastError());
    return B2D_OK;
  }
  cudaError_t e = cudaFuncSetAttribute(unexpanded_simt_kernel<kMetric>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       UX_SMEM_BYTES);
  B2D_CUDA(e);
  unexpanded_simt_kernel<kMetric><<<static_cast<unsigned>(tiles), UX_THREADS, UX_SMEM_BYTES, s>>>(p);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

// ------------------------------------------------------------------------------------------
__global__ void row_norm_kernel(float* out, const float* x, int64_t ldx, int64_t rows, int k, int type, int do_sqrt)
{
  const int lane  = threadIdx.x & 31;
  const int64_t r = static_cast<int64_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= rows) return;
  const float* row = x + r * ldx;
  double acc = 0.0;
  float mx   = 0.f;
  for (int t = lane; t < k; t += 32) {
    const float v = __ldg(row + t);
    if (type == B2D_L0PseudoNorm) acc += (v != 0.f) ? 1.0 : 0.0;
    else if (type == B2D_L1Norm) acc += fabs(static_cast<double>(v));
    else if (type == B2D_L2Norm) acc += static_cast<double>(v) * v;
    else mx = fmaxf(mx, fabsf(v));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    acc += __shfl_xor_sync(0xffffffffu, acc, o);
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  if (lane == 0) {
    double v = (type == B2D_LinfNorm) ? static_cast<double>(mx) : acc;
    if (do_sqrt) v = sqrt(v);
    out[r] = static_cast<float>(v);
  }
}

// raft::matrix::argmin (cpp/include/raft/matrix/argmin.cuh:25-37, detail/math.cuh:290-343): column index of the
// minimum of every row, ties -> the smaller index (cub::ArgMin), start value (0, +inf): a row of NaN / +inf gives 0.
// One pass over the matrix: HBM-read bound.  kWarp: one warp per row (short rows), else one 256-thread block per row.
template <bool kWarp>
__global__ void __launch_bounds__(256) row_argmin_kernel(int* out, const float* in, int64_t ld, int64_t rows, int64_t n)
{
  const int lane    = threadIdx.x & 31;
  const int64_t r   = kWarp ? static_cast<int64_t>(blockIdx.x) * 8 + (threadIdx.x >> 5) : blockIdx.x;
  const int t0      = kWarp ? lane : threadIdx.x;
  const int stride  = kWarp ? 32 : 256;
  float v = __int_as_float(0x7f800000);
  int ix  = 0;
  if (r < rows) {
    const float* row = in + r * ld;
    if ((reinterpret_cast<uintptr_t>(row) & 15) == 0 && (ld & 3) == 0) {
      const int64_t n4 = n >> 2;
      for (int64_t c = t0; c < n4; c += stride) {
        const float4 q4 = __ldcs(reinterpret_cast<const float4*>(row) + c);
        const int j     = static_cast<int>(c << 2);
        if (q4.x < v) { v = q4.x; ix = j; }
        if (q4.y < v) { v = q4.y; ix = j + 1; }
        if (q4.z < v) { v = q4.z; ix = j + 2; }
        if (q4.w < v) { v = q4.w; ix = j + 3; }
      }
      for (int64_t c = (n4 << 2) + t0; c < n; c += stride) {
        const float q1 = __ldcs(row + c);
        if (q1 < v) { v = q1; ix = static_cast<int>(c); }
      }
    } else {
      for (int64_t c = t0; c < n; c += stride) {
        const float q1 = __ldcs(row + c);
        if (q1 < v) { v = q1; ix = static_cast<int>(c); }
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi   = __shfl_xor_sync(0xffffffffu, ix, o);
    if (ov < v || (ov == v && oi < ix)) { v = ov; ix = oi; }
  }
  if (kWarp) {
    if (lane == 0 && r < rows) out[r] = ix;
    return;
  }
  __shared__ float sv[8];
  __shared__ int si[8];
  if (lane == 0) { sv[threadIdx.x >> 5] = v; si[threadIdx.x >> 5] = ix; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; ++w)
      if (sv[w] < v || (sv[w] == v && si[w] < ix)) { v = sv[w]; ix = si[w]; }
    out[r] = ix;
  }
}

}  // namespace b2d

using namespace b2d;

// fp64 path: one SIMT kernel per metric (fp64_simt.cuh)
template <int kMetric>
static int launch_f64_inst(cudaStream_t s, const F64Params& p, int64_t tiles)
{
  f64_pairwise_kernel<kMetric><<<static_cast<unsigned>(tiles), 256, 0, s>>>(p);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

static int pairwise_f64(cudaStream_t s, int metric, const double* x, int64_t xrs, int64_t xcs, const double* y, int64_t yrs,
                        int64_t ycs, double* dist, int64_t ldd, int64_t m, int64_t n, int64_t k, int swapped, double metric_arg,
                        void* workspace, size_t workspace_bytes, double gamma = 0.0, double coef0 = 0.0, int degree = 0)
{
  const int rc = check_workspace(workspace, workspace_bytes, align_up(static_cast<size_t>(m + n) * 16, 1024), 1);
  if (rc) return rc;
  double* xs = static_cast<double*>(workspace);
  double* ys = xs + 2 * m;
  f64_row_stats_kernel<<<static_cast<unsigned>((m + 7) / 8), 256, 0, s>>>(xs, x, xrs, xcs, m, static_cast<int>(k));
  f64_row_stats_kernel<<<static_cast<unsigned>((n + 7) / 8), 256, 0, s>>>(ys, y, yrs, ycs, n, static_cast<int>(k));
  B2D_CUDA(cudaGetLastError());
  F64Params p;
  p.x = x; p.y = y; p.dist = dist; p.xrs = xrs; p.xcs = xcs; p.yrs = yrs; p.ycs = ycs; p.ldd = ldd; p.m = m; p.n = n;
  p.k = static_cast<int>(k); p.metric = metric; p.swapped = swapped; p.p = metric_arg; p.inv_p = 1.0 / metric_arg;
  p.xs = xs; p.ys = ys;
  p.gamma = gamma; p.coef0 = coef0; p.degree = degree;
  p.tiles_n = static_cast<int>((n + F64_T - 1) / F64_T);
  const int64_t tiles = ((m + F64_T - 1) / F64_T) * p.tiles_n;
  switch (metric) {
#define B2D_F64_CASE(M) case M: return launch_f64_inst<M>(s, p, tiles);
    B2D_F64_CASE(B2D_L2Expanded) B2D_F64_CASE(B2D_L2SqrtExpanded) B2D_F64_CASE(B2D_CosineExpanded) B2D_F64_CASE(B2D_L1)
    B2D_F64_CASE(B2D_L2Unexpanded) B2D_F64_CASE(B2D_L2SqrtUnexpanded) B2D_F64_CASE(B2D_InnerProduct) B2D_F64_CASE(B2D_Linf)
    B2D_F64_CASE(B2D_Canberra) B2D_F64_CASE(B2D_LpUnexpanded) B2D_F64_CASE(B2D_CorrelationExpanded)
    B2D_F64_CASE(B2D_JaccardExpanded) B2D_F64_CASE(B2D_HellingerExpanded) B2D_F64_CASE(B2D_BrayCurtis)
    B2D_F64_CASE(B2D_JensenShannon) B2D_F64_CASE(B2D_HammingUnexpanded) B2D_F64_CASE(B2D_KLDivergence)
    B2D_F64_CASE(B2D_RusselRaoExpanded) B2D_F64_CASE(B2D_DiceExpanded)
    B2D_F64_CASE(F64_GRAM_POLY) B2D_F64_CASE(F64_GRAM_RBF) B2D_F64_CASE(F64_GRAM_TANH)
#undef B2D_F64_CASE
    default: return fail(B2D_ERR_UNSUPPORTED, "metric");
  }
}

// ------------------------------------------------------------------------------------------
// select_k (select_k.cuh): the layout is a function of the shape alone
namespace {
enum { SK_SORT_ROW = 0, SK_RADIX_ROW = 1, SK_SPLIT = 2 };
constexpr int64_t kSkSplitRows = 264;        // fewer rows than two CTAs per SM of an H100 SXM (132 SMs): split each row
constexpr int64_t kSkMinChunk  = 32768;      // columns per CTA of a split row, at least
constexpr size_t kSkCubTmp     = 1u << 20;   // cub::DeviceSegmentedRadixSort scratch (checked at run time)
constexpr int64_t kSkCubItems  = 1ll << 30;  // words per segmented sort call

struct SkPlan {
  int layout    = SK_SORT_ROW;
  int64_t chunk = 0, chunks = 1;   // SK_SPLIT: columns per CTA, CTAs per row
  bool list     = false;           // the k words of every row go through the workspace
  bool cub      = false;           // ... and are sorted there by cub (k > kSkSortMax)
  int sort_n    = 0;               // power-of-two size of the shared-memory sort
  int cap       = 0;               // SK_RADIX_ROW: live words the row kernel's buffer holds
  int64_t batch = 0;               // rows per segmented sort call
};

static SkPlan sk_plan(int64_t rows, int64_t len, int64_t k)
{
  SkPlan p;
  if (len <= kSkRowSort) {
    p.sort_n = sk_pow2(len);
    return p;
  }
  const int64_t chunks = std::min((len + kSkMinChunk - 1) / kSkMinChunk, (kSkSplitRows + rows - 1) / rows);
  p.layout = chunks > 1 ? SK_SPLIT : SK_RADIX_ROW;
  p.cub    = k > kSkSortMax;
  p.list   = p.layout == SK_SPLIT || p.cub;
  p.sort_n = p.cub ? 0 : sk_pow2(k);
  if (p.layout == SK_SPLIT) {
    p.chunk  = ((len + chunks - 1) / chunks + 3) / 4 * 4;
    p.chunks = (len + p.chunk - 1) / p.chunk;
  } else {
    p.cap = static_cast<int>((kSkRowSmem - kSkBuckets * 4 - (p.list ? 0 : p.sort_n * 8)) / 8);
  }
  if (p.cub) p.batch = std::min(rows, std::max<int64_t>(1, kSkCubItems / k));
  return p;
}

struct SkLayout {
  SkState* st    = nullptr;
  uint32_t* hist = nullptr;
  uint64_t* list = nullptr;
  uint64_t* alt  = nullptr;
  int* off       = nullptr;
  void* tmp      = nullptr;
  size_t bytes   = 0;
};

static SkLayout sk_layout(void* base, const SkPlan& p, int64_t rows, int64_t k)
{
  Carve c(base, 256);
  SkLayout w;
  if (p.layout == SK_SPLIT) {
    w.st   = c.take<SkState>(rows);
    w.hist = c.take<uint32_t>(static_cast<size_t>(rows) * kSkBuckets);
  }
  if (p.list) w.list = c.take<uint64_t>(static_cast<size_t>(rows) * k);
  if (p.cub) {
    w.alt = c.take<uint64_t>(static_cast<size_t>(p.batch) * k);
    w.off = c.take<int>(p.batch + 1);
    w.tmp = c.take<char>(kSkCubTmp);
  }
  w.bytes = c.bytes;
  return w;
}

static bool sk_extents_ok(int64_t rows, int64_t len, int64_t k)
{
  return rows >= 0 && rows <= 0x7fffffffll && k >= 1 && k <= len && len <= 0x7fffffffll;
}
}  // namespace

extern "C" {

int b2d_profile_begin(int capacity)
{
  std::lock_guard<std::mutex> lk(g_prof_mu);
  if (capacity < 1 || capacity > 4096) return fail(B2D_ERR_INVALID_ARG, "capacity must be in [1, 4096]");
  while (static_cast<int>(g_prof.ev.size()) < 2 * capacity) {
    cudaEvent_t e;
    B2D_CUDA(cudaEventCreate(&e));
    g_prof.ev.push_back(e);
  }
  g_prof.used = 0;
  g_prof.on   = true;
  g_prof_armed.store(true, std::memory_order_release);
  return B2D_OK;
}

int b2d_profile_end(float* ms, int max_count, int* count)
{
  std::lock_guard<std::mutex> lk(g_prof_mu);
  g_prof.on = false;
  g_prof_armed.store(false, std::memory_order_release);
  if (!ms || !count || max_count < 0) return fail(B2D_ERR_INVALID_ARG, "null ms / count");
  const int c = std::min(g_prof.used, max_count);
  for (int i = 0; i < c; ++i) {
    B2D_CUDA(cudaEventSynchronize(g_prof.ev[2 * i + 1]));
    B2D_CUDA(cudaEventElapsedTime(&ms[i], g_prof.ev[2 * i], g_prof.ev[2 * i + 1]));
  }
  *count = c;
  return B2D_OK;
}


int b2d_version(void) { return 200; }

int b2d_set_option(const char* name, double value)
{
  if (!name) return fail(B2D_ERR_INVALID_ARG, "null option name");
  const std::string n(name);
  if (n == "nn_tau") {
    if (!(value >= 0.0)) return fail(B2D_ERR_INVALID_ARG, "nn_tau must be >= 0");
    g_nn_tau.store(static_cast<float>(value));
  } else if (n == "nn_screen") {
    g_nn_screen.store(value != 0.0 ? 1 : 0);
  } else {
    return fail(B2D_ERR_INVALID_ARG, "unknown option '" + n + "' (nn_tau, nn_screen)");
  }
  return B2D_OK;
}

// Diagnostic (synchronises `stream`): the control words the last screened fusedL2NN chunk left in `workspace`
// [0] list slots in use (one incumbent per row + blocks of 64 reserved by the screen) [1] list overflow [2] go_screen [3] go_exact [4] redo_trial [5] candidates after the trial [6] candidates found by the screen (out7: 7 words)
int b2d_debug_nn_stats(void* stream, const void* workspace, int64_t m, int64_t n, int64_t k, unsigned* out6 /* 7 words */)
{
  if (!workspace || !out6 || m < 0 || n < 0 || k < 0) return fail(B2D_ERR_INVALID_ARG, "null workspace / out");
  TcWorkspace w = tc_layout(const_cast<void*>(workspace), m, n, k, true);
  B2D_CUDA(cudaStreamSynchronize(static_cast<cudaStream_t>(stream)));
  B2D_CUDA(cudaMemcpy(out6, w.cand_cnt, 7 * sizeof(unsigned), cudaMemcpyDeviceToHost));
  return B2D_OK;
}
const char* b2d_last_error(void) { return g_err.c_str(); }

// What one dense m x n result on the tensor path (EPI_STORE) is made of: the operand preparation (prep.cuh) and the
// epilogue's post-processing, with the kernel parameters of the Gram matrices (gram_post).
struct TcStore {
  int mode = PREP_L2, center = 0, post = POST_NONE, xform = 0;
  float coef_mul = 1.f, tx_const = 0.f;
  float gamma = 0.f, coef0 = 0.f;
  int degree = 0;
};

// The tensor path of b2d_pairwise_distance and b2d_gram_matrix: x [ma, k] and y [na, k] with element strides (xrs, xcs) and
// (yrs, ycs) (a column-major call arrives with the operands exchanged), dist [ma][ldd].  alias: x and y are the same matrix
// (then the L2 family has d(i, i) = 0 exactly).
static int tc_store(cudaStream_t s, const TcStore& c, int dtype, const void* xa, int64_t xrs, int64_t xcs, int64_t ma,
                    const void* ya, int64_t yrs, int64_t ycs, int64_t na, int64_t k, float* dist, int64_t ldd, bool alias,
                    void* workspace, size_t workspace_bytes)
{
  int rc = check_workspace(workspace, workspace_bytes, tc_layout(nullptr, ma, na, k, false).bytes);
  if (rc) return rc;
  TcWorkspace w = tc_layout(workspace, ma, na, k, false);
  rc = dtype == B2D_F32
         ? launch_prep<float>(s, w, xa, xrs, xcs, ma, ya, yrs, ycs, na, k, nullptr, nullptr, c.mode, c.center, c.xform,
                              c.coef_mul, c.tx_const)
         : launch_prep<__half>(s, w, xa, xrs, xcs, ma, ya, yrs, ycs, na, k, nullptr, nullptr, c.mode, c.center, c.xform,
                               c.coef_mul, c.tx_const);
  if (rc) return rc;
  TcParams p;
  memset(&p, 0, sizeof(p));
  p.m = ma; p.n = na; p.dist = dist; p.ldd = ldd;
  p.diag_zero = (c.post != POST_NONE && alias && c.mode == PREP_L2) ? 1 : 0;
  p.gamma = c.gamma; p.coef0 = c.coef0; p.degree = c.degree;
  // (dispatch_plan.cuh: TMA or register stores; k > 320: K chunks accumulated in dist, post-processed on the last)
  const TcStorePlan pl = tc_store_plan(c.post, ma, na, k, reinterpret_cast<uintptr_t>(dist), ldd);
  p.tma_store = pl.tma_store;
  ProfileScope prof(s);  // the main kernel(s) only: the operand preparation above is outside
  for (int i = 0; i < pl.launches; ++i) {
    const TcStoreLaunch l = tc_store_launch(pl, i);
    p.acc_mode = l.acc_mode;
    rc = launch_tc(s, w, p, k, EPI_STORE, c.post, l.kb0, l.nkb);
    if (rc) return rc;
  }
  return B2D_OK;
}

size_t b2d_pairwise_workspace_bytes(int metric, int dtype, int64_t m, int64_t n, int64_t k)
{
  if (dtype != B2D_F32 && dtype != B2D_F16 && dtype != B2D_F64) return static_cast<size_t>(-1);
  if (m < 0 || n < 0 || k < 0) return static_cast<size_t>(-1);
  if (dtype == B2D_F64)   // per-row (sum, sum of squares) of x and y
    return (is_expanded(metric) || is_unexpanded(metric)) ? align_up(static_cast<size_t>(m + n) * 16, 1024) : static_cast<size_t>(-1);
  if (is_unexpanded(metric)) return dtype == B2D_F32 ? 0 : static_cast<size_t>(-1);
  if (!is_expanded(metric)) return static_cast<size_t>(-1);
  return tc_layout(nullptr, m, n, k, false).bytes;
}

// The argument checks of b2d_pairwise_distance.  *empty: nothing to compute (m or n is 0).
static int pairwise_check(int metric, int dtype, const void* x, int64_t ldx, const void* y, int64_t ldy, const void* dist,
                          int64_t ldd, int64_t m, int64_t n, int64_t k, int row_major, float metric_arg, bool* empty)
{
  *empty = false;
  if (m < 0 || n < 0 || k < 0) return fail(B2D_ERR_INVALID_ARG, "negative extent");
  if (m == 0 || n == 0) { *empty = true; return B2D_OK; }
  if (k == 0) return fail(B2D_ERR_INVALID_ARG, "k must be positive");
  if (!x || !y || !dist) return fail(B2D_ERR_INVALID_ARG, "null x / y / dist");
  if (m > 0x7fffffffll * 128 || n > 0x7fffffffll || k > (1 << 24)) return fail(B2D_ERR_INVALID_ARG, "extent too large");
  if (row_major) {
    if (ldx < k || ldy < k || ldd < n) return fail(B2D_ERR_INVALID_ARG, "leading dimension smaller than the row length");
  } else {
    if (ldx < m || ldy < n || ldd < m) return fail(B2D_ERR_INVALID_ARG, "leading dimension smaller than the column length");
  }
  if (!is_expanded(metric) && !is_unexpanded(metric))
    return fail(B2D_ERR_UNSUPPORTED, "metric " + std::to_string(metric) + " is not on the tensor-core / SIMT distance path");
  if (dtype != B2D_F32 && dtype != B2D_F16 && dtype != B2D_F64) return fail(B2D_ERR_UNSUPPORTED, "dtype");
  if (metric == B2D_LpUnexpanded && !(metric_arg > 0.f)) return fail(B2D_ERR_INVALID_ARG, "LpUnexpanded needs p > 0");
  if (dtype == B2D_F16 && !is_expanded(metric)) return fail(B2D_ERR_UNSUPPORTED, "unexpanded metrics take fp32 inputs");
  return B2D_OK;
}

// The operands as the fp32 / fp16 kernels take them: dist is always written as a row-major [ma][ldd] matrix.
// Fortran order: D^T (row-major [n,m]) = metric(y_j, x_i).  Every metric here is symmetric except
// KLDivergence, which switches to the kernel with the operand roles exchanged (UX_KL_REV).
struct PairwiseOperands {
  const void *xa, *ya;
  int64_t ma, na, xrs, xcs, yrs, ycs;
};
static PairwiseOperands pairwise_operands(const void* x, int64_t ldx, const void* y, int64_t ldy, int64_t m, int64_t n,
                                          int row_major)
{
  if (row_major) return PairwiseOperands{x, y, m, n, ldx, 1, ldy, 1};
  return PairwiseOperands{y, x, n, m, 1, ldy, 1, ldx};
}

// preparation and epilogue of the expanded metrics on the tensor path
static TcStore pairwise_tc_store(int metric, int64_t k)
{
  TcStore c;
  if (metric == B2D_L2Expanded) { c.post = POST_CLAMP; }
  else if (metric == B2D_L2SqrtExpanded) { c.post = POST_CLAMP_SQRT; }
  else if (metric == B2D_CosineExpanded) { c.mode = PREP_COSINE; }
  else if (metric == B2D_CorrelationExpanded) { c.mode = PREP_COSINE; c.center = 1; }
  else if (metric == B2D_HellingerExpanded) { c.mode = PREP_INNER; c.post = POST_CLAMP_SQRT; c.xform = 1; c.coef_mul = -1.f; c.tx_const = 1.f; }
  else if (metric == B2D_RusselRaoExpanded) { c.mode = PREP_INNER; c.coef_mul = -1.f / static_cast<float>(k); c.tx_const = 1.f; }
  else if (metric == B2D_JaccardExpanded) { c.mode = PREP_INNER_NORM; c.post = POST_JACCARD; }
  else if (metric == B2D_DiceExpanded) { c.mode = PREP_INNER_NORM; c.post = POST_DICE; }
  else { c.mode = PREP_INNER; }
  return c;
}

int b2d_debug_pairwise_plan(int metric, int dtype, const void* x, int64_t ldx, const void* y, int64_t ldy, const void* dist,
                            int64_t ldd, int64_t m, int64_t n, int64_t k, int row_major, int* out, int out_len)
{
  if (!out || out_len < 6) return fail(B2D_ERR_INVALID_ARG, "out must hold at least 6 words");
  bool empty = false;
  const int rc = pairwise_check(metric, dtype, x, ldx, y, ldy, dist, ldd, m, n, k, row_major, 2.0f, &empty);
  if (rc) return rc;
  for (int i = 0; i < out_len; ++i) out[i] = 0;
  if (empty) { out[0] = B2D_PLAN_NONE; return B2D_OK; }
  if (dtype == B2D_F64) { out[0] = B2D_PLAN_F64_SIMT; return B2D_OK; }
  const PairwiseOperands o = pairwise_operands(x, ldx, y, ldy, m, n, row_major);
  if (is_expanded(metric)) {
    const TcStorePlan pl = tc_store_plan(pairwise_tc_store(metric, k).post, o.ma, o.na, k, reinterpret_cast<uintptr_t>(dist), ldd);
    out[0] = B2D_PLAN_TENSOR; out[1] = pl.tma_store; out[2] = pl.vec2; out[5] = pl.launches;
    for (int i = 0; i < pl.launches && 6 + 4 * i + 3 < out_len; ++i) {
      const TcStoreLaunch l = tc_store_launch(pl, i);
      out[6 + 4 * i] = l.kb0; out[7 + 4 * i] = l.nkb; out[8 + 4 * i] = l.acc_mode; out[9 + 4 * i] = l.resident;
    }
    return B2D_OK;
  }
  const UxPlan ux = ux_plan(o.xrs, o.xcs, reinterpret_cast<uintptr_t>(o.xa), o.yrs, o.ycs, reinterpret_cast<uintptr_t>(o.ya), k);
  out[0] = ux.tma ? B2D_PLAN_F32_TMA : B2D_PLAN_F32_SIMT; out[3] = ux.vec_x; out[4] = ux.vec_y;
  out[5] = 1;
  return B2D_OK;
}

int b2d_pairwise_distance(void* stream, int metric, int dtype, const void* x, int64_t ldx, const void* y,
                          int64_t ldy, void* dist_v, int64_t ldd, int64_t m, int64_t n, int64_t k,
                          int row_major, float metric_arg, void* workspace, size_t workspace_bytes)
{
  float* dist = static_cast<float*>(dist_v);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  bool empty = false;
  int rc = pairwise_check(metric, dtype, x, ldx, y, ldy, dist_v, ldd, m, n, k, row_major, metric_arg, &empty);
  if (rc || empty) return rc;
  if (dtype == B2D_F64) {   // double in / double out: the SIMT fp64 path, every metric
    if (row_major)
      return pairwise_f64(s, metric, static_cast<const double*>(x), ldx, 1, static_cast<const double*>(y), ldy, 1,
                          static_cast<double*>(dist_v), ldd, m, n, k, 0, metric_arg, workspace, workspace_bytes);
    return pairwise_f64(s, metric, static_cast<const double*>(y), 1, ldy, static_cast<const double*>(x), 1, ldx,
                        static_cast<double*>(dist_v), ldd, n, m, k, 1, metric_arg, workspace, workspace_bytes);
  }
  const PairwiseOperands o = pairwise_operands(x, ldx, y, ldy, m, n, row_major);
  if (is_expanded(metric))
    return tc_store(s, pairwise_tc_store(metric, k), dtype, o.xa, o.xrs, o.xcs, o.ma, o.ya, o.yrs, o.ycs, o.na, k, dist, ldd,
                    x == y && m == n && ldx == ldy, workspace, workspace_bytes);

  UxParams p;
  memset(&p, 0, sizeof(p));
  p.x = static_cast<const float*>(o.xa); p.y = static_cast<const float*>(o.ya); p.dist = dist;
  p.xrs = o.xrs; p.xcs = o.xcs; p.yrs = o.yrs; p.ycs = o.ycs; p.ldd = ldd; p.m = o.ma; p.n = o.na; p.k = static_cast<int>(k);
  const UxPlan ux = ux_plan(o.xrs, o.xcs, reinterpret_cast<uintptr_t>(o.xa), o.yrs, o.ycs, reinterpret_cast<uintptr_t>(o.ya), k);
  p.vec_x = ux.vec_x; p.vec_y = ux.vec_y;
  p.p = metric_arg; p.inv_p = metric == B2D_HammingUnexpanded ? 1.f / static_cast<float>(k) : 1.f / metric_arg;
  p.tiles_n = static_cast<int>((o.na + UX_BN - 1) / UX_BN);
  const int64_t tiles = ((o.ma + UX_BM - 1) / UX_BM) * p.tiles_n;
  int sms = 0;
  rc      = device_sms(&sms);
  if (rc) return rc;
  switch (metric) {
    case B2D_L1: return launch_ux_inst<UX_L1>(s, p, tiles, ux.tma);
    case B2D_L2Unexpanded: return launch_ux_inst<UX_L2>(s, p, tiles, ux.tma);
    case B2D_L2SqrtUnexpanded: return launch_ux_inst<UX_L2SQRT>(s, p, tiles, ux.tma);
    case B2D_Linf: return launch_ux_inst<UX_LINF>(s, p, tiles, ux.tma);
    case B2D_Canberra: return launch_ux_inst<UX_CANBERRA>(s, p, tiles, ux.tma);
    case B2D_HammingUnexpanded: return launch_ux_inst<UX_HAMMING>(s, p, tiles, ux.tma);
    case B2D_KLDivergence:
      return row_major ? launch_ux_inst<UX_KL>(s, p, tiles, ux.tma) : launch_ux_inst<UX_KL_REV>(s, p, tiles, ux.tma);
    case B2D_JensenShannon: return launch_ux_inst<UX_JS>(s, p, tiles, ux.tma);
    case B2D_BrayCurtis: return launch_ux_inst<UX_BRAYCURTIS>(s, p, tiles, ux.tma);
    default: return launch_ux_inst<UX_LP>(s, p, tiles, ux.tma);
  }
}

size_t b2d_fused_l2_nn_workspace_bytes(int64_t m, int64_t n, int64_t k)
{
  if (m < 0 || n < 0 || k < 0) return static_cast<size_t>(-1);
  return tc_layout(nullptr, m, n, k, true).bytes;
}

// one chunk of y (prep + search); keys carry the result so far (and act as the rows' bounds)
static int fused_nn_keys_chunk(cudaStream_t s, int64_t* keys, const float* x, int64_t ldx, const float* y, int64_t ldy,
                               const float* xn, const float* yn, int64_t m, int64_t n, int64_t k, int64_t idx_offset,
                               void* workspace, int mode, int center, bool allow_screen, bool have_bounds)
{
  TcWorkspace w = tc_layout(workspace, m, n, k, true);
  const int nkb = static_cast<int>((k + 31) / 32);
  // (k <= 64: the exact kernel is already epilogue-bound, screening would not pay)
  const bool screen = (mode == PREP_L2 || mode == PREP_COSINE) && nkb >= 3 && nkb <= TC_MAX_RES_KB && n >= 16384 && allow_screen;
  const int unit_norm = mode == PREP_COSINE ? 1 : 0;
  // The coarse pass bounds a whole 32-column group at once: c * max_j(acc_ij) + min_j |y_j|^2 (screen_tc.cuh).  That is
  // only tight when the rows of a group have nearly equal norms, so the L2 search packs the chunk in the order of
  // its squared row norms (stable radix sort on the top 24 bits of the fp32 norm: deterministic); the kernels
  // translate a packed position back to the source row where an index leaves them (col_map).  The cosine family
  // needs none of this: its column term is the constant 0.
  const int* col_map = nullptr;
  if (screen && !unit_norm && n > 0) {
    if (n > kNnChunkRows) return fail(B2D_ERR_INVALID_ARG, "internal: screened chunk larger than 2^20 rows");
    nn_sortkey_kernel<<<static_cast<unsigned>((n + 7) / 8), 256, 0, s>>>(y, ldy, n, static_cast<int>(k), yn, w.sort_key[0], w.sort_val[0]);
    B2D_CUDA(cudaGetLastError());
    cub::DoubleBuffer<unsigned> dk(w.sort_key[0], w.sort_key[1]);
    cub::DoubleBuffer<int> dv(w.sort_val[0], w.sort_val[1]);
    size_t tmp_need = 0;
    B2D_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_need, dk, dv, static_cast<int>(n), 8, 32, s));
    if (tmp_need > kSortTmpBytes) return fail(B2D_ERR_WORKSPACE, "internal: radix sort scratch " + std::to_string(tmp_need) + " bytes");
    B2D_CUDA(cub::DeviceRadixSort::SortPairs(w.sort_tmp, tmp_need, dk, dv, static_cast<int>(n), 8, 32, s));
    col_map = dv.Current();
  }
  int rc = launch_prep<float>(s, w, x, ldx, 1, m, y, ldy, 1, n, k, xn, yn, mode, center, 0, 1.f, 0.f, col_map);
  if (rc) return rc;
  if (n == 0) return B2D_OK;
  TcParams p;
  memset(&p, 0, sizeof(p));
  p.m = m; p.n = n; p.keys = reinterpret_cast<long long*>(keys); p.idx_offset = idx_offset;
  p.col_map = col_map;
  if (!screen) return launch_tc(s, w, p, k, EPI_MINLOC, POST_NONE);

  // Screened search (screen_tc.cuh).  With S = 32 and r = index of a 256-row y block modulo S:
  //   A  exact arg-min kernel on the blocks r == 0            -> every row has an upper bound U_i
  //   T  coarse 1-product screen on the SAME blocks (trial)   -> the incumbent again and everything within the margin
  //      of it.  Two jobs: (1) A chooses among near-ties (1e-5 relative) with tensor arithmetic and keeps one column;
  //      the others must reach the exact re-evaluation like any candidate of the other blocks, or the result is only
  //      as good as A's arithmetic; (2) the number of candidates per row is the measure of whether screening pays:
  //      many (data whose norms dwarf the nearest-neighbour distances: the margin is relative to |x||y|) -> the
  //      remaining blocks take the exact kernel
  //   R  coarse screen on the blocks r >= 1                   (if screening pays)
  //   E  exact re-evaluation of every candidate, straight from the fp32 inputs
  //   X  exact kernel on r >= 1                               (only where candidates were dropped -- list overflow --
  //                                                            or where screening was called off)
  // Every launch after T is conditional on a device flag: no host round trip, no wrong answer.
  constexpr int kSel = 32;
  const float tau = g_nn_tau.load(std::memory_order_relaxed);
  unsigned* flags = w.cand_cnt;  // [0] slots [1] overflow [2] go_screen [3] go_exact [4] - [5] candidates after T [6] candidates
  // `have_bounds`: the keys already carry every row's best over earlier chunks / shards (a later chunk of this call, or
  // a call that continues from exchanged keys).  A sample of this chunk would add next to nothing to such a bound, so A
  // is skipped -- T and R then cover every block, and so does X if it has to run.  (Correct for ANY keys: a row
  // without a finite bound makes everything a candidate, the list overflows and X takes over; only slower.)
  p.sel_s = kSel; p.sel_lo = 0; p.sel_hi = 1;
  if (!have_bounds) {
    rc = launch_tc(s, w, p, k, EPI_MINLOC, POST_NONE);
    if (rc) return rc;
  }
  nn_seed_kernel<<<static_cast<unsigned>((m + 255) / 256), 256, 0, s>>>(reinterpret_cast<long long*>(keys), w.aux, w.xt, w.xlo,
                                                                         w.cand, flags, m, n, idx_offset);
  B2D_CUDA(cudaGetLastError());
  rc = launch_screen(s, w, m, n, k, kSel, 0, 1, flags + 1, nullptr, unit_norm, col_map);
  if (rc) return rc;
  // (tau + 1: the trial finds every row's incumbent again)
  nn_decide_kernel<<<1, 1, 0, s>>>(flags, static_cast<unsigned>(m), tau + 1.f, 1, w.nonuni);
  B2D_CUDA(cudaGetLastError());
  rc = launch_screen(s, w, m, n, k, kSel, 1, kSel, flags + 1, flags + 2, unit_norm, col_map);
  if (rc) return rc;
  nn_decide_kernel<<<1, 1, 0, s>>>(flags, static_cast<unsigned>(m), tau, 2, w.nonuni);
  B2D_CUDA(cudaGetLastError());
  int sms = 0;
  rc = device_sms(&sms);
  if (rc) return rc;
  nn_exact_kernel<<<sms * 8, 256, 0, s>>>(reinterpret_cast<long long*>(keys), w.cand, w.cand_cnt, w.cand_cap, x, ldx, y,
                                          ldy, static_cast<int>(k), idx_offset, unit_norm, center, static_cast<unsigned>(m), col_map);
  B2D_CUDA(cudaGetLastError());
  p.sel_lo = have_bounds ? 0 : 1; p.sel_hi = kSel; p.run_flag = flags + 3;
  rc = launch_tc(s, w, p, k, EPI_MINLOC, POST_NONE);
  if (rc) return rc;
  return B2D_OK;
}

static int fused_nn_keys(void* stream, int64_t* keys, const float* x, int64_t ldx, const float* y, int64_t ldy,
                         const float* xn, const float* yn, int64_t m, int64_t n, int64_t k, int64_t idx_offset,
                         int init_keys, void* workspace, size_t workspace_bytes, int mode, int center)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (m < 0 || n < 0 || k < 0) return fail(B2D_ERR_INVALID_ARG, "negative extent");
  if (m == 0) return B2D_OK;
  if (k == 0) return fail(B2D_ERR_INVALID_ARG, "k must be positive");
  if (!keys || !x || (n > 0 && !y)) return fail(B2D_ERR_INVALID_ARG, "null keys / x / y");
  if (ldx < k || ldy < k) return fail(B2D_ERR_INVALID_ARG, "leading dimension smaller than k");
  if (n + idx_offset > 0xFFFFFFFFll || idx_offset < 0) return fail(B2D_ERR_INVALID_ARG, "index range exceeds 32 bits");
  const int rc = check_workspace(workspace, workspace_bytes, tc_layout(nullptr, m, n, k, true).bytes);
  if (rc) return rc;
  const bool screen_off = g_nn_screen.load(std::memory_order_relaxed) == 0;
  if (init_keys) {
    minloc_init_kernel<<<static_cast<unsigned>((m + 255) / 256), 256, 0, s>>>(reinterpret_cast<long long*>(keys), m);
    B2D_CUDA(cudaGetLastError());
  }
  // The screened search (below) works through y in chunks of 2^20 rows: the candidate list is sized per
  // chunk, and every chunk starts from the bounds the earlier ones left in the keys.
  const int nkb_all    = static_cast<int>((k + 31) / 32);
  const bool screen_ok = (mode == PREP_L2 || mode == PREP_COSINE) && nkb_all >= 3 && nkb_all <= TC_MAX_RES_KB && !screen_off;
  constexpr int64_t kChunkRows = kNnChunkRows;
  if (!screen_ok || n <= kChunkRows)
    return fused_nn_keys_chunk(s, keys, x, ldx, y, ldy, xn, yn, m, n, k, idx_offset, workspace, mode, center, screen_ok,
                               init_keys == 0);
  for (int64_t off = 0; off < n; off += kChunkRows) {
    const int64_t nc = std::min<int64_t>(kChunkRows, n - off);
    int rc = fused_nn_keys_chunk(s, keys, x, ldx, y + off * ldy, ldy, xn, yn ? yn + off : nullptr, m, nc, k,
                                 idx_offset + off, workspace, mode, center, true, init_keys == 0 || off > 0);
    if (rc) return rc;
  }
  return B2D_OK;
}

int b2d_fused_l2_nn_keys(void* stream, int64_t* keys, const float* x, int64_t ldx, const float* y, int64_t ldy,
                         const float* xn, const float* yn, int64_t m, int64_t n, int64_t k, int64_t idx_offset,
                         int init_keys, void* workspace, size_t workspace_bytes)
{
  return fused_nn_keys(stream, keys, x, ldx, y, ldy, xn, yn, m, n, k, idx_offset, init_keys, workspace,
                       workspace_bytes, PREP_L2, 0);
}

int b2d_fused_l2_nn_finalize(void* stream, b2d_kvp_if* out, const int64_t* keys, int64_t m, int do_sqrt,
                             const void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (m < 0) return fail(B2D_ERR_INVALID_ARG, "negative extent");
  if (m == 0) return B2D_OK;
  if (!out || !keys || !workspace) return fail(B2D_ERR_INVALID_ARG, "null out / keys / workspace");
  if (workspace_bytes < 1024 + static_cast<size_t>(m) * 4) return fail(B2D_ERR_WORKSPACE, "workspace too small");
  // (the keys hold the full distance, so nothing is read back from the workspace any more; the argument stays
  // for ABI stability)
  minloc_finalize_kernel<<<static_cast<unsigned>((m + 255) / 256), 256, 0, s>>>(
    reinterpret_cast<KvpIF*>(out), reinterpret_cast<const long long*>(keys), m, do_sqrt, 0);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

// fusedL2NN and fusedDistanceNN: the keys of every row in the workspace, then unpacked into out.  (The cosine family,
// mode PREP_COSINE: rows are normalised in prep, keys hold -cos, the row term t_x = 1 turns it into 1 - cos.)
static int fused_nn(void* stream, b2d_kvp_if* out, const float* x, int64_t ldx, const float* y, int64_t ldy,
                    const float* xn, const float* yn, int64_t m, int64_t n, int64_t k, int mode, int center, int do_sqrt,
                    int init_out, void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (m < 0 || n < 0 || k < 0) return fail(B2D_ERR_INVALID_ARG, "negative extent");
  if (m == 0) return B2D_OK;
  if (!out) return fail(B2D_ERR_INVALID_ARG, "null out");
  // (the alignment is checked by fused_nn_keys, after the rest of its arguments)
  int rc = check_workspace(workspace, workspace_bytes, tc_layout(nullptr, m, n, k, true).bytes, 1);
  if (rc) return rc;
  TcWorkspace w = tc_layout(workspace, m, n, k, true);
  rc = fused_nn_keys(stream, reinterpret_cast<int64_t*>(w.keys), x, ldx, y, ldy, xn, yn, m, n, k, 0, 1, workspace,
                     workspace_bytes, mode, center);
  if (rc) return rc;
  minloc_finalize_kernel<<<static_cast<unsigned>((m + 255) / 256), 256, 0, s>>>(
    reinterpret_cast<KvpIF*>(out), w.keys, m, do_sqrt, init_out ? 0 : 1);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

int b2d_fused_l2_nn(void* stream, b2d_kvp_if* out, const float* x, int64_t ldx, const float* y, int64_t ldy,
                    const float* xn, const float* yn, int64_t m, int64_t n, int64_t k, int do_sqrt, int init_out,
                    void* workspace, size_t workspace_bytes)
{
  return fused_nn(stream, out, x, ldx, y, ldy, xn, yn, m, n, k, PREP_L2, 0, do_sqrt, init_out, workspace, workspace_bytes);
}

// ------------------------------------------------------------------------------------------
// Single-process multi-GPU fusedL2NN (SURVEY.md 8(e)): the reference's SNMG pattern -- one ncclComm_t per device,
// created by the caller with a grouped ncclCommInitRank / ncclCommInitAll
// (cpp/include/raft/core/resource/nccl_comm.hpp:43-62, core/device_resources_snmg.hpp:35-154).  NCCL is resolved at
// run time (dlopen of the libnccl.so.2 the process already uses), so the library has no link-time NCCL dependency.
namespace {
struct NcclApi {
  int (*all_reduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  int (*group_start)()                                                          = nullptr;
  int (*group_end)()                                                            = nullptr;
  const char* (*err_string)(int)                                                = nullptr;
  bool ok                                                                       = false;
};
const NcclApi& nccl_api()
{
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return;
    api.all_reduce  = reinterpret_cast<decltype(api.all_reduce)>(dlsym(h, "ncclAllReduce"));
    api.group_start = reinterpret_cast<decltype(api.group_start)>(dlsym(h, "ncclGroupStart"));
    api.group_end   = reinterpret_cast<decltype(api.group_end)>(dlsym(h, "ncclGroupEnd"));
    api.err_string  = reinterpret_cast<decltype(api.err_string)>(dlsym(h, "ncclGetErrorString"));
    api.ok          = api.all_reduce && api.group_start && api.group_end;
  });
  return api;
}
constexpr int kNcclInt64 = 4, kNcclMin = 3;  // ncclInt64 / ncclMin of nccl.h (stable ABI values since NCCL 2.0)
constexpr int64_t kShardHeadRows = 1 << 15;
}  // namespace

int b2d_fused_l2_nn_multi(int ngpu, const int* devices, void* const* streams, void* const* comms, b2d_kvp_if* const* out,
                          const float* const* x, int64_t ldx, const float* const* y, int64_t ldy, const int64_t* n_shard,
                          const int64_t* idx_offset, int64_t m, int64_t k, int do_sqrt, int64_t* const* keys,
                          void* const* workspace, const size_t* workspace_bytes)
{
  if (ngpu < 1 || ngpu > 64) return fail(B2D_ERR_INVALID_ARG, "ngpu must be in [1, 64]");
  if (!devices || !streams || !out || !x || !y || !n_shard || !idx_offset || !keys || !workspace || !workspace_bytes)
    return fail(B2D_ERR_INVALID_ARG, "null argument array");
  if (ngpu > 1 && !comms) return fail(B2D_ERR_INVALID_ARG, "null comms");
  const NcclApi& nccl = nccl_api();
  if (ngpu > 1 && !nccl.ok) return fail(B2D_ERR_CUDA, "NCCL (libnccl.so.2) could not be loaded");
  int prev = 0;
  B2D_CUDA(cudaGetDevice(&prev));
  // exchange plan: identical on every device (it depends on the SMALLEST shard): a 32768-row head, then sub-chunks
  // growing x4, one all-reduce of the packed keys after each (raft_b200/distance/fused_l2_nn.py: plan_exchanges)
  int64_t smin = n_shard[0];
  for (int g = 1; g < ngpu; ++g) smin = std::min(smin, n_shard[g]);
  std::vector<int64_t> plan;
  if (ngpu > 1 && smin > 0) {
    int64_t left = smin, step = kShardHeadRows;
    while (left > 4 * step && plan.size() < 3) { plan.push_back(step); left -= step; step *= 4; }
    plan.push_back(left);
  } else {
    plan.push_back(smin);
  }
  std::vector<int64_t> done(ngpu, 0);
  int rc = B2D_OK;
  for (size_t c = 0; c < plan.size() && rc == B2D_OK; ++c) {
    const bool last = c + 1 == plan.size();
    for (int g = 0; g < ngpu && rc == B2D_OK; ++g) {
      if (cudaSetDevice(devices[g]) != cudaSuccess) { rc = fail(B2D_ERR_CUDA, "cudaSetDevice failed"); break; }
      const int64_t rows = last ? n_shard[g] - done[g] : std::min(plan[c], n_shard[g] - done[g]);
      rc = b2d_fused_l2_nn_keys(streams[g], keys[g], x[g], ldx, y[g] + done[g] * ldy, ldy, nullptr, nullptr, m, rows, k,
                                idx_offset[g] + done[g], c == 0 ? 1 : 0, workspace[g], workspace_bytes[g]);
      done[g] += rows;
    }
    if (rc == B2D_OK && ngpu > 1) {
      int st = nccl.group_start();
      for (int g = 0; g < ngpu && st == 0; ++g)
        st = nccl.all_reduce(keys[g], keys[g], static_cast<size_t>(m), kNcclInt64, kNcclMin, comms[g],
                             static_cast<cudaStream_t>(streams[g]));
      const int st2 = nccl.group_end();
      if (st == 0) st = st2;
      if (st != 0) rc = fail(B2D_ERR_CUDA, std::string("ncclAllReduce(int64, min): ") + (nccl.err_string ? nccl.err_string(st) : "error"));
    }
  }
  for (int g = 0; g < ngpu && rc == B2D_OK; ++g) {
    if (cudaSetDevice(devices[g]) != cudaSuccess) { rc = fail(B2D_ERR_CUDA, "cudaSetDevice failed"); break; }
    rc = b2d_fused_l2_nn_finalize(streams[g], out[g], keys[g], m, do_sqrt, workspace[g], workspace_bytes[g]);
  }
  cudaSetDevice(prev);
  return rc;
}

int b2d_fused_distance_nn(void* stream, b2d_kvp_if* out, int metric, const float* x, int64_t ldx, const float* y,
                          int64_t ldy, const float* xn, const float* yn, int64_t m, int64_t n, int64_t k, int init_out,
                          void* workspace, size_t workspace_bytes)
{
  if (metric == B2D_L2Expanded || metric == B2D_L2SqrtExpanded)
    return b2d_fused_l2_nn(stream, out, x, ldx, y, ldy, xn, yn, m, n, k, metric == B2D_L2SqrtExpanded ? 1 : 0, init_out,
                           workspace, workspace_bytes);
  if (metric != B2D_CosineExpanded && metric != B2D_CorrelationExpanded)
    return fail(B2D_ERR_UNSUPPORTED, "fusedDistanceNN supports L2Expanded, L2SqrtExpanded, CosineExpanded, CorrelationExpanded");
  return fused_nn(stream, out, x, ldx, y, ldy, nullptr, nullptr, m, n, k, PREP_COSINE,
                  metric == B2D_CorrelationExpanded ? 1 : 0, 0, init_out, workspace, workspace_bytes);
}

// ------------------------------------------------------------------------------------------
// Masked fusedL2NN (masked_nn.cuh): the operands of the tensor-core path (without the screened search's scratch), then
// the keys and the mask's device tables
namespace {
struct MaskedLayout {
  TcWorkspace w;      // w.keys: [m]
  unsigned* bad;      // [1] group_idxs is invalid
  int* grp;           // [n] group of every row of y
  unsigned* bits;     // [ceil(m/32)][G] adjacency bits
  uint8_t* cls;       // [tiles_n][tiles_m] tile classes
  size_t bytes;
};
}  // namespace

static MaskedLayout masked_layout(void* base, int64_t m, int64_t n, int64_t k, int64_t G)
{
  Carve c(base, 1024);
  MaskedLayout L;
  L.w      = tc_layout(c, m, n, k, false);
  L.w.keys = c.take<long long>(m);
  L.bad    = c.take<unsigned>(8);
  L.grp    = c.take<int>(n);
  L.bits   = c.take<unsigned>(static_cast<size_t>((m + 31) / 32) * G);
  L.cls    = c.take<uint8_t>(static_cast<size_t>((m + TC_BM - 1) / TC_BM) * ((n + TC_BN - 1) / TC_BN));
  L.bytes  = c.bytes;
  return L;
}

// The masked arg-min of the prepared x rows (w's x side) against the prepared y rows into keys (KEY_EMPTY or earlier
// minima on entry), for a valid group_idxs whose group map of y is grp: adjacency bits, tile classes, the
// EPI_MINLOC_MASKED launch
static int masked_keys(cudaStream_t s, const TcWorkspace& w, long long* keys, const int* grp, unsigned* bits, uint8_t* cls,
                       const unsigned* bad, const uint8_t* adj, int64_t ld_adj, const int32_t* group_idxs, int64_t G,
                       int64_t m, int64_t n, int64_t k)
{
  masked_adj_bits_kernel<<<static_cast<unsigned>((m + 31) / 32), 256, 0, s>>>(bits, adj, ld_adj, m, G);
  B2D_CUDA(cudaGetLastError());
  const int tiles_m = static_cast<int>((m + TC_BM - 1) / TC_BM), tiles_n = static_cast<int>((n + TC_BN - 1) / TC_BN);
  const int64_t ntiles = static_cast<int64_t>(tiles_m) * tiles_n;
  masked_classify_kernel<<<static_cast<unsigned>((ntiles + 255) / 256), 256, 0, s>>>(cls, bits, group_idxs, G, m, n,
                                                                                     tiles_m, tiles_n, bad);
  B2D_CUDA(cudaGetLastError());
  TcParams p;
  memset(&p, 0, sizeof(p));
  p.m = m; p.n = n; p.keys = keys;
  p.mask_cls = cls; p.mask_grp = grp; p.mask_bits = bits; p.mask_groups = G;
  ProfileScope prof(s);
  return launch_tc(s, w, p, k, EPI_MINLOC_MASKED, POST_NONE);
}

size_t b2d_masked_l2_nn_workspace_bytes(int64_t m, int64_t n, int64_t k, int64_t num_groups)
{
  if (m < 0 || n < 0 || k < 0 || num_groups < 0) return static_cast<size_t>(-1);
  return masked_layout(nullptr, m, n, k, num_groups).bytes;
}

int b2d_masked_l2_nn(void* stream, b2d_kvp_if* out, const float* x, int64_t ldx, const float* y, int64_t ldy,
                     const float* xn, const float* yn, const uint8_t* adj, int64_t ld_adj, const int32_t* group_idxs,
                     int64_t num_groups, int64_t m, int64_t n, int64_t k, int do_sqrt, int init_out, void* workspace,
                     size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int64_t G = num_groups;
  if (m < 0 || n < 0 || k < 0 || G < 0) return fail(B2D_ERR_INVALID_ARG, "negative extent");
  if (m == 0) return B2D_OK;
  if (k == 0) return fail(B2D_ERR_INVALID_ARG, "k must be positive");
  if (!out || !x || (n > 0 && !y)) return fail(B2D_ERR_INVALID_ARG, "null out / x / y");
  if (G > 0 && (!adj || !group_idxs)) return fail(B2D_ERR_INVALID_ARG, "null adj / group_idxs");
  if (ld_adj < G) return fail(B2D_ERR_INVALID_ARG, "ld_adj smaller than num_groups");
  if (ldx < k || ldy < k) return fail(B2D_ERR_INVALID_ARG, "leading dimension smaller than k");
  if (m > 0x7fffffffll || n > 0x7fffffffll || G > 0x7fffffffll) return fail(B2D_ERR_INVALID_ARG, "index range exceeds 32 bits");
  int rc = check_workspace(workspace, workspace_bytes, masked_layout(nullptr, m, n, k, G).bytes);
  if (rc) return rc;
  MaskedLayout L = masked_layout(workspace, m, n, k, G);
  const unsigned mblocks = static_cast<unsigned>((m + 255) / 256);
  minloc_init_kernel<<<mblocks, 256, 0, s>>>(L.w.keys, m);
  B2D_CUDA(cudaGetLastError());
  masked_validate_kernel<<<1, 1024, 0, s>>>(L.bad, group_idxs, G, n);
  B2D_CUDA(cudaGetLastError());
  if (n > 0 && G > 0) {
    rc = launch_prep<float>(s, L.w, x, ldx, 1, m, y, ldy, 1, n, k, xn, yn, PREP_L2, 0);
    if (rc) return rc;
    masked_group_map_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, s>>>(L.grp, group_idxs, G, n);
    B2D_CUDA(cudaGetLastError());
    rc = masked_keys(s, L.w, L.w.keys, L.grp, L.bits, L.cls, L.bad, adj, ld_adj, group_idxs, G, m, n, k);
    if (rc) return rc;
  }
  minloc_finalize_kernel<<<mblocks, 256, 0, s>>>(reinterpret_cast<KvpIF*>(out), L.w.keys, m, do_sqrt, init_out ? 0 : 1);
  B2D_CUDA(cudaGetLastError());
  masked_poison_kernel<<<mblocks, 256, 0, s>>>(reinterpret_cast<KvpIF*>(out), L.bad, m);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

// ------------------------------------------------------------------------------------------
// Fused brute-force kNN (SURVEY.md 8(f2)): raft::neighbors::brute_force::knn / fused_l2_knn for the
// L2 metrics without ever writing the m x n matrix (expanded_tc.cuh, EPI_TOPK).

// The tensor-core workspace with keys, then the kNN's own regions.  Two regions of the tensor workspace are borrowed:
// thr and cnt live in aux ([m] floats, then [m] counters: 8 of its 16 bytes per row), and the per-row candidate lists
// (KNN_CAP entries of 8 bytes per row) in cand, which b2d_knn guards with m * KNN_CAP <= cand_cap.
namespace {
struct KnnLayout {
  TcWorkspace w;
  long long* topk;      // [m][n_neighbors]
  float* thr;           // [m]
  unsigned* cnt;        // [m]
  long long* dropmin;   // [m] best key that did not fit into a row's list this pass
  int* dirty;           // [m] rows to redo for the current pass
  unsigned* repaired;   // [m] 1 once a row has been repaired in some pass
  int* rep_list;        // [m] the repaired rows ...
  unsigned* dirty_cnt;  // [64] one counter per pass
  unsigned* rep_cnt;    // [1] ... and their count, right behind dirty_cnt
  size_t bytes;
};
}  // namespace

static KnnLayout knn_layout(void* base, int64_t m, int64_t n, int64_t k, int64_t n_neighbors)
{
  Carve c(base, 1024);
  KnnLayout L;
  L.w         = tc_layout(c, m, n, k, true);
  L.thr       = reinterpret_cast<float*>(L.w.aux);
  L.cnt       = L.w.aux ? reinterpret_cast<unsigned*>(L.w.aux) + m : nullptr;
  L.topk      = c.take<long long>(static_cast<size_t>(m) * n_neighbors);
  L.dropmin   = c.take<long long>(m);
  L.dirty     = c.take<int>(m);
  L.repaired  = c.take<unsigned>(m);
  L.rep_list  = c.take<int>(m);
  L.dirty_cnt = c.take<unsigned>(65);
  L.rep_cnt   = L.dirty_cnt ? L.dirty_cnt + 64 : nullptr;
  L.bytes     = c.bytes;
  return L;
}

size_t b2d_knn_l2_workspace_bytes(int64_t m, int64_t n, int64_t k, int64_t n_neighbors)
{
  if (m < 0 || n < 0 || k < 0 || n_neighbors < 1 || n_neighbors > KNN_MAX_K) return static_cast<size_t>(-1);
  return knn_layout(nullptr, m, n, k, n_neighbors).bytes;
}

namespace {
struct KnnCtx {
  cudaStream_t s;
  KnnLayout L;
  TcParams p;       // m, knn_* set; n / idx_offset per pass
  int64_t k;
  bool any_fix;         // a knn_fix_kernel was launched
  int pass;
  const float* x; int64_t ldx;
  const float* y; int64_t ldy;
  int family, center;
  int kk;
};
}  // namespace

// one pass over y rows [off, off + width): append, fold into the top-k, redo the rows whose lists overflowed in a way
// that matters (knn_merge_kernel / knn_fix_kernel) -- all on the device: the call only enqueues work
static int knn_pass(KnnCtx& c, int64_t off, int64_t width)
{
  const KnnLayout& L = c.L;
  TcWorkspace w2 = tc_rows(L.w, 1, off, c.k);
  TcParams p     = c.p;
  p.n            = width;
  p.idx_offset   = off;
  int rc         = launch_tc(c.s, w2, p, c.k, EPI_TOPK, POST_NONE);
  if (rc) return rc;
  unsigned* dc = L.dirty_cnt + (c.pass & 63);
  knn_merge_kernel<<<static_cast<unsigned>((c.p.m + 7) / 8), 256, 0, c.s>>>(L.topk, c.p.knn_cand, L.cnt, L.thr, L.dropmin, L.dirty,
                                                                            dc, L.repaired, L.rep_list, L.rep_cnt, c.p.m, c.kk);
  B2D_CUDA(cudaGetLastError());
  if (width > KNN_CAP) {  // (a pass of at most KNN_CAP columns cannot overflow)
    int sms = 0;
    rc = device_sms(&sms);
    if (rc) return rc;
    knn_fix_kernel<<<sms * 2, 256, 0, c.s>>>(L.topk, L.thr, L.dirty, dc, c.x, c.ldx, c.y, c.ldy, static_cast<int>(c.k), c.kk, off,
                                             width, c.family, c.center);
    B2D_CUDA(cudaGetLastError());
    c.any_fix = true;
  }
  ++c.pass;
  return B2D_OK;
}

int b2d_knn_l2(void* stream, int64_t* out_idx, float* out_dist, const float* x, int64_t ldx, const float* y,
               int64_t ldy, int64_t m, int64_t n, int64_t k, int64_t n_neighbors, int do_sqrt, void* workspace,
               size_t workspace_bytes)
{
  return b2d_knn(stream, out_idx, out_dist, do_sqrt ? B2D_L2SqrtExpanded : B2D_L2Expanded, x, ldx, y, ldy, m, n, k,
                 n_neighbors, workspace, workspace_bytes);
}

int b2d_knn(void* stream, int64_t* out_idx, float* out_dist, int metric, const float* x, int64_t ldx, const float* y,
            int64_t ldy, int64_t m, int64_t n, int64_t k, int64_t n_neighbors, void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  int mode = PREP_L2, center = 0, do_sqrt = 0;
  if (metric == B2D_L2Expanded || metric == B2D_L2Unexpanded) {}
  else if (metric == B2D_L2SqrtExpanded || metric == B2D_L2SqrtUnexpanded) do_sqrt = 1;
  else if (metric == B2D_CosineExpanded) mode = PREP_COSINE;
  else if (metric == B2D_CorrelationExpanded) { mode = PREP_COSINE; center = 1; }
  else return fail(B2D_ERR_UNSUPPORTED, "kNN supports the L2 metrics, CosineExpanded and CorrelationExpanded");
  if (m < 0 || n < 0 || k < 0) return fail(B2D_ERR_INVALID_ARG, "negative extent");
  if (n_neighbors < 1 || n_neighbors > n) return fail(B2D_ERR_INVALID_ARG, "n_neighbors must be in [1, n]");
  if (n_neighbors > KNN_MAX_K) return fail(B2D_ERR_UNSUPPORTED, "n_neighbors > 64 is not supported");
  if (m == 0) return B2D_OK;
  if (k == 0) return fail(B2D_ERR_INVALID_ARG, "k must be positive");
  if (k > 320) return fail(B2D_ERR_UNSUPPORTED, "kNN supports k <= 320 (see DESIGN.md section 3)");
  if (!out_idx || !out_dist || !x || !y) return fail(B2D_ERR_INVALID_ARG, "null out / x / y");
  if (ldx < k || ldy < k) return fail(B2D_ERR_INVALID_ARG, "leading dimension smaller than k");
  if (n > 0xFFFFFFFFll) return fail(B2D_ERR_INVALID_ARG, "index range exceeds 32 bits");
  const KnnLayout need = knn_layout(nullptr, m, n, k, n_neighbors);
  if (m * static_cast<int64_t>(KNN_CAP) > need.w.cand_cap)
    return fail(B2D_ERR_UNSUPPORTED, "kNN: too many query rows for one call (m * 128 must stay below 2^31): split the queries");
  int rc = check_workspace(workspace, workspace_bytes, need.bytes);
  if (rc) return rc;
  KnnCtx c;
  c.s   = s;
  c.L   = knn_layout(workspace, m, n, k, n_neighbors);
  c.k   = k;
  c.kk  = static_cast<int>(n_neighbors);
  c.pass = 0; c.any_fix = false; c.x = x; c.ldx = ldx; c.y = y; c.ldy = ldy;
  c.family = mode == PREP_COSINE ? 1 : 0; c.center = center;
  const KnnLayout& L = c.L;
  rc = launch_prep<float>(s, L.w, x, ldx, 1, m, y, ldy, 1, n, k, nullptr, nullptr, mode, center);
  if (rc) return rc;
  const int64_t total = m * n_neighbors;
  knn_init_kernel<<<static_cast<unsigned>((std::max<int64_t>(std::max<int64_t>(total, m), 65) + 255) / 256), 256, 0, s>>>(L.topk, L.thr, L.cnt, L.dropmin, L.dirty_cnt, L.repaired, m, c.kk);
  B2D_CUDA(cudaGetLastError());
  memset(&c.p, 0, sizeof(c.p));
  c.p.m = m;
  c.p.knn_thr = L.thr; c.p.knn_cnt = L.cnt; c.p.knn_cand = reinterpret_cast<long long*>(L.w.cand);
  c.p.knn_cap = KNN_CAP; c.p.knn_dropmin = L.dropmin;
  // pass widths KNN_CAP, KNN_CAP, 2 KNN_CAP, 4 KNN_CAP, ...: with the k-th best of the s columns seen so far as
  // threshold, a pass over the next s columns appends ~n_neighbors entries per row on unordered data
  int64_t off = 0;
  while (off < n) {
    const int64_t width = std::min<int64_t>(off == 0 ? KNN_CAP : off, n - off);
    rc = knn_pass(c, off, width);
    if (rc) return rc;
    off += width;
  }
  if (c.any_fix) {  // every row repaired in some pass: measured again over all n columns, so one arithmetic ranks it
    int sms = 0;
    rc = device_sms(&sms);
    if (rc) return rc;
    knn_fix_kernel<<<sms * 2, 256, 0, s>>>(L.topk, L.thr, L.rep_list, L.rep_cnt, x, ldx, y, ldy, static_cast<int>(k), c.kk, 0, n,
                                           c.family, c.center);
    B2D_CUDA(cudaGetLastError());
  }
  knn_finalize_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, s>>>(out_idx, out_dist, L.topk, total, do_sqrt);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

// ------------------------------------------------------------------------------------------
// raft::stats::silhouette_score on the distance engine (SURVEY.md 8(f3); stats.cuh)

namespace {
// silhouette and trustworthiness work through the n x n distances in [chunk x n] fp32 slabs, row pitch ld: chunk is the
// caller's row count or about 1 GiB, a multiple of 128 and at most max(n, 1)
struct Slab {
  int64_t chunk, ld;
};
Slab slab_shape(int64_t n, int64_t chunk_rows)
{
  Slab sl;
  sl.ld     = (n + 3) / 4 * 4;
  int64_t c = chunk_rows > 0 ? chunk_rows : (int64_t(1) << 30) / (4 * std::max<int64_t>(sl.ld, 1));
  c         = std::max<int64_t>(128, c / 128 * 128);
  sl.chunk  = std::min<int64_t>(c, std::max<int64_t>(n, 1));
  return sl;
}

struct SilLayout {
  Slab sl;
  int *counts, *offsets, *cursor;  // zeroed together with bad and total: everything in front of where
  unsigned* bad;
  double* total;
  int* where;
  float *ys, *slab;
  void* pw;                        // b2d_pairwise_distance's workspace
  size_t pw_bytes, bytes;
};
SilLayout sil_layout(void* base, int64_t n, int64_t k, int n_labels, int metric, int64_t chunk_rows)
{
  Carve c(base, 1024);
  SilLayout L;
  L.sl       = slab_shape(n, chunk_rows);
  L.counts   = c.take<int>(n_labels);
  L.offsets  = c.take<int>(n_labels + 1);
  L.cursor   = c.take<int>(n_labels);
  L.bad      = c.take<unsigned>(1);
  L.total    = c.take<double>(1);
  L.where    = c.take<int>(n);
  L.ys       = c.take<float>(static_cast<size_t>(n) * k);
  L.slab     = c.take<float>(static_cast<size_t>(L.sl.chunk) * L.sl.ld);
  L.pw_bytes = b2d_pairwise_workspace_bytes(metric, B2D_F32, L.sl.chunk, n, k);
  L.pw       = c.take<char>(L.pw_bytes == static_cast<size_t>(-1) ? 0 : L.pw_bytes);
  L.bytes    = c.bytes;
  return L;
}
}  // namespace

size_t b2d_silhouette_score_workspace_bytes(int64_t n, int64_t k, int n_labels, int metric, int64_t chunk_rows)
{
  if (n < 0 || k < 0 || n_labels < 1 || chunk_rows < 0) return static_cast<size_t>(-1);
  if (b2d_pairwise_workspace_bytes(metric, B2D_F32, 1, 1, k) == static_cast<size_t>(-1)) return static_cast<size_t>(-1);
  return sil_layout(nullptr, n, k, n_labels, metric, chunk_rows).bytes;
}

int b2d_silhouette_score(void* stream, float* score, float* per_sample, const float* x, int64_t ldx, const int* labels,
                         int64_t n, int64_t k, int n_labels, int metric, float metric_arg, int64_t chunk_rows,
                         void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (n < 0 || k <= 0 || chunk_rows < 0) return fail(B2D_ERR_INVALID_ARG, "bad extent");
  if (!score || !x || !labels) return fail(B2D_ERR_INVALID_ARG, "null score / x / labels");
  if (n_labels < 2 || n_labels > n - 1)
    return fail(B2D_ERR_INVALID_ARG, "silhouette score is not defined for this number of labels (need 2 <= n_labels <= n - 1)");
  if (n_labels > 12000) return fail(B2D_ERR_UNSUPPORTED, "n_labels > 12000");
  if (ldx < k) return fail(B2D_ERR_INVALID_ARG, "leading dimension smaller than k");
  const size_t need = b2d_silhouette_score_workspace_bytes(n, k, n_labels, metric, chunk_rows);
  if (need == static_cast<size_t>(-1)) return fail(B2D_ERR_UNSUPPORTED, "metric " + std::to_string(metric) + " is not on the tensor-core / SIMT distance path");
  int rc = check_workspace(workspace, workspace_bytes, need);
  if (rc) return rc;
  const SilLayout L = sil_layout(workspace, n, k, n_labels, metric, chunk_rows);
  B2D_CUDA(cudaMemsetAsync(workspace, 0, reinterpret_cast<char*>(L.where) - static_cast<char*>(workspace), s));
  const unsigned nb = static_cast<unsigned>((n + 255) / 256);
  sil_count_kernel<<<nb, 256, 0, s>>>(labels, L.counts, n, n_labels, L.bad);
  sil_scan_kernel<<<1, 32, 0, s>>>(L.counts, L.offsets, L.cursor, n_labels);
  sil_gather_kernel<<<static_cast<unsigned>((n + 7) / 8), 256, 0, s>>>(x, ldx, labels, L.cursor, L.ys, L.where, n, static_cast<int>(k), n_labels);
  B2D_CUDA(cudaGetLastError());
  // labels outside [0, n_labels) are detected on the device (no host round trip: the call stays asynchronous);
  // they poison the result: *score and the per-sample values of the offending rows become NaN
  for (int64_t r0 = 0; r0 < n; r0 += L.sl.chunk) {
    const int64_t rows = std::min<int64_t>(L.sl.chunk, n - r0);
    rc = b2d_pairwise_distance(stream, metric, B2D_F32, x + r0 * ldx, ldx, L.ys, k, L.slab, L.sl.ld, rows, n, k, 1,
                               metric_arg, L.pw, L.pw_bytes);
    if (rc) return rc;
    sil_row_kernel<<<static_cast<unsigned>(rows), 256, static_cast<size_t>(n_labels) * 4, s>>>(
      L.slab, L.sl.ld, r0, rows, labels, L.counts, L.offsets, L.where, n_labels, per_sample, L.total);
    B2D_CUDA(cudaGetLastError());
  }
  sil_finish_kernel<<<1, 32, 0, s>>>(L.total, score, n, L.bad, L.counts, n_labels);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

// raft::stats::trustworthiness_score on the kNN + distance engine (stats.cuh)
namespace {
struct TrustLayout {
  Slab sl;
  unsigned long long* penalty;
  int64_t* emb_idx;
  float *emb_dist, *slab;
  void* scratch;    // the kNN's workspace, then b2d_pairwise_distance's
  size_t knn_bytes, pw_bytes, bytes;
};
TrustLayout trust_layout(void* base, int64_t n, int64_t m, int64_t d, int n_neighbors, int metric, int64_t batch_rows)
{
  Carve c(base, 1024);
  TrustLayout L;
  L.sl        = slab_shape(n, batch_rows);
  L.penalty   = c.take<unsigned long long>(1);
  L.emb_idx   = c.take<int64_t>(static_cast<size_t>(n) * (n_neighbors + 1));
  L.emb_dist  = c.take<float>(static_cast<size_t>(n) * (n_neighbors + 1));
  L.slab      = c.take<float>(static_cast<size_t>(L.sl.chunk) * L.sl.ld);
  L.knn_bytes = b2d_knn_l2_workspace_bytes(n, n, d, n_neighbors + 1);
  L.pw_bytes  = b2d_pairwise_workspace_bytes(metric, B2D_F32, L.sl.chunk, n, m);
  const size_t a = L.knn_bytes == static_cast<size_t>(-1) ? 0 : L.knn_bytes;
  const size_t b = L.pw_bytes == static_cast<size_t>(-1) ? 0 : L.pw_bytes;
  L.scratch   = c.take<char>(std::max(a, b));
  L.bytes     = c.bytes;
  return L;
}
}  // namespace

size_t b2d_trustworthiness_score_workspace_bytes(int64_t n, int64_t m, int64_t d, int n_neighbors, int metric,
                                                 int64_t batch_rows)
{
  if (n < 0 || m < 0 || d < 0 || n_neighbors < 1 || n_neighbors + 1 > KNN_MAX_K || batch_rows < 0) return static_cast<size_t>(-1);
  if (b2d_pairwise_workspace_bytes(metric, B2D_F32, 1, 1, m) == static_cast<size_t>(-1)) return static_cast<size_t>(-1);
  return trust_layout(nullptr, n, m, d, n_neighbors, metric, batch_rows).bytes;
}

int b2d_trustworthiness_score(void* stream, double* score, const float* x, int64_t ldx, const float* x_embedded,
                              int64_t lde, int64_t n, int64_t m, int64_t d, int n_neighbors, int metric,
                              int64_t batch_rows, void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (n < 0 || m <= 0 || d <= 0 || batch_rows < 0) return fail(B2D_ERR_INVALID_ARG, "bad extent");
  if (!score || !x || !x_embedded) return fail(B2D_ERR_INVALID_ARG, "null score / x / x_embedded");
  // the reference uses distance_type for BOTH spaces (trustworthiness_score<math_t, distance_type>,
  // cpp/include/raft/stats/detail/trustworthiness_score.cuh:113-211): the embedded-space neighbours come from
  // the fused kNN, which covers the L2 and the cosine families
  int knn_metric = metric;
  if (metric == B2D_L2Unexpanded) knn_metric = B2D_L2Expanded;
  if (metric == B2D_L2SqrtUnexpanded) knn_metric = B2D_L2SqrtExpanded;
  if (knn_metric != B2D_L2Expanded && knn_metric != B2D_L2SqrtExpanded && knn_metric != B2D_CosineExpanded &&
      knn_metric != B2D_CorrelationExpanded)
    return fail(B2D_ERR_UNSUPPORTED, "trustworthiness_score supports the L2 metrics, CosineExpanded and CorrelationExpanded");
  if (n_neighbors < 1 || n_neighbors + 1 > KNN_MAX_K) return fail(B2D_ERR_UNSUPPORTED, "n_neighbors must be in [1, 63]");
  if (2 * n - 3 * static_cast<int64_t>(n_neighbors) - 1 <= 0 || n_neighbors + 1 > n)
    return fail(B2D_ERR_INVALID_ARG, "n_neighbors must be smaller than n / 2");
  if (ldx < m || lde < d) return fail(B2D_ERR_INVALID_ARG, "leading dimension smaller than the row length");
  const size_t need = b2d_trustworthiness_score_workspace_bytes(n, m, d, n_neighbors, metric, batch_rows);
  if (need == static_cast<size_t>(-1)) return fail(B2D_ERR_UNSUPPORTED, "metric " + std::to_string(metric) + " is not on the tensor-core / SIMT distance path");
  int rc = check_workspace(workspace, workspace_bytes, need);
  if (rc) return rc;
  const TrustLayout L = trust_layout(workspace, n, m, d, n_neighbors, metric, batch_rows);
  const int kk1       = n_neighbors + 1;
  B2D_CUDA(cudaMemsetAsync(L.penalty, 0, 8, s));
  // neighbours in the embedded space (the sample itself included, as in the reference)
  rc = b2d_knn(stream, L.emb_idx, L.emb_dist, knn_metric, x_embedded, lde, x_embedded, lde, n, n, d, kk1, L.scratch,
               L.knn_bytes);
  if (rc) return rc;
  for (int64_t r0 = 0; r0 < n; r0 += L.sl.chunk) {
    const int64_t rows = std::min<int64_t>(L.sl.chunk, n - r0);
    rc = b2d_pairwise_distance(stream, metric, B2D_F32, x + r0 * ldx, ldx, x, ldx, L.slab, L.sl.ld, rows, n, m, 1, 2.0f,
                               L.scratch, L.pw_bytes);
    if (rc) return rc;
    trust_rank_kernel<<<static_cast<unsigned>(rows), 256, 0, s>>>(L.slab, L.sl.ld, r0, n, L.emb_idx, kk1, n_neighbors, L.penalty);
    B2D_CUDA(cudaGetLastError());
  }
  trust_finish_kernel<<<1, 1, 0, s>>>(L.penalty, score, n, n_neighbors);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

int b2d_row_argmin(void* stream, int32_t* out, const float* in, int64_t ld, int64_t rows, int64_t n)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (rows < 0 || n < 0 || ld < n) return fail(B2D_ERR_INVALID_ARG, "bad extents");
  if (n > 0x7fffffffll) return fail(B2D_ERR_INVALID_ARG, "row length exceeds 31 bits");
  if (rows == 0) return B2D_OK;
  if (!out || (!in && n > 0)) return fail(B2D_ERR_INVALID_ARG, "null out / in");
  if (n <= 2048)
    row_argmin_kernel<true><<<static_cast<unsigned>((rows + 7) / 8), 256, 0, s>>>(out, in, ld, rows, n);
  else
    row_argmin_kernel<false><<<static_cast<unsigned>(rows), 256, 0, s>>>(out, in, ld, rows, n);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

int b2d_row_norm(void* stream, float* out, const float* x, int64_t ldx, int64_t rows, int64_t k, int norm_type,
                 int do_sqrt)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (rows < 0 || k < 0 || ldx < k) return fail(B2D_ERR_INVALID_ARG, "bad extents");
  if (norm_type < B2D_L0PseudoNorm || norm_type > B2D_LinfNorm) return fail(B2D_ERR_INVALID_ARG, "norm type");
  if (rows == 0) return B2D_OK;
  if (!out || !x) return fail(B2D_ERR_INVALID_ARG, "null out / x");
  row_norm_kernel<<<static_cast<unsigned>((rows + 7) / 8), 256, 0, s>>>(out, x, ldx, rows, static_cast<int>(k),
                                                                        norm_type, do_sqrt);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

size_t b2d_select_k_workspace_bytes(int64_t rows, int64_t len, int64_t k)
{
  if (!sk_extents_ok(rows, len, k)) return SIZE_MAX;
  if (rows == 0) return 0;
  return sk_layout(nullptr, sk_plan(rows, len, k), rows, k).bytes;
}

int b2d_select_k(void* stream, const float* in_val, int64_t ld, const int64_t* in_idx, int64_t rows, int64_t len, int64_t k,
                 int select_min, float* out_val, int64_t* out_idx, void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (rows < 0 || len < 0) return fail(B2D_ERR_INVALID_ARG, "bad extents");
  if (k < 1 || k > len) return fail(B2D_ERR_INVALID_ARG, "k must be in [1, len]");
  if (len > 0x7fffffffll || rows > 0x7fffffffll) return fail(B2D_ERR_UNSUPPORTED, "rows and len must be below 2^31");
  if (ld < len) return fail(B2D_ERR_INVALID_ARG, "ld < len");
  if (rows == 0) return B2D_OK;
  if (!in_val || !out_val || !out_idx) return fail(B2D_ERR_INVALID_ARG, "null in_val / out_val / out_idx");
  const bool mn    = select_min != 0;
  const SkPlan p   = sk_plan(rows, len, k);
  const int rc      = check_workspace(workspace, workspace_bytes, sk_layout(nullptr, p, rows, k).bytes);
  if (rc) return rc;
  const SkLayout w = sk_layout(workspace, p, rows, k);
  const unsigned R = static_cast<unsigned>(rows);
  if (p.layout == SK_SORT_ROW) {
    const int threads = std::max(32, std::min(512, p.sort_n / 2));
    select_k_sort_row_kernel<<<R, threads, p.sort_n * 8, s>>>(in_val, ld, len, k, mn, in_idx, out_val, out_idx, p.sort_n);
    B2D_CUDA(cudaGetLastError());
    return B2D_OK;
  }
  if (p.layout == SK_RADIX_ROW) {
    B2D_CUDA(cudaFuncSetAttribute(select_k_radix_row_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSkRowSmem));
    select_k_radix_row_kernel<<<R, kSkThreads, kSkRowSmem, s>>>(in_val, ld, len, k, mn, in_idx, out_val, out_idx,
                                                                 p.list ? 0 : p.sort_n, p.cap, w.list);
  } else {
    B2D_CUDA(cudaMemsetAsync(w.st, 0, static_cast<size_t>(rows) * sizeof(SkState), s));
    B2D_CUDA(cudaMemsetAsync(w.hist, 0, static_cast<size_t>(rows) * kSkBuckets * 4, s));
    const dim3 grid(static_cast<unsigned>(p.chunks), R);
    for (int pass = 0; pass <= kSkPasses; ++pass) {
      select_k_split_read_kernel<<<grid, kSkThreads, 0, s>>>(in_val, ld, len, p.chunk, k, mn, w.st, w.hist, w.list, pass);
      if (pass < kSkPasses) select_k_split_scan_kernel<<<R, kSkThreads, 0, s>>>(w.st, w.hist, k, pass);
    }
  }
  B2D_CUDA(cudaGetLastError());
  if (!p.list) return B2D_OK;
  if (!p.cub) {
    select_k_sort_list_kernel<<<R, kSkThreads, p.sort_n * 8, s>>>(w.list, in_val, ld, k, in_idx, out_val, out_idx, p.sort_n);
    B2D_CUDA(cudaGetLastError());
    return B2D_OK;
  }
  select_k_offsets_kernel<<<static_cast<unsigned>((p.batch + 256) / 256), 256, 0, s>>>(w.off, p.batch, k);
  B2D_CUDA(cudaGetLastError());
  for (int64_t r0 = 0; r0 < rows; r0 += p.batch) {
    const int64_t nb = std::min(p.batch, rows - r0);
    cub::DoubleBuffer<unsigned long long> db(reinterpret_cast<unsigned long long*>(w.list + r0 * k),
                                             reinterpret_cast<unsigned long long*>(w.alt));
    size_t tmp_need = 0;
    B2D_CUDA(cub::DeviceSegmentedRadixSort::SortKeys(nullptr, tmp_need, db, static_cast<int>(nb * k), static_cast<int>(nb),
                                                     w.off, w.off + 1, 0, 64, s));
    if (tmp_need > kSkCubTmp)
      return fail(B2D_ERR_WORKSPACE, "internal: segmented sort scratch " + std::to_string(tmp_need) + " bytes");
    B2D_CUDA(cub::DeviceSegmentedRadixSort::SortKeys(w.tmp, tmp_need, db, static_cast<int>(nb * k), static_cast<int>(nb),
                                                     w.off, w.off + 1, 0, 64, s));
    select_k_gather_kernel<<<static_cast<unsigned>((nb * k + 255) / 256), 256, 0, s>>>(
      reinterpret_cast<const uint64_t*>(db.Current()), in_val, ld, k, in_idx, out_val, out_idx, r0, nb);
    B2D_CUDA(cudaGetLastError());
  }
  return B2D_OK;
}

// ------------------------------------------------------------------------------------------
// Epsilon neighbourhood (raft::neighbors::epsilon_neighborhood): the L2Expanded distance of pairwise_distance compared with
// eps in the epilogue of the tensor kernel (expanded_tc.cuh, EPI_EPS), so the m x n matrix is never written.

size_t b2d_eps_neighbors_l2sq_workspace_bytes(int64_t m, int64_t n, int64_t k)
{
  if (m < 0 || n < 0 || k < 0) return static_cast<size_t>(-1);
  return tc_layout(nullptr, m, n, k, false).bytes;
}

int b2d_eps_neighbors_l2sq(void* stream, uint8_t* adj, int64_t ld_adj, void* vd, int vd_int64, int init_vd,
                           const float* x, int64_t ldx, const float* y, int64_t ldy, int64_t m, int64_t n, int64_t k,
                           float eps, void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (m < 0 || n < 0 || k < 0) return fail(B2D_ERR_INVALID_ARG, "negative extent");
  if (!adj && !vd) return fail(B2D_ERR_INVALID_ARG, "adj and vd are both null: nothing to compute");
  if (m > 0x7fffffffll || n > 0x7fffffffll) return fail(B2D_ERR_INVALID_ARG, "m and n must be below 2^31");
  const bool work = m > 0 && n > 0;
  if (work) {
    if (k == 0) return fail(B2D_ERR_INVALID_ARG, "k must be positive");
    if (k > 320) return fail(B2D_ERR_UNSUPPORTED, "eps_neighbors_l2sq supports k <= 320 (the whole distance at once)");
    if (!x || !y) return fail(B2D_ERR_INVALID_ARG, "null x / y");
    if (adj && ld_adj < n) return fail(B2D_ERR_INVALID_ARG, "ld_adj smaller than n");
    if (ldx < k || ldy < k) return fail(B2D_ERR_INVALID_ARG, "leading dimension smaller than k");
    const int rc = check_workspace(workspace, workspace_bytes, tc_layout(nullptr, m, n, k, false).bytes);
    if (rc) return rc;
  }
  if (vd && init_vd) B2D_CUDA(cudaMemsetAsync(vd, 0, static_cast<size_t>(n + 1) * (vd_int64 ? 8 : 4), s));
  if (!work) return B2D_OK;
  TcWorkspace w = tc_layout(workspace, m, n, k, false);
  int rc = launch_prep<float>(s, w, x, ldx, 1, m, y, ldy, 1, n, k, nullptr, nullptr, PREP_L2, 0);
  if (rc) return rc;
  TcParams p;
  memset(&p, 0, sizeof(p));
  p.m = m; p.n = n;
  p.adj = adj; p.ld_adj = ld_adj; p.vd = vd; p.vd64 = vd_int64 ? 1 : 0; p.eps = eps;
  // y is a window of x's rows (same memory, same pitch): row j of y is row j + off of x
  p.diag_off = TC_NO_DIAG;
  const intptr_t dy = reinterpret_cast<intptr_t>(y) - reinterpret_cast<intptr_t>(x);
  if (ldx == ldy && dy % (ldx * static_cast<intptr_t>(sizeof(float))) == 0)
    p.diag_off = dy / (ldx * static_cast<intptr_t>(sizeof(float)));
  // adj leaves through the staging boxes where TMA can address it: 16-byte aligned base and pitch, and rows that end on a
  // 16-byte boundary (the byte analogue of pairwise_distance's n % 4 rule for fp32 above); coordinates fit int32 (m, n <
  // 2^31 above).  Otherwise the epilogue stores from registers.
  p.tma_store = (adj && reinterpret_cast<uintptr_t>(adj) % 16 == 0 && ld_adj % 16 == 0 && n % 16 == 0) ? 1 : 0;
  ProfileScope prof(s);
  return launch_tc(s, w, p, k, EPI_EPS, POST_CLAMP);
}

// ------------------------------------------------------------------------------------------
// Kernel Gram matrices (raft::distance::kernels): pairwise_distance's InnerProduct (LINEAR, POLYNOMIAL, TANH) or
// L2Expanded (RBF) value, transformed in the epilogue of the same kernel (expanded_tc.cuh gram_post; fp64: f64_gram).

// the pairwise metric whose value a kernel transforms
static int gram_base_metric(int kernel) { return kernel == B2D_KERNEL_RBF ? B2D_L2Expanded : B2D_InnerProduct; }
static bool gram_kernel_known(int kernel) { return kernel >= B2D_KERNEL_LINEAR && kernel <= B2D_KERNEL_TANH; }

size_t b2d_gram_matrix_workspace_bytes(int kernel, int dtype, int64_t m, int64_t n, int64_t k)
{
  if (!gram_kernel_known(kernel)) return static_cast<size_t>(-1);
  return b2d_pairwise_workspace_bytes(gram_base_metric(kernel), dtype, m, n, k);
}

int b2d_gram_matrix(void* stream, int kernel, int degree, double gamma, double coef0, int dtype, const void* x, int64_t ldx,
                    const void* y, int64_t ldy, void* out, int64_t ldo, int64_t m, int64_t n, int64_t k, int row_major,
                    void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (!gram_kernel_known(kernel)) return fail(B2D_ERR_INVALID_ARG, "unknown kernel " + std::to_string(kernel));
  if (dtype != B2D_F32 && dtype != B2D_F16 && dtype != B2D_F64) return fail(B2D_ERR_UNSUPPORTED, "dtype");
  // gamma and coef0 in the precision they are used in: double for fp64 inputs, float otherwise
  const bool finite = dtype == B2D_F64 ? std::isfinite(gamma) && std::isfinite(coef0)
                                       : std::isfinite(static_cast<float>(gamma)) && std::isfinite(static_cast<float>(coef0));
  if (!finite) return fail(B2D_ERR_INVALID_ARG, "gamma and coef0 must be finite");
  if (kernel == B2D_KERNEL_POLYNOMIAL && degree < 0) return fail(B2D_ERR_INVALID_ARG, "degree must be >= 0");
  if (m < 0 || n < 0 || k < 0) return fail(B2D_ERR_INVALID_ARG, "negative extent");
  if (m == 0 || n == 0) return B2D_OK;
  if (k == 0) return fail(B2D_ERR_INVALID_ARG, "k must be positive");
  if (!x || !y || !out) return fail(B2D_ERR_INVALID_ARG, "null x / y / out");
  if (m > 0x7fffffffll * 128 || n > 0x7fffffffll || k > (1 << 24)) return fail(B2D_ERR_INVALID_ARG, "extent too large");
  if (row_major) {
    if (ldx < k || ldy < k || ldo < n) return fail(B2D_ERR_INVALID_ARG, "leading dimension smaller than the row length");
  } else {
    if (ldx < m || ldy < n || ldo < m) return fail(B2D_ERR_INVALID_ARG, "leading dimension smaller than the column length");
  }
  if (kernel != B2D_KERNEL_POLYNOMIAL) degree = 0;
  if (dtype == B2D_F64) {
    const int metric = kernel == B2D_KERNEL_LINEAR ? B2D_InnerProduct
                     : kernel == B2D_KERNEL_POLYNOMIAL ? F64_GRAM_POLY
                     : kernel == B2D_KERNEL_RBF ? F64_GRAM_RBF : F64_GRAM_TANH;
    if (row_major)
      return pairwise_f64(s, metric, static_cast<const double*>(x), ldx, 1, static_cast<const double*>(y), ldy, 1,
                          static_cast<double*>(out), ldo, m, n, k, 0, 2.0, workspace, workspace_bytes, gamma, coef0, degree);
    return pairwise_f64(s, metric, static_cast<const double*>(y), 1, ldy, static_cast<const double*>(x), 1, ldx,
                        static_cast<double*>(out), ldo, n, m, k, 1, 2.0, workspace, workspace_bytes, gamma, coef0, degree);
  }
  // Fortran order: the row-major [n, m] matrix of K(y_j, x_i), the same values (every kernel is symmetric)
  TcStore c;
  c.mode   = kernel == B2D_KERNEL_RBF ? PREP_L2 : PREP_INNER;
  c.post   = kernel == B2D_KERNEL_LINEAR ? POST_NONE
           : kernel == B2D_KERNEL_POLYNOMIAL ? POST_POLY
           : kernel == B2D_KERNEL_RBF ? POST_RBF : POST_TANH;
  c.gamma  = static_cast<float>(gamma);
  c.coef0  = static_cast<float>(coef0);
  c.degree = degree;
  const bool alias = x == y && m == n && ldx == ldy;
  if (row_major) return tc_store(s, c, dtype, x, ldx, 1, m, y, ldy, 1, n, k, static_cast<float*>(out), ldo, alias, workspace, workspace_bytes);
  return tc_store(s, c, dtype, y, 1, ldy, n, x, 1, ldx, m, k, static_cast<float*>(out), ldo, alias, workspace, workspace_bytes);
}

// ------------------------------------------------------------------------------------------
// k-means (kmeans.cuh): Lloyd's iterations on the exact EPI_MINLOC arg-min, the deterministic centroid update and the
// k-means++ / Random initialisations.  Every call only enqueues work; the loop of a fit runs max_iter conditional
// iterations on the device (run word in KmCtrl).
namespace {
constexpr int64_t kKmHistCap = 1ll << 24;   // histogram words (n_clusters x row blocks) the layout allows

// The stable counting sort of m rows by a label in [0, nc) (km_assign_kernel's histogram, km_scan_*, km_scatter_kernel):
// row blocks of 2048 rows, or more when nc x blocks would exceed kKmHistCap words.  A function of (m, nc) only, so the
// summation order of k-means never depends on the device.
struct KmSortPlan {
  int64_t rb, nblk, nhist;
};

static KmSortPlan km_sort_plan(int64_t m, int64_t nc)
{
  const int64_t mm = std::max<int64_t>(m, 1), ncc = std::max<int64_t>(nc, 1);
  KmSortPlan P;
  P.rb = kKmSub;
  if (ncc * ((mm + kKmSub - 1) / kKmSub) > kKmHistCap) {
    const int64_t nblk = std::max<int64_t>(1, kKmHistCap / ncc);
    P.rb = ((mm + nblk - 1) / nblk + kKmSub - 1) / kKmSub * kKmSub;
  }
  P.nblk   = (mm + P.rb - 1) / P.rb;
  P.nhist  = ncc * P.nblk;
  return P;
}

// the sort's regions in the workspace
struct KmSort {
  unsigned* hist;   // label counts per (label, row block), scanned in place into the sort cursors
  unsigned* tiles;  // scan tile sums
  int* perm;        // [m] row ids sorted by label
  int* slab;        // [m] their labels
  KmCtrl* ctrl;     // receives the scan total
};

// Sized for the plan of exactly nc labels, or with any_count for the plan of any label count up to nc:
// km_sort_plan(m, c).nhist <= min(c * ceil(m / 2048), max(c, kKmHistCap)), which grows with c.  The histogram holds at
// least nc words, so its tiles also serve a scan of nc words (km_scan).
static KmSort km_sort_regions(Carve& c, int64_t m, int64_t nc, bool any_count)
{
  const int64_t mm = std::max<int64_t>(m, 1), ncc = std::max<int64_t>(nc, 1);
  const int64_t words = any_count ? std::min(ncc * ((mm + kKmSub - 1) / kKmSub), std::max(ncc, kKmHistCap))
                                  : km_sort_plan(m, nc).nhist;
  KmSort S;
  S.hist  = c.take<unsigned>(words);
  S.tiles = c.take<unsigned>((words + kKmScanTile - 1) / kKmScanTile);
  S.perm  = c.take<int>(m);
  S.slab  = c.take<int>(m);
  S.ctrl  = c.take<KmCtrl>(1);
  return S;
}

static unsigned km_grid(int64_t n, int per = 256) { return static_cast<unsigned>(std::max<int64_t>(1, std::min<int64_t>((n + per - 1) / per, 1 << 16))); }

// exclusive scan of the words a[0, n) in place, the total into ctrl->total
static int km_scan(cudaStream_t s, const unsigned* run, unsigned* a, int64_t n, unsigned* tiles, KmCtrl* ctrl)
{
  const unsigned ntiles = static_cast<unsigned>((n + kKmScanTile - 1) / kKmScanTile);
  km_scan_tiles_kernel<<<ntiles, kKmThreads, 0, s>>>(run, a, n, tiles);
  km_scan_kernel<<<ntiles, kKmThreads, 0, s>>>(run, a, n, tiles, ctrl);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

// the histogram of given labels (km_assign fuses it into the arg-min)
static int km_sort_count(cudaStream_t s, const KmSort& S, const KmSortPlan& P, const int* labels, int64_t m, int64_t nc)
{
  km_begin_kernel<<<km_grid(P.nhist), 256, 0, s>>>(nullptr, nullptr, 0, nullptr, nullptr, S.hist, P.nhist);
  km_assign_kernel<<<static_cast<unsigned>(P.nblk), kKmThreads, 0, s>>>(nullptr, nullptr, const_cast<int*>(labels), nullptr, m,
                                                                        static_cast<int>(nc), P.rb, P.nblk, S.hist, nullptr);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

// the histogram scanned into the sort cursors, then the rows scattered into perm / slab
static int km_sort_scatter(cudaStream_t s, const unsigned* run, const KmSort& S, const KmSortPlan& P, const int* labels,
                           int64_t m, int64_t nc)
{
  int rc = km_scan(s, run, S.hist, P.nhist, S.tiles, S.ctrl);
  if (rc) return rc;
  const int end_bit = 32 - __builtin_clz(static_cast<unsigned>(nc));
  km_scatter_kernel<<<static_cast<unsigned>(P.nblk), kKmThreads, 0, s>>>(run, labels, m, static_cast<int>(nc), end_bit, P.rb,
                                                                         P.nblk, S.hist, S.perm, S.slab);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

struct KmLayout {
  TcWorkspace tc;   // x (side 0) and the centroids (side 1) of the arg-min, keys[m]
  KmSortPlan P;
  KmSort sort;
  KmCtrl* ctrl;     // the fit's control words: sort.ctrl
  int* labels;      // [m]
  float* w;         // [m] the normalised weights
  float* rowf;      // [m] k-means++ D^2 / Random: the uniforms
  double *sums, *wsums, *part, *wpart, *shift, *ipart, *bs;
  float* best;      // [nc * k] n_init: the best centroids so far
  float* sk_val;    // Random: select_k outputs and workspace
  int64_t* sk_idx;
  void* sk_ws;
  size_t sk_bytes;
  int64_t nchunks, nb;
  size_t bytes;
};

static KmLayout km_layout(void* base, int64_t m, int64_t k, int64_t nc)
{
  Carve c(base, 1024);
  KmLayout L{};
  L.tc      = tc_layout(c, m, nc, k, false);
  L.tc.keys = c.take<long long>(m);
  const int64_t mm = std::max<int64_t>(m, 1);
  L.P       = km_sort_plan(m, nc);
  L.nchunks = (mm + kKmChunk - 1) / kKmChunk;
  L.nb      = (mm + kKmPpBlock - 1) / kKmPpBlock;
  L.labels = c.take<int>(m);
  L.w      = c.take<float>(m);
  L.rowf   = c.take<float>(m);
  L.sort   = km_sort_regions(c, m, nc, false);
  L.ctrl   = L.sort.ctrl;
  L.sums   = c.take<double>(static_cast<size_t>(nc) * k);
  L.wsums  = c.take<double>(nc);
  L.part   = c.take<double>(static_cast<size_t>(L.nchunks) * 2 * k);
  L.wpart  = c.take<double>(L.nchunks * 2);
  L.shift  = c.take<double>(nc);
  L.ipart  = c.take<double>(L.P.nblk);
  L.bs     = c.take<double>(static_cast<size_t>(L.nb) * kKmPpMaxTrials);
  L.best   = c.take<float>(static_cast<size_t>(nc) * k);
  L.sk_val = c.take<float>(nc);
  L.sk_idx = c.take<int64_t>(nc);
  L.sk_bytes = (nc >= 1 && nc <= m) ? b2d_select_k_workspace_bytes(1, m, nc) : 0;
  L.sk_ws  = c.take<char>(L.sk_bytes);
  L.bytes  = c.bytes;
  return L;
}

static int km_args(const float* x, int64_t ldx, int64_t m, int64_t k, int64_t nc, const void* c)
{
  if (m < 0 || k < 0) return fail(B2D_ERR_INVALID_ARG, "negative extent");
  if (k < 1 || k > (1 << 24)) return fail(B2D_ERR_INVALID_ARG, "k must be in [1, 2^24]");
  if (m > 0x7fffffffll) return fail(B2D_ERR_INVALID_ARG, "m must be below 2^31");
  if (nc < 1 || nc > m) return fail(B2D_ERR_INVALID_ARG, "n_clusters must be in [1, m]");
  if (!x || !c) return fail(B2D_ERR_INVALID_ARG, "null x / centroids");
  if (ldx < k) return fail(B2D_ERR_INVALID_ARG, "leading dimension smaller than k");
  return B2D_OK;
}

// arg-min of every row against the prepared centroids: labels, inertia partials, label histogram (when hist)
static int km_assign(cudaStream_t s, const KmLayout& L, int64_t m, int64_t k, int64_t nc, const float* c, const float* w,
                     int* labels, const unsigned* run, bool prep_y, bool hist)
{
  const int64_t nh = hist ? L.P.nhist : 0;
  // (the centroid side's exponent and scale flag are zeroed only where it is prepared again below)
  km_begin_kernel<<<km_grid(std::max(m, nh)), 256, 0, s>>>(run, L.tc.keys, m, prep_y ? L.tc.gmax : nullptr, L.tc.nonuni,
                                                           hist ? L.sort.hist : nullptr, nh);
  B2D_CUDA(cudaGetLastError());
  if (prep_y) {
    int rc = launch_prep<float>(s, L.tc, nullptr, 0, 1, m, c, k, 1, nc, k, nullptr, nullptr, PREP_L2, 0, 0, 1.f, 0.f,
                                nullptr, true, run);
    if (rc) return rc;
  }
  TcParams p;
  memset(&p, 0, sizeof(p));
  p.m = m; p.n = nc; p.keys = L.tc.keys; p.run_flag = run;
  int rc = launch_tc(s, L.tc, p, k, EPI_MINLOC, POST_NONE);
  if (rc) return rc;
  km_assign_kernel<<<static_cast<unsigned>(L.P.nblk), kKmThreads, 0, s>>>(run, L.tc.keys, labels, w, m, static_cast<int>(nc),
                                                                          L.P.rb, L.P.nblk, hist ? L.sort.hist : nullptr,
                                                                          L.ipart);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

// new centroids from the histogram km_assign (or km_sort_count) left: scan, stable scatter, fp64 sums
static int km_update(cudaStream_t s, const KmLayout& L, const float* x, int64_t ldx, int64_t m, int64_t k, int64_t nc,
                     const float* w, const int* labels, const float* old_c, float* out_c, float* wpc, const unsigned* run)
{
  int rc = km_sort_scatter(s, run, L.sort, L.P, labels, m, nc);
  if (rc) return rc;
  const dim3 g(static_cast<unsigned>(L.nchunks), static_cast<unsigned>(std::min<int64_t>((k + kKmCols - 1) / kKmCols, 65535)));
  km_sum_kernel<<<g, kKmCols, 0, s>>>(run, x, ldx, static_cast<int>(k), w, L.sort.perm, L.sort.slab, L.sort.hist, L.P.nblk,
                                      L.ctrl, L.sums, L.wsums, L.part, L.wpart);
  B2D_CUDA(cudaGetLastError());
  km_finalize_kernel<<<static_cast<unsigned>(nc), kKmCols, 0, s>>>(run, static_cast<int>(k), L.sort.hist, L.P.nblk, L.sums,
                                                                   L.wsums, L.part, L.wpart, old_c, out_c, L.shift, wpc);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

// fit / predict weights: scaled to sum to m; a negative or NaN weight, or a zero sum, marks the inertia NaN
static const float* km_weights(cudaStream_t s, const KmLayout& L, const float* w, int64_t m, bool normalize)
{
  if (!w) return nullptr;
  km_wsum_kernel<<<static_cast<unsigned>(L.nb), kKmThreads, 0, s>>>(w, m, L.bs, L.ctrl);
  km_wscale_kernel<<<1, kKmThreads, 0, s>>>(L.bs, L.nb, m, L.ctrl);
  if (!normalize) return w;
  km_wapply_kernel<<<km_grid(m), 256, 0, s>>>(w, L.w, m, L.ctrl);
  return L.w;
}

static int km_plus_plus(cudaStream_t s, const KmLayout& L, const float* x, int64_t ldx, const float* w, int64_t m, int64_t k,
                        int64_t nc, uint64_t seed, float* c)
{
  const int trials = std::min(kKmPpMaxTrials, 2 + static_cast<int>(std::floor(std::log(static_cast<double>(nc)))));
  km_pp_init_kernel<<<static_cast<unsigned>(L.nb), kKmThreads, 0, s>>>(w, m, L.rowf, L.bs, L.ctrl);
  B2D_CUDA(cudaGetLastError());
  km_pp_choose_kernel<<<1, kKmThreads, 0, s>>>(x, ldx, static_cast<int>(k), w, m, L.rowf, L.bs, L.nb, L.ctrl, c, -1,
                                               static_cast<int>(nc), trials, seed);
  B2D_CUDA(cudaGetLastError());
  for (int64_t r = 0; r < nc; ++r) {
    km_pp_pass_kernel<<<static_cast<unsigned>(L.nb), kKmThreads, 0, s>>>(x, ldx, static_cast<int>(k), w, m, L.rowf, L.bs, L.ctrl);
    B2D_CUDA(cudaGetLastError());
    km_pp_choose_kernel<<<1, kKmThreads, 0, s>>>(x, ldx, static_cast<int>(k), w, m, L.rowf, L.bs, L.nb, L.ctrl, c,
                                                 static_cast<int>(r), static_cast<int>(nc), trials, seed);
    B2D_CUDA(cudaGetLastError());
  }
  return B2D_OK;
}

// n_clusters distinct rows: the positions of the n_clusters smallest of m seeded uniforms (select_k)
static int km_random(cudaStream_t s, const KmLayout& L, const float* x, int64_t ldx, int64_t m, int64_t k, int64_t nc,
                     uint64_t seed, float* c)
{
  km_uniforms_kernel<<<km_grid(m), 256, 0, s>>>(L.rowf, m, seed);
  B2D_CUDA(cudaGetLastError());
  int rc = b2d_select_k(s, L.rowf, m, nullptr, 1, m, nc, 1, L.sk_val, L.sk_idx, L.sk_ws, L.sk_bytes);
  if (rc) return rc;
  km_gather_rows_kernel<int64_t><<<static_cast<unsigned>(nc), 128, 0, s>>>(x, ldx, static_cast<int>(k), L.sk_idx,
                                                                           static_cast<int>(nc), c);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}
}  // namespace

size_t b2d_kmeans_workspace_bytes(int64_t m, int64_t k, int64_t n_clusters)
{
  if (m < 0 || k < 0 || n_clusters < 0) return static_cast<size_t>(-1);
  return km_layout(nullptr, m, k, n_clusters).bytes;
}

int b2d_kmeans_fit(void* stream, int n_clusters, int max_iter, double tol, int init, int n_init, uint64_t seed,
                   int inertia_check, const float* x, int64_t ldx, const float* sample_weight, int64_t m, int64_t k,
                   float* centroids, double* inertia, int32_t* n_iter, void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (m == 0) return B2D_OK;
  int rc = km_args(x, ldx, m, k, n_clusters, centroids);
  if (rc) return rc;
  if (!inertia || !n_iter) return fail(B2D_ERR_INVALID_ARG, "null inertia / n_iter");
  if (max_iter < 0) return fail(B2D_ERR_INVALID_ARG, "max_iter must be >= 0");
  if (!(tol >= 0.0)) return fail(B2D_ERR_INVALID_ARG, "tol must be >= 0");
  if (init != B2D_KMEANS_INIT_PLUS_PLUS && init != B2D_KMEANS_INIT_RANDOM && init != B2D_KMEANS_INIT_ARRAY)
    return fail(B2D_ERR_INVALID_ARG, "unknown init method " + std::to_string(init));
  if (n_init < 1) return fail(B2D_ERR_INVALID_ARG, "n_init must be >= 1");
  const int64_t nc = n_clusters;
  rc = check_workspace(workspace, workspace_bytes, km_layout(nullptr, m, k, nc).bytes);
  if (rc) return rc;
  const KmLayout L = km_layout(workspace, m, k, nc);
  km_ctrl_init_kernel<<<1, 1, 0, s>>>(L.ctrl);
  B2D_CUDA(cudaGetLastError());
  const float* w = km_weights(s, L, sample_weight, m, true);
  B2D_CUDA(cudaGetLastError());
  const int runs = init == B2D_KMEANS_INIT_ARRAY ? 1 : n_init;
  unsigned* run  = &L.ctrl->run;
  for (int r = 0; r < runs; ++r) {
    if (init == B2D_KMEANS_INIT_RANDOM) rc = km_random(s, L, x, ldx, m, k, nc, seed + r, centroids);
    if (init == B2D_KMEANS_INIT_PLUS_PLUS) rc = km_plus_plus(s, L, x, ldx, w, m, k, nc, seed + r, centroids);
    if (rc) return rc;
    km_fit_begin_kernel<<<1, 1, 0, s>>>(L.ctrl);
    B2D_CUDA(cudaGetLastError());
    if (r == 0) {   // x is prepared once per fit; every iteration prepares the centroids alone
      rc = launch_prep<float>(s, L.tc, x, ldx, 1, m, centroids, k, 1, nc, k, nullptr, nullptr, PREP_L2, 0);
      if (rc) return rc;
    }
    for (int it = 0; it < max_iter; ++it) {
      rc = km_assign(s, L, m, k, nc, centroids, w, L.labels, run, true, true);
      if (rc) return rc;
      rc = km_update(s, L, x, ldx, m, k, nc, w, L.labels, centroids, centroids, nullptr, run);
      if (rc) return rc;
      km_converge_kernel<<<1, kKmThreads, 0, s>>>(run, L.ctrl, L.shift, static_cast<int>(nc), L.ipart, L.P.nblk, tol,
                                                  inertia_check);
      B2D_CUDA(cudaGetLastError());
    }
    // the inertia of the returned centroids
    rc = km_assign(s, L, m, k, nc, centroids, w, L.labels, nullptr, true, false);
    if (rc) return rc;
    km_cost_kernel<<<static_cast<unsigned>(L.P.nblk), kKmThreads, 0, s>>>(x, ldx, static_cast<int>(k), centroids, L.labels,
                                                                          w, m, L.P.rb, L.ipart);
    km_finish_kernel<<<1, kKmThreads, 0, s>>>(L.ctrl, L.ipart, L.P.nblk, runs == 1 ? inertia : nullptr,
                                              runs == 1 ? n_iter : nullptr);
    B2D_CUDA(cudaGetLastError());
    if (runs > 1) {
      km_best_decide_kernel<<<1, 1, 0, s>>>(L.ctrl, r == 0 ? 1 : 0);
      km_copy_kernel<<<km_grid(nc * k), 256, 0, s>>>(L.ctrl, 1, centroids, L.best, nc * k);
      B2D_CUDA(cudaGetLastError());
    }
  }
  if (runs > 1) {
    km_copy_kernel<<<km_grid(nc * k), 256, 0, s>>>(L.ctrl, 0, L.best, centroids, nc * k);
    km_best_out_kernel<<<1, 1, 0, s>>>(L.ctrl, inertia, n_iter);
    B2D_CUDA(cudaGetLastError());
  }
  return B2D_OK;
}

int b2d_kmeans_predict(void* stream, const float* x, int64_t ldx, const float* sample_weight, int64_t m, int64_t k,
                       const float* centroids, int n_clusters, int32_t* labels, double* inertia, int normalize_weight,
                       void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (m == 0) return B2D_OK;
  int rc = km_args(x, ldx, m, k, n_clusters, centroids);
  if (rc) return rc;
  const int64_t nc = n_clusters;
  rc = check_workspace(workspace, workspace_bytes, km_layout(nullptr, m, k, nc).bytes);
  if (rc) return rc;
  const KmLayout L = km_layout(workspace, m, k, nc);
  km_ctrl_init_kernel<<<1, 1, 0, s>>>(L.ctrl);
  B2D_CUDA(cudaGetLastError());
  const float* w = km_weights(s, L, sample_weight, m, normalize_weight != 0);
  B2D_CUDA(cudaGetLastError());
  rc = launch_prep<float>(s, L.tc, x, ldx, 1, m, centroids, k, 1, nc, k, nullptr, nullptr, PREP_L2, 0);
  if (rc) return rc;
  int* lab = labels ? labels : L.labels;
  rc = km_assign(s, L, m, k, nc, centroids, w, lab, nullptr, false, false);
  if (rc) return rc;
  km_cost_kernel<<<static_cast<unsigned>(L.P.nblk), kKmThreads, 0, s>>>(x, ldx, static_cast<int>(k), centroids, lab, w, m,
                                                                        L.P.rb, L.ipart);
  km_finish_kernel<<<1, kKmThreads, 0, s>>>(L.ctrl, L.ipart, L.P.nblk, inertia, nullptr);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

int b2d_kmeans_update_centroids(void* stream, const float* x, int64_t ldx, const float* sample_weight, const int32_t* labels,
                                int64_t m, int64_t k, const float* old_centroids, int n_clusters, float* new_centroids,
                                float* weight_per_cluster, void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (m == 0) return B2D_OK;
  int rc = km_args(x, ldx, m, k, n_clusters, old_centroids);
  if (rc) return rc;
  if (!labels || !new_centroids) return fail(B2D_ERR_INVALID_ARG, "null labels / new_centroids");
  const int64_t nc = n_clusters;
  rc = check_workspace(workspace, workspace_bytes, km_layout(nullptr, m, k, nc).bytes);
  if (rc) return rc;
  const KmLayout L = km_layout(workspace, m, k, nc);
  rc = km_sort_count(s, L.sort, L.P, labels, m, nc);
  if (rc) return rc;
  return km_update(s, L, x, ldx, m, k, nc, sample_weight, labels, old_centroids, new_centroids, weight_per_cluster, nullptr);
}

int b2d_kmeans_init_plus_plus(void* stream, const float* x, int64_t ldx, const float* sample_weight, int64_t m, int64_t k,
                              int n_clusters, uint64_t seed, float* centroids, void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (m == 0) return B2D_OK;
  int rc = km_args(x, ldx, m, k, n_clusters, centroids);
  if (rc) return rc;
  const int64_t nc = n_clusters;
  rc = check_workspace(workspace, workspace_bytes, km_layout(nullptr, m, k, nc).bytes);
  if (rc) return rc;
  const KmLayout L = km_layout(workspace, m, k, nc);
  return km_plus_plus(s, L, x, ldx, sample_weight, m, k, nc, seed, centroids);
}

// ------------------------------------------------------------------------------------------
// Minimum spanning forest and single-linkage clustering (single_linkage.cuh): edge-list Borůvka under the key order
// key_pack(w, e); single_linkage runs it on the kNN graph, connects the components the graph leaves apart with the
// masked arg-min, and builds the dendrogram on the host.
namespace {
constexpr int64_t kSlMaxRows  = 1ll << 30;
constexpr int64_t kSlMaxEdges = 0xFFFFFFFFll;   // positions are the low 32 bits of a key (2^32 - 1 only in KEY_EMPTY)

struct MstLayout {
  SlCtrl* ctrl;
  int* colour;        // [n] component of every vertex (the id of a vertex of it)
  int* parent;        // [n] hook forest of the components of a round; at the end the smallest vertex of each tree
  long long* best;    // [n] minimum key of every component in a round
  long long* keys;    // [n] keys of the forest edges in the order they were chosen (KEY_EMPTY behind them)
  long long* alt;     // [n] the other buffer of the radix sort
  void* sort_tmp;
  size_t sort_bytes;
  size_t bytes;
};

// (extern "C": no overloads)
static MstLayout mst_regions(Carve& c, int64_t n)
{
  MstLayout L{};
  L.ctrl       = c.take<SlCtrl>(1);
  L.colour     = c.take<int>(n);
  L.parent     = c.take<int>(n);
  L.best       = c.take<long long>(n);
  L.keys       = c.take<long long>(n);
  L.alt        = c.take<long long>(n);
  L.sort_bytes = kSortTmpBytes + static_cast<size_t>(n) * 4;   // (checked at run time)
  L.sort_tmp   = c.take<char>(L.sort_bytes);
  L.bytes      = c.bytes;
  return L;
}

static MstLayout mst_layout(void* base, int64_t n)
{
  Carve c(base, 1024);
  return mst_regions(c, n);
}

static unsigned sl_grid(int64_t n) { return static_cast<unsigned>(std::max<int64_t>(1, (n + 255) / 256)); }

static int ceil_log2(int64_t n)
{
  int r = 0;
  while ((1ll << r) < n) ++r;
  return r;
}

// Borůvka rounds over the edges [e0, e1) of a graph on n vertices with at most `comps` components, every other edge
// already inside a component.  Only enqueues: the non-isolated components at least halve in every round, so
// ceil(log2 comps) rounds finish, and every kernel after a round that appended nothing returns at once.
static int mst_rounds(cudaStream_t s, const MstLayout& L, const int* src, const int* dst, const float* w, int64_t n,
                      int64_t e0, int64_t e1, int64_t comps)
{
  const int rounds = ceil_log2(comps) + 1;
  const int jumps  = std::min(kSlMaxJumps, ceil_log2(comps) + 1);   // hook chains are shorter than comps
  const unsigned ge = static_cast<unsigned>(std::max<int64_t>(1, std::min<int64_t>((e1 - e0 + 255) / 256, 1 << 16)));
  for (int r = 0; r < rounds; ++r) {
    sl_round_begin_kernel<<<sl_grid(std::max<int64_t>(n, kSlMaxJumps)), 256, 0, s>>>(L.ctrl, L.best, n);
    sl_edge_kernel<<<ge, 256, 0, s>>>(L.ctrl, src, dst, w, e0, e1, n, L.colour, L.best);
    sl_hook_kernel<<<sl_grid(n), 256, 0, s>>>(L.ctrl, src, dst, L.colour, L.best, L.parent, L.keys, n);
    for (int j = 0; j < jumps; ++j) sl_jump_kernel<<<sl_grid(n), 256, 0, s>>>(L.ctrl, L.colour, L.parent, n, j);
    sl_relabel_kernel<<<sl_grid(n), 256, 0, s>>>(L.ctrl, L.colour, L.parent, n);
    sl_round_end_kernel<<<1, 1, 0, s>>>(L.ctrl);
    B2D_CUDA(cudaGetLastError());
  }
  return B2D_OK;
}

// the forest edges in key order: endpoints, weights (their square roots with do_sqrt) and the count
static int mst_emit(cudaStream_t s, const MstLayout& L, const int* src, const int* dst, const float* w, int64_t n,
                    int do_sqrt, int* out_src, int* out_dst, float* out_w, int* out_count)
{
  cub::DoubleBuffer<long long> db(L.keys, L.alt);
  size_t need = 0;
  B2D_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, need, db, static_cast<int>(n), 0, 64, s));
  if (need > L.sort_bytes) return fail(B2D_ERR_WORKSPACE, "internal: radix sort scratch " + std::to_string(need) + " bytes");
  B2D_CUDA(cub::DeviceRadixSort::SortKeys(L.sort_tmp, need, db, static_cast<int>(n), 0, 64, s));
  sl_emit_kernel<<<sl_grid(n), 256, 0, s>>>(L.ctrl, db.Current(), src, dst, w, std::max<int64_t>(n - 1, 0), do_sqrt,
                                            out_src, out_dst, out_w, out_count);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

// kNN neighbours of single_linkage: min(m, max(2, floor(log2 m) + c))
static int64_t sl_neighbors(int64_t m, int64_t c)
{
  if (m < 1) return 0;
  const int64_t fl = 63 - __builtin_clzll(static_cast<unsigned long long>(m));
  return std::min<int64_t>(m, std::max<int64_t>(2, fl + c));
}

// Rows of x per masked arg-min launch of connect_components: the m x c adjacency bytes (and its m c / 8 bytes of bits)
// stay below 128 m, and the tile classes below 64 MiB; a multiple of TC_BM, at least TC_BM (c <= m).
static int64_t sl_max_chunk(int64_t m)
{
  const int64_t mm = std::max<int64_t>(m, 1);
  const int64_t cap = std::max<int64_t>(TC_BM, ((1ll << 40) / mm) / TC_BM * TC_BM);
  return std::min<int64_t>((mm + TC_BM - 1) / TC_BM * TC_BM, cap);
}

static int64_t sl_chunk_rows(int64_t m, int64_t c)
{
  const int64_t r = std::max<int64_t>(TC_BM, (128 * m / std::max<int64_t>(c, 1)) / TC_BM * TC_BM);
  return std::min(r, sl_max_chunk(m));
}

// Persistent regions first (the forest, the edge list, the host copies), then one scratch region used by the kNN phase
// and, afterwards, by connect_components.  Sized for any number of components up to m, so the workspace depends on
// (m, d, n_nb) only.
struct SlLayout {
  MstLayout mst;            // over the m rows
  int *src, *dst;           // [m n_nb + m] edge list: the kNN graph (position i n_nb + s), then the connecting edges
  float* w;                 //              squared L2 weights
  int *hsrc, *hdst;         // [m] forest edges in key order, for the host
  void* knn_ws;             // kNN phase: b2d_knn's workspace, then its outputs
  size_t knn_bytes;
  int64_t* idx;             // [m n_nb]
  float* dist;              // [m n_nb]
  TcWorkspace tc;           // connect phase: the colour-sorted rows as both operands
  float* xs;                // [m, d] the colour-sorted rows
  long long *keys, *cbest;  // [m] masked arg-min of every sorted row, [c] best row of every component
  unsigned* bad;            // [8] masked_classify's flag: 0 (the component ends are valid by construction)
  int *grp, *lab, *ends;    // [m]
  unsigned* ids;            // [m] root flags, scanned into dense component ids
  KmSort sort;              // the rows sorted by component, for up to m components
  unsigned* bits;           // [5 m] adjacency bits of one chunk
  uint8_t* cls;             // tile classes of one chunk
  uint8_t* adj;             // [128 m] adjacency of one chunk
  size_t bytes;
};

static SlLayout sl_layout(void* base, int64_t m, int64_t d, int64_t n_nb)
{
  Carve c(base, 1024);
  SlLayout L{};
  L.mst  = mst_regions(c, m);
  const size_t ne = static_cast<size_t>(m) * n_nb + m;
  L.src  = c.take<int>(ne);
  L.dst  = c.take<int>(ne);
  L.w    = c.take<float>(ne);
  L.hsrc = c.take<int>(m);
  L.hdst = c.take<int>(m);
  char* scratch = base ? static_cast<char*>(base) + c.bytes : nullptr;
  // kNN phase
  const KnnLayout K = knn_layout(nullptr, m, m, d, n_nb);
  Carve a(scratch, 1024);
  L.knn_ws    = a.take<char>(K.bytes);
  L.knn_bytes = K.bytes;
  L.idx       = a.take<int64_t>(static_cast<size_t>(m) * n_nb);
  L.dist      = a.take<float>(static_cast<size_t>(m) * n_nb);
  // connect phase
  Carve b(scratch, 1024);
  L.tc    = tc_layout(b, m, m, d, false);
  L.xs    = b.take<float>(static_cast<size_t>(m) * d);
  L.keys  = b.take<long long>(m);
  L.cbest = b.take<long long>(m);
  L.bad   = b.take<unsigned>(8);
  L.grp   = b.take<int>(m);
  L.lab   = b.take<int>(m);
  L.ends  = b.take<int>(m);
  L.ids   = b.take<unsigned>(m);
  L.sort  = km_sort_regions(b, m, m, true);
  const int64_t mm = std::max<int64_t>(m, 1);
  L.bits  = b.take<unsigned>(static_cast<size_t>(5) * mm);
  L.cls   = b.take<uint8_t>(static_cast<size_t>(sl_max_chunk(m) / TC_BM) * ((mm + TC_BN - 1) / TC_BN));
  L.adj   = b.take<uint8_t>(static_cast<size_t>(128) * mm);
  L.bytes = c.bytes + std::max(a.bytes, b.bytes);
  return L;
}

// One round of connect_components for c > 1 components: dense component ids, the rows sorted by component (stable),
// the masked arg-min of every sorted row against the rows of other components in row chunks, and for every component
// the edge from its row of smallest (distance, row) to that row's nearest row: edges [e0, e0 + c).
static int sl_connect(cudaStream_t s, const SlLayout& L, const float* x, int64_t ldx, int64_t m, int64_t d, int64_t c,
                      int64_t e0)
{
  const MstLayout& T = L.mst;
  const KmSort& S = L.sort;
  sl_root_flags_kernel<<<sl_grid(m), 256, 0, s>>>(T.colour, L.ids, m);
  int rc = km_scan(s, nullptr, L.ids, m, S.tiles, S.ctrl);
  if (rc) return rc;
  sl_dense_label_kernel<<<sl_grid(m), 256, 0, s>>>(T.colour, L.ids, L.lab, m);
  B2D_CUDA(cudaGetLastError());
  const KmSortPlan P = km_sort_plan(m, c);
  rc = km_sort_count(s, S, P, L.lab, m, c);
  if (rc) return rc;
  rc = km_sort_scatter(s, nullptr, S, P, L.lab, m, c);
  if (rc) return rc;
  sl_ends_kernel<<<sl_grid(c), 256, 0, s>>>(S.hist, P.nblk, c, L.ends);
  km_gather_rows_kernel<int><<<static_cast<unsigned>(m), 128, 0, s>>>(x, ldx, static_cast<int>(d), S.perm,
                                                                      static_cast<int>(m), L.xs);
  B2D_CUDA(cudaGetLastError());
  // y (and x) prepared once per round; every chunk takes a window of the x side
  rc = launch_prep<float>(s, L.tc, L.xs, d, 1, m, L.xs, d, 1, m, d, nullptr, nullptr, PREP_L2, 0);
  if (rc) return rc;
  masked_group_map_kernel<<<sl_grid(m), 256, 0, s>>>(L.grp, L.ends, c, m);
  B2D_CUDA(cudaMemsetAsync(L.bad, 0, 32, s));
  minloc_init_kernel<<<sl_grid(m), 256, 0, s>>>(L.keys, m);
  minloc_init_kernel<<<sl_grid(c), 256, 0, s>>>(L.cbest, c);
  B2D_CUDA(cudaGetLastError());
  const int64_t mc = sl_chunk_rows(m, c);
  for (int64_t r0 = 0; r0 < m; r0 += mc) {
    const int64_t rows = std::min(mc, m - r0);
    sl_adj_kernel<<<km_grid(rows * c), 256, 0, s>>>(S.slab, r0, rows, c, L.adj);
    B2D_CUDA(cudaGetLastError());
    rc = masked_keys(s, tc_rows(L.tc, 0, r0, d), L.keys + r0, L.grp, L.bits, L.cls, L.bad, L.adj, c, L.ends, c, rows, m, d);
    if (rc) return rc;
  }
  sl_comp_best_kernel<<<sl_grid(m), 256, 0, s>>>(L.keys, S.slab, m, L.cbest);
  sl_connect_kernel<<<sl_grid(c), 256, 0, s>>>(L.cbest, L.keys, S.perm, S.slab, c, e0, L.src, L.dst, L.w, T.ctrl);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

static int sl_read_ctrl(cudaStream_t s, const SlCtrl* d, SlCtrl* h)
{
  B2D_CUDA(cudaMemcpyAsync(h, d, sizeof(SlCtrl), cudaMemcpyDeviceToHost, s));
  B2D_CUDA(cudaStreamSynchronize(s));
  return B2D_OK;
}

static int uf_find(std::vector<int>& p, int v)
{
  while (p[v] != v) v = p[v] = p[p[v]];
  return v;
}
}  // namespace

size_t b2d_mst_workspace_bytes(int64_t n_vertices, int64_t n_edges)
{
  if (n_vertices < 0 || n_edges < 0) return static_cast<size_t>(-1);
  return mst_layout(nullptr, n_vertices).bytes;
}

int b2d_mst(void* stream, const int32_t* src, const int32_t* dst, const float* w, int64_t n_vertices, int64_t n_edges,
            int32_t* out_src, int32_t* out_dst, float* out_w, int32_t* out_colour, int32_t* out_count, void* workspace,
            size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int64_t n = n_vertices, E = n_edges;
  if (n < 0 || E < 0) return fail(B2D_ERR_INVALID_ARG, "negative extent");
  if (n >= kSlMaxRows) return fail(B2D_ERR_UNSUPPORTED, "mst: n_vertices must be below 2^30");
  if (E >= kSlMaxEdges) return fail(B2D_ERR_UNSUPPORTED, "mst: n_edges must be below 2^32 - 1");
  if (E > 0 && (!src || !dst || !w)) return fail(B2D_ERR_INVALID_ARG, "null src / dst / w");
  if (!out_count || (n > 0 && !out_colour) || (n > 1 && (!out_src || !out_dst || !out_w)))
    return fail(B2D_ERR_INVALID_ARG, "null out_src / out_dst / out_w / out_colour / out_count");
  int rc = check_workspace(workspace, workspace_bytes, mst_layout(nullptr, n).bytes);
  if (rc) return rc;
  if (n == 0) {
    B2D_CUDA(cudaMemsetAsync(out_count, 0, sizeof(int32_t), s));
    return B2D_OK;
  }
  const MstLayout L = mst_layout(workspace, n);
  sl_mst_init_kernel<<<sl_grid(n), 256, 0, s>>>(L.ctrl, L.colour, L.keys, n);
  B2D_CUDA(cudaGetLastError());
  rc = mst_rounds(s, L, src, dst, w, n, 0, E, n);
  if (rc) return rc;
  rc = mst_emit(s, L, src, dst, w, n, 0, out_src, out_dst, out_w, out_count);
  if (rc) return rc;
  sl_fill_kernel<<<sl_grid(n), 256, 0, s>>>(L.parent, 0x7fffffff, n);
  sl_min_vertex_kernel<<<sl_grid(n), 256, 0, s>>>(L.colour, L.parent, n);
  sl_colour_out_kernel<<<sl_grid(n), 256, 0, s>>>(L.colour, L.parent, out_colour, n);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

size_t b2d_single_linkage_workspace_bytes(int64_t m, int64_t d, int c)
{
  if (m < 0 || d < 0) return static_cast<size_t>(-1);
  const int64_t n_nb = sl_neighbors(m, c);
  if (n_nb > KNN_MAX_K || m >= kSlMaxRows) return static_cast<size_t>(-1);
  return sl_layout(nullptr, m, d, n_nb).bytes;
}

int b2d_single_linkage(void* stream, int metric, const float* x, int64_t ldx, int64_t m, int64_t d, int c, int n_clusters,
                       int32_t* children, float* deltas, int32_t* sizes, int32_t* labels, int32_t* n_components_out,
                       void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (metric != B2D_L2Expanded && metric != B2D_L2SqrtExpanded)
    return fail(B2D_ERR_UNSUPPORTED, "single_linkage supports the L2Expanded and L2SqrtExpanded metrics");
  if (m < 1 || d < 1) return fail(B2D_ERR_INVALID_ARG, "m and d must be positive");
  if (d > 320) return fail(B2D_ERR_UNSUPPORTED, "single_linkage supports d <= 320 (the fused kNN's limit)");
  if (m >= kSlMaxRows) return fail(B2D_ERR_UNSUPPORTED, "single_linkage: m must be below 2^30");
  if (n_clusters < 1 || n_clusters > m) return fail(B2D_ERR_INVALID_ARG, "n_clusters must be in [1, m]");
  const int64_t n_nb = sl_neighbors(m, c);
  if (n_nb > KNN_MAX_K)
    return fail(B2D_ERR_UNSUPPORTED, "single_linkage: min(m, max(2, floor(log2 m) + c)) = " + std::to_string(n_nb) +
                                         " neighbours exceeds 64: lower c (" + std::to_string(c) + ")");
  if (m * n_nb + m >= kSlMaxEdges)
    return fail(B2D_ERR_UNSUPPORTED, "single_linkage: m * (n_nb + 1) edges must stay below 2^32 - 1");
  if (!x || !labels || !n_components_out || (m > 1 && (!children || !deltas || !sizes)))
    return fail(B2D_ERR_INVALID_ARG, "null x / children / deltas / sizes / labels / n_components_out");
  if (ldx < d) return fail(B2D_ERR_INVALID_ARG, "leading dimension smaller than d");
  int rc = check_workspace(workspace, workspace_bytes, sl_layout(nullptr, m, d, n_nb).bytes);
  if (rc) return rc;
  const SlLayout L = sl_layout(workspace, m, d, n_nb);
  const MstLayout& T = L.mst;
  SlCtrl h;
  sl_mst_init_kernel<<<sl_grid(m), 256, 0, s>>>(T.ctrl, T.colour, T.keys, m);
  sl_finite_kernel<<<km_grid(m * d), 256, 0, s>>>(x, ldx, m, static_cast<int>(d), T.ctrl);
  B2D_CUDA(cudaGetLastError());
  // 1. the kNN graph (squared distances, whatever the metric)
  if (m > 1) {
    rc = b2d_knn(s, L.idx, L.dist, B2D_L2Expanded, x, ldx, x, ldx, m, m, d, n_nb, L.knn_ws, L.knn_bytes);
    if (rc) return rc;
    sl_knn_edges_kernel<<<sl_grid(m * n_nb), 256, 0, s>>>(L.idx, L.dist, m, static_cast<int>(n_nb), L.src, L.dst, L.w);
    B2D_CUDA(cudaGetLastError());
    // 2.-3. its minimum spanning forest
    rc = mst_rounds(s, T, L.src, L.dst, L.w, m, 0, m * n_nb, m);
    if (rc) return rc;
  }
  rc = sl_read_ctrl(s, T.ctrl, &h);
  if (rc) return rc;
  if (h.bad & 1u) return fail(B2D_ERR_INVALID_ARG, "single_linkage: X holds a non-finite value");
  int64_t comps = m - h.n_mst;
  *n_components_out = static_cast<int32_t>(comps);
  // 4. connect_components: each round at least halves the components
  int64_t e = m * n_nb;
  while (comps > 1) {
    rc = sl_connect(s, L, x, ldx, m, d, comps, e);
    if (rc) return rc;
    sl_rearm_kernel<<<1, 1, 0, s>>>(T.ctrl);
    B2D_CUDA(cudaGetLastError());
    rc = mst_rounds(s, T, L.src, L.dst, L.w, m, e, e + comps, comps);
    if (rc) return rc;
    e += comps;
    rc = sl_read_ctrl(s, T.ctrl, &h);
    if (rc) return rc;
    const int64_t next = m - h.n_mst;
    if ((h.bad & 2u) || 2 * next > comps)
      return fail(B2D_ERR_CUDA, "internal: connect_components left " + std::to_string(next) + " of " +
                                    std::to_string(comps) + " components");
    comps = next;
  }
  // 5. dendrogram: the m - 1 forest edges in key order, union-find on the host
  std::vector<int> hs(m - 1), hd(m - 1);
  if (m > 1) {
    rc = mst_emit(s, T, L.src, L.dst, L.w, m, metric == B2D_L2SqrtExpanded ? 1 : 0, L.hsrc, L.hdst, deltas, nullptr);
    if (rc) return rc;
    B2D_CUDA(cudaMemcpyAsync(hs.data(), L.hsrc, (m - 1) * sizeof(int), cudaMemcpyDeviceToHost, s));
    B2D_CUDA(cudaMemcpyAsync(hd.data(), L.hdst, (m - 1) * sizeof(int), cudaMemcpyDeviceToHost, s));
    B2D_CUDA(cudaStreamSynchronize(s));
  }
  std::vector<int> uf(m), cid(m), sz(m, 1), hch(2 * (m - 1)), hsz(m - 1), hlab(m);
  for (int64_t i = 0; i < m; ++i) uf[i] = cid[i] = static_cast<int>(i);
  const int64_t cut = m - n_clusters;   // labels: the components after the first m - n_clusters merges
  for (int64_t t = 0; t < m - 1; ++t) {
    if (t == cut)
      for (int64_t i = 0; i < m; ++i) hlab[i] = uf_find(uf, static_cast<int>(i));
    const int a = uf_find(uf, hs[t]), b = uf_find(uf, hd[t]);
    if (a == b) return fail(B2D_ERR_CUDA, "internal: the spanning tree has a cycle");
    hch[2 * t]     = std::min(cid[a], cid[b]);
    hch[2 * t + 1] = std::max(cid[a], cid[b]);
    hsz[t]         = sz[a] + sz[b];
    uf[b]          = a;
    sz[a]          = hsz[t];
    cid[a]         = static_cast<int>(m + t);
  }
  if (cut == m - 1)
    for (int64_t i = 0; i < m; ++i) hlab[i] = uf_find(uf, static_cast<int>(i));
  std::vector<int> num(m, -1);   // numbered in order of each cluster's smallest row
  int next_label = 0;
  for (int64_t i = 0; i < m; ++i) {
    int& l = num[hlab[i]];
    if (l < 0) l = next_label++;
    hlab[i] = l;
  }
  if (m > 1) {
    B2D_CUDA(cudaMemcpyAsync(children, hch.data(), hch.size() * sizeof(int), cudaMemcpyHostToDevice, s));
    B2D_CUDA(cudaMemcpyAsync(sizes, hsz.data(), hsz.size() * sizeof(int), cudaMemcpyHostToDevice, s));
  }
  B2D_CUDA(cudaMemcpyAsync(labels, hlab.data(), m * sizeof(int), cudaMemcpyHostToDevice, s));
  B2D_CUDA(cudaStreamSynchronize(s));
  return B2D_OK;
}

// ------------------------------------------------------------------------------------------
// DBSCAN (dbscan.cuh): the epsilon neighbourhood of x against itself in column batches of the prepared rows, a device
// union-find over the core points and the border rule.  Only enqueues work.
namespace {
constexpr int64_t kDbDefaultBatchBytes = 1ll << 30;

// columns per batch: min(m, max(256, floor(max_bytes / m / 256) * 256)); max_bytes 0 means 2^30
static int64_t db_batch(int64_t m, int64_t max_bytes)
{
  const int64_t mm = std::max<int64_t>(m, 1);
  const int64_t mb = max_bytes > 0 ? max_bytes : kDbDefaultBatchBytes;
  return std::min(mm, std::max<int64_t>(256, mb / mm / 256 * 256));
}

struct DbLayout {
  TcWorkspace tc;    // x prepared once, as both operands
  int64_t b, nb;     // columns per batch, batches
  int64_t ld;        // adjacency row pitch: b rounded up to 16
  unsigned* deg;     // [m + nb] per-column degrees, each batch's total behind its columns
  int* parent;       // [m] union-find forest over the core rows (-1: not core)
  int* border;       // [m] smallest root reaching a non-core row (INT_MAX: none)
  unsigned* root;    // [m] root flags, scanned into cluster numbers
  unsigned* core;    // [m] core flags, scanned into core_sample_indices positions
  unsigned* tiles;   // scan tile sums
  KmCtrl* ctrl;      // [2] scan totals: clusters, core rows
  uint8_t* adj;      // [m][ld] adjacency of one batch
  size_t bytes;
};

static DbLayout db_layout(void* base, int64_t m, int64_t d, int64_t max_bytes)
{
  Carve c(base, 1024);
  DbLayout L{};
  L.tc     = tc_layout(c, m, m, d, false);
  L.b      = db_batch(m, max_bytes);
  L.nb     = (m + L.b - 1) / L.b;
  L.ld     = (L.b + 15) / 16 * 16;
  L.deg    = c.take<unsigned>(m + L.nb);
  L.parent = c.take<int>(m);
  L.border = c.take<int>(m);
  L.root   = c.take<unsigned>(m);
  L.core   = c.take<unsigned>(m);
  L.tiles  = c.take<unsigned>((m + kKmScanTile - 1) / kKmScanTile);
  L.ctrl   = c.take<KmCtrl>(2);
  L.adj    = c.take<uint8_t>(static_cast<size_t>(m) * L.ld);
  L.bytes  = c.bytes;
  return L;
}

// One EPI_EPS launch over the columns [s, s + w) of the prepared x (batch t): the adjacency into L.adj (adj) and / or
// the degrees of those columns into deg[s + t, s + t + w] (deg).  diag_off = s keeps the self pairs.
static int db_eps(cudaStream_t s, const DbLayout& L, int64_t m, int64_t d, float e, int64_t t, bool adj, bool deg)
{
  const int64_t c0 = t * L.b, w = std::min(L.b, m - c0);
  TcParams p;
  memset(&p, 0, sizeof(p));
  p.m = m; p.n = w;
  p.adj = adj ? L.adj : nullptr; p.ld_adj = L.ld;
  p.vd = deg ? L.deg + c0 + t : nullptr; p.vd64 = 0; p.eps = e;
  p.diag_off = c0;
  p.tma_store = (adj && w % 16 == 0) ? 1 : 0;   // (L.adj is 1024-byte aligned and L.ld a multiple of 16)
  return launch_tc(s, tc_rows(L.tc, 1, c0, d), p, d, EPI_EPS, POST_CLAMP);
}

static unsigned db_warp_grid(int64_t m) { return static_cast<unsigned>(std::min<int64_t>((m + 7) / 8, 1 << 16)); }
}  // namespace

size_t b2d_dbscan_workspace_bytes(int64_t m, int64_t d, int64_t max_bytes_per_batch)
{
  if (m < 0 || d < 0 || max_bytes_per_batch < 0) return static_cast<size_t>(-1);
  return db_layout(nullptr, m, d, max_bytes_per_batch).bytes;
}

int b2d_dbscan_fit(void* stream, int metric, const float* x, int64_t ldx, int64_t m, int64_t d, double eps,
                   int64_t min_samples, int64_t max_bytes_per_batch, int32_t* labels, int32_t* core_sample_indices,
                   int32_t* n_clusters, void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (metric != B2D_L2SqrtExpanded && metric != B2D_L2Expanded && metric != B2D_CosineExpanded)
    return fail(B2D_ERR_UNSUPPORTED, "dbscan supports the L2SqrtExpanded, L2Expanded and CosineExpanded metrics");
  if (m < 0 || d < 0 || max_bytes_per_batch < 0) return fail(B2D_ERR_INVALID_ARG, "negative extent or batch size");
  if (m == 0) return B2D_OK;
  if (m > 0x7fffffffll) return fail(B2D_ERR_INVALID_ARG, "dbscan: m must be below 2^31");
  if (d < 1) return fail(B2D_ERR_INVALID_ARG, "d must be positive");
  if (d > 320) return fail(B2D_ERR_UNSUPPORTED, "dbscan supports d <= 320 (the whole distance at once)");
  if (min_samples < 1) return fail(B2D_ERR_INVALID_ARG, "min_samples must be >= 1");
  if (!x || !labels) return fail(B2D_ERR_INVALID_ARG, "null x / labels");
  if (ldx < d) return fail(B2D_ERR_INVALID_ARG, "leading dimension smaller than d");
  int rc = check_workspace(workspace, workspace_bytes, db_layout(nullptr, m, d, max_bytes_per_batch).bytes);
  if (rc) return rc;
  const DbLayout L = db_layout(workspace, m, d, max_bytes_per_batch);
  // the threshold on the distance the kernel compares: eps^2 (rounded once from fp64) for L2SqrtExpanded; a NaN or
  // negative eps matches nothing (every distance is >= 0 or NaN)
  const float e = !(eps >= 0.0) ? -INFINITY : static_cast<float>(metric == B2D_L2SqrtExpanded ? eps * eps : eps);
  const unsigned ms = static_cast<unsigned>(std::min<int64_t>(min_samples, m + 1));
  // 0. x prepared once, as both operands; every batch takes a window of the y side
  rc = launch_prep<float>(s, L.tc, x, ldx, 1, m, x, ldx, 1, m, d, nullptr, nullptr,
                          metric == B2D_CosineExpanded ? PREP_COSINE : PREP_L2, 0);
  if (rc) return rc;
  // 1. degrees, then the core flags (one batch: the adjacency in the same launch)
  B2D_CUDA(cudaMemsetAsync(L.deg, 0, static_cast<size_t>(m + L.nb) * sizeof(unsigned), s));
  const bool one = L.nb == 1;
  for (int64_t t = 0; t < L.nb; ++t) {
    rc = db_eps(s, L, m, d, e, t, one, true);
    if (rc) return rc;
  }
  db_core_kernel<<<sl_grid(m), 256, 0, s>>>(L.deg, m, L.b, ms, L.parent, L.border, L.core);
  B2D_CUDA(cudaGetLastError());
  // 2. links between core points
  for (int64_t t = 0; t < L.nb; ++t) {
    const int64_t c0 = t * L.b, w = std::min(L.b, m - c0);
    if (!one) {
      rc = db_eps(s, L, m, d, e, t, true, false);
      if (rc) return rc;
    }
    db_link_kernel<<<db_warp_grid(m), kDbThreads, 0, s>>>(L.adj, L.ld, m, c0, w, L.core, L.parent);
    B2D_CUDA(cudaGetLastError());
  }
  db_compress_kernel<<<sl_grid(m), 256, 0, s>>>(L.parent, m, L.root);
  B2D_CUDA(cudaGetLastError());
  // 3. border points
  for (int64_t t = 0; t < L.nb; ++t) {
    const int64_t c0 = t * L.b, w = std::min(L.b, m - c0);
    if (!one) {
      rc = db_eps(s, L, m, d, e, t, true, false);
      if (rc) return rc;
    }
    db_border_kernel<<<db_warp_grid(m), kDbThreads, 0, s>>>(L.adj, L.ld, m, c0, w, L.parent, L.border);
    B2D_CUDA(cudaGetLastError());
  }
  // 4. cluster numbers = ranks of the roots; core_sample_indices positions = ranks of the core rows
  rc = km_scan(s, nullptr, L.root, m, L.tiles, L.ctrl);
  if (rc) return rc;
  rc = km_scan(s, nullptr, L.core, m, L.tiles, L.ctrl + 1);
  if (rc) return rc;
  db_label_kernel<<<sl_grid(m), 256, 0, s>>>(L.parent, L.border, L.root, L.core, m, &L.ctrl[0].total, &L.ctrl[1].total,
                                             labels, core_sample_indices, n_clusters);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

}  // extern "C"
