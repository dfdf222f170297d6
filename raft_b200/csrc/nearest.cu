// Fused 1-NN: fusedL2NN / fusedDistanceNN with the screened search, the single-process multi-GPU path, and the masked
// arg-min (masked_nn.cuh).
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <algorithm>
#include <atomic>
#include <mutex>
#include <string>
#include <vector>
#include <cub/device/device_radix_sort.cuh>

#include "host.cuh"
#include "fused_nn.cuh"
#include "masked_nn.cuh"

namespace b2d {

// process-wide tuning / test hooks (b2d_set_option): nothing on the hot path reads the environment
static std::atomic<float> g_nn_tau{6.0f};   // screened fusedL2NN: candidates per row above which the trial calls screening off
static std::atomic<int> g_nn_screen{1};     // 0: always the exact arg-min kernel

void minloc_init(cudaStream_t s, unsigned grid, long long* keys, int64_t m)
{
  minloc_init_kernel<<<grid, 256, 0, s>>>(keys, m);
}

void masked_group_map(cudaStream_t s, unsigned grid, int* grp, const int* group_idxs, int64_t G, int64_t n)
{
  masked_group_map_kernel<<<grid, 256, 0, s>>>(grp, group_idxs, G, n);
}

}  // namespace b2d

using namespace b2d;

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

size_t b2d_fused_l2_nn_workspace_bytes(int64_t m, int64_t n, int64_t k)
{
  if (m < 0 || n < 0 || k < 0) return static_cast<size_t>(-1);
  return tc_layout(nullptr, m, n, k, true).bytes;
}

// one chunk of y (prep + search); keys carry the result so far (and act as the rows' bounds)
static int fused_nn_keys_chunk(cudaStream_t s, int64_t* keys, const float* x, int64_t ldx, const float* y, int64_t ldy,
                               const float* xn, const float* yn, int64_t m, int64_t n, int64_t k, int64_t idx_offset,
                               void* workspace, const TcMetric& tm, bool allow_screen, bool have_bounds)
{
  TcWorkspace w = tc_layout(workspace, m, n, k, true);
  const int nkb = static_cast<int>((k + 31) / 32);
  // (k <= 64: the exact kernel is already epilogue-bound, screening would not pay)
  const bool screen = (tm.mode == PREP_L2 || tm.mode == PREP_COSINE) && nkb >= 3 && nkb <= TC_MAX_RES_KB && n >= 16384 &&
                      allow_screen;
  const int unit_norm = tm.mode == PREP_COSINE ? 1 : 0;
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
  int rc = launch_prep<float>(s, w, x, ldx, 1, m, y, ldy, 1, n, k, xn, yn, tm, col_map);
  if (rc) return rc;
  if (n == 0) return B2D_OK;
  TcParams p{};
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
                                          ldy, static_cast<int>(k), idx_offset, unit_norm, tm.center, static_cast<unsigned>(m), col_map);
  B2D_CUDA(cudaGetLastError());
  p.sel_lo = have_bounds ? 0 : 1; p.sel_hi = kSel; p.run_flag = flags + 3;
  rc = launch_tc(s, w, p, k, EPI_MINLOC, POST_NONE);
  if (rc) return rc;
  return B2D_OK;
}

static int fused_nn_keys(void* stream, int64_t* keys, const float* x, int64_t ldx, const float* y, int64_t ldy,
                         const float* xn, const float* yn, int64_t m, int64_t n, int64_t k, int64_t idx_offset,
                         int init_keys, void* workspace, size_t workspace_bytes, const TcMetric& tm)
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
  const bool screen_ok = (tm.mode == PREP_L2 || tm.mode == PREP_COSINE) && nkb_all >= 3 && nkb_all <= TC_MAX_RES_KB && !screen_off;
  constexpr int64_t kChunkRows = kNnChunkRows;
  if (!screen_ok || n <= kChunkRows)
    return fused_nn_keys_chunk(s, keys, x, ldx, y, ldy, xn, yn, m, n, k, idx_offset, workspace, tm, screen_ok,
                               init_keys == 0);
  for (int64_t off = 0; off < n; off += kChunkRows) {
    const int64_t nc = std::min<int64_t>(kChunkRows, n - off);
    int rc = fused_nn_keys_chunk(s, keys, x, ldx, y + off * ldy, ldy, xn, yn ? yn + off : nullptr, m, nc, k,
                                 idx_offset + off, workspace, tm, true, init_keys == 0 || off > 0);
    if (rc) return rc;
  }
  return B2D_OK;
}

int b2d_fused_l2_nn_keys(void* stream, int64_t* keys, const float* x, int64_t ldx, const float* y, int64_t ldy,
                         const float* xn, const float* yn, int64_t m, int64_t n, int64_t k, int64_t idx_offset,
                         int init_keys, void* workspace, size_t workspace_bytes)
{
  return fused_nn_keys(stream, keys, x, ldx, y, ldy, xn, yn, m, n, k, idx_offset, init_keys, workspace,
                       workspace_bytes, TC_L2);
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

// fusedL2NN and fusedDistanceNN: the keys of every row in the workspace, then unpacked into out (the square root taken
// for POST_CLAMP_SQRT).  (The cosine family, mode PREP_COSINE: rows are normalised in prep, keys hold -cos, the row term
// t_x = 1 turns it into 1 - cos.)
static int fused_nn(void* stream, b2d_kvp_if* out, const float* x, int64_t ldx, const float* y, int64_t ldy,
                    const float* xn, const float* yn, int64_t m, int64_t n, int64_t k, const TcMetric& tm, int init_out,
                    void* workspace, size_t workspace_bytes)
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
                     workspace_bytes, tm);
  if (rc) return rc;
  minloc_finalize_kernel<<<static_cast<unsigned>((m + 255) / 256), 256, 0, s>>>(
    reinterpret_cast<KvpIF*>(out), w.keys, m, tm.post == POST_CLAMP_SQRT ? 1 : 0, init_out ? 0 : 1);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

int b2d_fused_l2_nn(void* stream, b2d_kvp_if* out, const float* x, int64_t ldx, const float* y, int64_t ldy,
                    const float* xn, const float* yn, int64_t m, int64_t n, int64_t k, int do_sqrt, int init_out,
                    void* workspace, size_t workspace_bytes)
{
  TcMetric tm;
  tc_metric(do_sqrt ? B2D_L2SqrtExpanded : B2D_L2Expanded, k, &tm);
  return fused_nn(stream, out, x, ldx, y, ldy, xn, yn, m, n, k, tm, init_out, workspace, workspace_bytes);
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
  TcMetric tm;
  if ((metric != B2D_L2Expanded && metric != B2D_L2SqrtExpanded && metric != B2D_CosineExpanded &&
       metric != B2D_CorrelationExpanded) || !tc_metric(metric, k, &tm))
    return fail(B2D_ERR_UNSUPPORTED, "fusedDistanceNN supports L2Expanded, L2SqrtExpanded, CosineExpanded, CorrelationExpanded");
  // (xn / yn are the squared norms of the L2 metrics; the cosine family computes its own)
  const bool l2 = tm.mode == PREP_L2;
  return fused_nn(stream, out, x, ldx, y, ldy, l2 ? xn : nullptr, l2 ? yn : nullptr, m, n, k, tm, init_out, workspace,
                  workspace_bytes);
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

namespace b2d {
int masked_keys(cudaStream_t s, const TcWorkspace& w, long long* keys, const int* grp, unsigned* bits, uint8_t* cls,
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
  TcParams p{};
  p.m = m; p.n = n; p.keys = keys;
  p.mask_cls = cls; p.mask_grp = grp; p.mask_bits = bits; p.mask_groups = G;
  ProfileScope prof(s);
  return launch_tc(s, w, p, k, EPI_MINLOC_MASKED, POST_NONE);
}
}  // namespace b2d

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
    rc = launch_prep<float>(s, L.w, x, ldx, 1, m, y, ldy, 1, n, k, xn, yn, TC_L2);
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
