// Mean shift (mean_shift.cuh, DESIGN.md K18): sklearn.cluster.MeanShift on the epsilon neighbourhood of the tensor path.
#include <cuda.h>
#include <cuda_runtime.h>
#include <algorithm>
#include <cmath>
#include <cub/device/device_merge_sort.cuh>
#include <cub/device/device_radix_sort.cuh>

#include "host.cuh"
#include "mean_shift.cuh"

using namespace b2d;

namespace {
constexpr int64_t kMsDefaultBatchBytes = 1ll << 30;

// fp32 partials per seed of the neighbour sums: one per chunk of kMsChunk data rows
int64_t ms_nchunks(int64_t n) { return (n + kMsChunk - 1) / kMsChunk; }

// The workspace of a fit with n data rows and a seed capacity S (the caller's seed count, or n): the tensor path's
// operands for max(n, S) rows on both sides (seeds x data while iterating, candidates x candidates for the walk, data x
// centres for the labels), the seed state, one batch of adjacency and partials, and the sort regions.
struct MsLayout {
  TcWorkspace tc;
  int64_t S;
  int64_t b;          // seeds per batch (a multiple of 128)
  int64_t ld;         // adjacency row pitch: max(n, S) rounded up to 16
  int64_t nchunks;    // ceil(n / kMsChunk)
  MsCtrl* ctrl;
  KmCtrl* scan;       // [2] scan totals: survivors, distinct means
  float* mean;        // [S][d] the seeds' current means
  unsigned* state;    // [S] MsState
  int* iters;         // [S] completed iterations
  unsigned* inten;    // [S] |N| of the last step
  unsigned* flag;     // [max(n, S)] flags, scanned in place into positions
  unsigned* tiles;    // scan tile sums
  int* order;         // [S] seeds in mean order
  int* order2;        // [S] distinct means in walk order
  float* cand;        // [S][d] the candidates in walk order
  uint8_t* status;    // [S] walk status
  int* kept;          // [S] kept candidates
  unsigned* part_cnt; // [nchunks][b]
  float* part;        // [nchunks][b][d]
  long long* keys;    // [n] arg-min keys of the labels
  unsigned long long* hkey[2];  // [n] bin seeding: bin hashes
  int* hval[2];                 // [n] their rows
  unsigned* leader;   // [n]
  unsigned* freq;     // [n]
  void* tmp;          // cub scratch
  size_t tmp_bytes;
  uint8_t* adj;       // [b][ld]
  size_t bytes;
};

// seeds per batch: min(S rounded up to 128, max(128, floor(max_bytes / ld / 128) * 128)); max_bytes 0 means 2^30
int64_t ms_batch(int64_t S, int64_t ld, int64_t max_bytes)
{
  const int64_t mb = max_bytes > 0 ? max_bytes : kMsDefaultBatchBytes;
  const int64_t all = (std::max<int64_t>(S, 1) + kMsTileM - 1) / kMsTileM * kMsTileM;
  return std::min(all, std::max<int64_t>(kMsTileM, mb / ld / kMsTileM * kMsTileM));
}

MsLayout ms_layout(void* base, int64_t n, int64_t d, int64_t n_seeds, int64_t max_bytes)
{
  Carve c(base, 1024);
  MsLayout L{};
  L.S       = n_seeds > 0 ? n_seeds : n;
  const int64_t R = std::max(n, L.S);
  L.tc      = tc_layout(c, R, R, d, false);
  L.ld      = (std::max<int64_t>(R, 1) + 15) / 16 * 16;
  L.b       = ms_batch(L.S, L.ld, max_bytes);
  L.nchunks = ms_nchunks(n);
  L.ctrl    = c.take<MsCtrl>(1);
  L.scan    = c.take<KmCtrl>(2);
  L.mean    = c.take<float>(static_cast<size_t>(L.S) * d);
  L.state   = c.take<unsigned>(L.S);
  L.iters   = c.take<int>(L.S);
  L.inten   = c.take<unsigned>(L.S);
  L.flag    = c.take<unsigned>(R);
  L.tiles   = c.take<unsigned>((R + kKmScanTile - 1) / kKmScanTile);
  L.order   = c.take<int>(L.S);
  L.order2  = c.take<int>(L.S);
  L.cand    = c.take<float>(static_cast<size_t>(L.S) * d);
  L.status  = c.take<uint8_t>(L.S);
  L.kept    = c.take<int>(L.S);
  L.part_cnt = c.take<unsigned>(static_cast<size_t>(L.nchunks) * L.b);
  L.part    = c.take<float>(static_cast<size_t>(L.nchunks) * L.b * d);
  L.keys    = c.take<long long>(n);
  const int64_t nb = n_seeds > 0 ? 0 : n;   // bin seeding needs its regions only without caller seeds
  for (int i = 0; i < 2; ++i) {
    L.hkey[i] = c.take<unsigned long long>(nb);
    L.hval[i] = c.take<int>(nb);
  }
  L.leader    = c.take<unsigned>(nb);
  L.freq      = c.take<unsigned>(nb);
  L.tmp_bytes = (4u << 20) + 8 * static_cast<size_t>(R);
  L.tmp       = c.take<char>(L.tmp_bytes);
  L.adj       = c.take<uint8_t>(static_cast<size_t>(L.b) * L.ld);
  L.bytes     = c.bytes;
  return L;
}

unsigned ms_grid(int64_t n, int per) { return static_cast<unsigned>(std::max<int64_t>(1, (n + per - 1) / per)); }

// The adjacency of rows [r0, r0 + w) of the prepared x side against the n rows of the y side into L.adj (diag_off as
// TcParams: TC_NO_DIAG unless x and y are the same prepared matrix)
int ms_eps(cudaStream_t s, const MsLayout& L, int64_t r0, int64_t w, int64_t n, int64_t d, float e, int64_t diag_off,
           const unsigned* run)
{
  TcParams p{};
  p.m = w; p.n = n;
  p.adj = L.adj; p.ld_adj = L.ld; p.eps = e;
  p.diag_off = diag_off;
  p.run_flag = run;
  p.tma_store = n % 16 == 0 ? 1 : 0;   // (L.adj is 1024-byte aligned and L.ld a multiple of 16)
  return launch_tc(s, tc_rows(L.tc, 0, r0, d), p, d, EPI_EPS, POST_CLAMP);
}

template <int G>
int ms_sum_launch(cudaStream_t s, const CUtensorMap& ma, const CUtensorMap& mb, MsSumParams p, int grid)
{
  constexpr size_t smem = MsCarve<G>::bytes;
  p.stages = MsCarve<G>::stages;
  B2D_CUDA(cudaFuncSetAttribute(ms_sum_kernel<G>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  ms_sum_kernel<G><<<grid, kMsThreads, smem, s>>>(ma, mb, p);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

// How ms_sums cut its work (b2d_debug_mean_shift_sums reports it)
struct MsSumPlan {
  int gsz, ngroups, nchunks;
  int64_t n_items;
  int grid;
};

// The neighbour sums of the w seeds of adj [w][ld] (bytes, columns [0, n) read; ld a multiple of 16) against the n data
// rows prepared as the y side of tc: part [ms_nchunks(n)][w][d] and cnt [ms_nchunks(n)][w] (ms_sum_kernel)
int ms_sums(cudaStream_t s, const TcWorkspace& tc, const uint8_t* adj, int64_t ld, int64_t w, int64_t n, int64_t d,
            float* part, unsigned* cnt, const unsigned* run, MsSumPlan* plan = nullptr)
{
  int sms = 0;
  int rc  = device_sms(&sms);
  if (rc) return rc;
  MsSumParams p{};
  p.m = w; p.n = n; p.d = static_cast<int>(d); p.nkb = static_cast<int>((d + 31) / 32);
  p.gsz     = p.nkb >= 3 ? 4 : p.nkb;
  p.ngroups = (p.nkb + p.gsz - 1) / p.gsz;
  p.tiles_m = static_cast<int>((w + kMsTileM - 1) / kMsTileM);
  p.nchunks = static_cast<int>(ms_nchunks(n));
  p.n_items = static_cast<int64_t>(p.tiles_m) * p.nchunks * p.ngroups;
  p.ysc = tc.ysc; p.nonuni = tc.nonuni; p.part = part; p.cnt = cnt; p.run_flag = run;
  const int grid = static_cast<int>(std::min<int64_t>(p.n_items, sms));
  if (plan) *plan = MsSumPlan{p.gsz, p.ngroups, p.nchunks, p.n_items, grid};
  CUtensorMap ma, mb;
  rc = encode_2d(&ma, CU_TENSOR_MAP_DATA_TYPE_UINT8, adj, n, w, ld, kMsKs, kMsTileM, CU_TENSOR_MAP_SWIZZLE_128B,
                 CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "(mean_shift adj)");
  if (rc) return rc;
  rc = encode_2d(&mb, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, tc.yop, static_cast<int64_t>(p.nkb) * 64, n,
                 static_cast<int64_t>(p.nkb) * 128, 64, kMsKs, CU_TENSOR_MAP_SWIZZLE_128B,
                 CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "(mean_shift data)");
  if (rc) return rc;
  if (p.gsz == 1) return ms_sum_launch<1>(s, ma, mb, p, grid);
  if (p.gsz == 2) return ms_sum_launch<2>(s, ma, mb, p, grid);
  return ms_sum_launch<4>(s, ma, mb, p, grid);
}

// the data rows of tc's y side with a non-finite element out of every sum (ms_clear_nonfinite_kernel)
int ms_clear_nonfinite(cudaStream_t s, const TcWorkspace& tc, int64_t n, int64_t d)
{
  ms_clear_nonfinite_kernel<<<ms_grid(n, 256), 256, 0, s>>>(tc.yt, n, static_cast<int>((d + 31) / 32), tc.yop);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

__global__ void ms_ctrl_init_kernel(MsCtrl* ctrl)
{
  *ctrl     = MsCtrl{};
  ctrl->run = 1u;
}
__global__ void ms_finish_kernel(const MsCtrl* ctrl, int* n_centers, int* n_iter)
{
  if (n_centers) *n_centers = static_cast<int>(ctrl->n_kept);
  if (n_iter) *n_iter = ctrl->n_iter;
}

int ms_read(cudaStream_t s, const unsigned* dev, unsigned* host)
{
  B2D_CUDA(cudaMemcpyAsync(host, dev, sizeof(unsigned), cudaMemcpyDeviceToHost, s));
  B2D_CUDA(cudaStreamSynchronize(s));
  return B2D_OK;
}

template <class Cmp>
int ms_sort(cudaStream_t s, const MsLayout& L, int* keys, int64_t count, Cmp cmp)
{
  size_t need = 0;
  B2D_CUDA(cub::DeviceMergeSort::StableSortKeys(nullptr, need, keys, static_cast<int>(count), cmp, s));
  if (need > L.tmp_bytes) return fail(B2D_ERR_UNSUPPORTED, "mean_shift: internal sort scratch too small");
  B2D_CUDA(cub::DeviceMergeSort::StableSortKeys(L.tmp, need, keys, static_cast<int>(count), cmp, s));
  return B2D_OK;
}

// bin seeding into L.mean; *s_out = the seed count (read back: the iterations are sized by it)
int ms_bin_seeds(cudaStream_t s, const MsLayout& L, const float* x, int64_t ldx, int64_t n, int64_t d, double h,
                 int64_t min_bin_freq, int64_t* s_out)
{
  const int dd = static_cast<int>(d);
  ms_bin_hash_kernel<<<ms_grid(n, 256), 256, 0, s>>>(x, ldx, n, dd, h, L.hkey[0], L.hval[0]);
  B2D_CUDA(cudaGetLastError());
  cub::DoubleBuffer<unsigned long long> dk(L.hkey[0], L.hkey[1]);
  cub::DoubleBuffer<int> dv(L.hval[0], L.hval[1]);
  size_t need = 0;
  B2D_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, need, dk, dv, static_cast<int>(n), 0, 64, s));
  if (need > L.tmp_bytes) return fail(B2D_ERR_UNSUPPORTED, "mean_shift: internal sort scratch too small");
  B2D_CUDA(cub::DeviceRadixSort::SortPairs(L.tmp, need, dk, dv, static_cast<int>(n), 0, 64, s));
  B2D_CUDA(cudaMemsetAsync(L.freq, 0, static_cast<size_t>(n) * sizeof(unsigned), s));
  ms_bin_count_kernel<<<ms_grid(n, 256), 256, 0, s>>>(x, ldx, n, dd, h, dk.Current(), dv.Current(), L.leader, L.freq);
  B2D_CUDA(cudaGetLastError());
  const unsigned mf = static_cast<unsigned>(std::min<int64_t>(min_bin_freq, 0xffffffffll));
  ms_bin_flag_kernel<<<ms_grid(n, 256), 256, 0, s>>>(L.leader, L.freq, n, mf, L.flag);
  B2D_CUDA(cudaGetLastError());
  int rc = km_scan(s, nullptr, L.flag, n, L.tiles, L.scan);
  if (rc) return rc;
  ms_bin_seed_kernel<<<ms_grid(n, 8), 256, 0, s>>>(x, ldx, n, dd, h, L.leader, L.freq, mf, L.flag, &L.scan->total, L.mean);
  B2D_CUDA(cudaGetLastError());
  unsigned cnt = 0;
  rc = ms_read(s, &L.scan->total, &cnt);
  if (rc) return rc;
  *s_out = cnt;
  return B2D_OK;
}
}  // namespace

size_t b2d_mean_shift_fit_workspace_bytes(int64_t n, int64_t d, int64_t n_seeds, int64_t max_bytes_per_batch)
{
  if (n < 0 || d < 0 || n_seeds < 0 || max_bytes_per_batch < 0) return static_cast<size_t>(-1);
  return ms_layout(nullptr, n, d, n_seeds, max_bytes_per_batch).bytes;
}

int b2d_mean_shift_fit(void* stream, const float* x, int64_t ldx, int64_t n, int64_t d, double bandwidth,
                       const float* seeds, int64_t lds, int64_t n_seeds, int bin_seeding, int64_t min_bin_freq,
                       int cluster_all, int max_iter, int64_t max_bytes_per_batch, float* centers, int32_t* n_centers,
                       int32_t* labels, int32_t* n_iter, void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (n < 0 || d < 0 || n_seeds < 0 || max_bytes_per_batch < 0)
    return fail(B2D_ERR_INVALID_ARG, "negative extent, seed count or batch size");
  if (n > 0x7fffffffll || n_seeds > 0x7fffffffll) return fail(B2D_ERR_INVALID_ARG, "mean_shift: n and n_seeds must be below 2^31");
  if (d < 1) return fail(B2D_ERR_INVALID_ARG, "d must be positive");
  if (d > 320) return fail(B2D_ERR_UNSUPPORTED, "mean_shift supports d <= 320 (the whole distance at once)");
  if (!std::isfinite(bandwidth) || !(bandwidth > 0.0)) return fail(B2D_ERR_INVALID_ARG, "bandwidth must be finite and > 0");
  if (!std::isfinite(static_cast<float>(bandwidth * bandwidth)))
    return fail(B2D_ERR_INVALID_ARG, "bandwidth^2 is not finite in fp32");
  if (max_iter < 0) return fail(B2D_ERR_INVALID_ARG, "max_iter must be >= 0");
  if ((seeds == nullptr) != (n_seeds == 0)) return fail(B2D_ERR_INVALID_ARG, "seeds and n_seeds: both or neither");
  if (seeds && lds < d) return fail(B2D_ERR_INVALID_ARG, "seeds leading dimension smaller than d");
  if (bin_seeding && min_bin_freq < 1) return fail(B2D_ERR_INVALID_ARG, "min_bin_freq must be >= 1");
  if (n == 0) return fail(B2D_ERR_INVALID_ARG, "n must be positive");
  if (!x || !centers || !labels || !n_centers) return fail(B2D_ERR_INVALID_ARG, "null x / centers / labels / n_centers");
  if (ldx < d) return fail(B2D_ERR_INVALID_ARG, "leading dimension smaller than d");
  int rc = check_workspace(workspace, workspace_bytes, ms_layout(nullptr, n, d, n_seeds, max_bytes_per_batch).bytes);
  if (rc) return rc;
  const MsLayout L = ms_layout(workspace, n, d, n_seeds, max_bytes_per_batch);
  const float e    = static_cast<float>(bandwidth * bandwidth);
  const double thr = 1e-3 * bandwidth;
  unsigned* run    = &L.ctrl->run;
  const int dd     = static_cast<int>(d);

  // 1. seeds into L.mean [s][d]
  ms_ctrl_init_kernel<<<1, 1, 0, s>>>(L.ctrl);
  B2D_CUDA(cudaGetLastError());
  int64_t ns = n_seeds;
  if (seeds) {
    B2D_CUDA(cudaMemcpy2DAsync(L.mean, d * sizeof(float), seeds, lds * sizeof(float), d * sizeof(float), ns,
                               cudaMemcpyDeviceToDevice, s));
  } else if (bin_seeding) {
    rc = ms_bin_seeds(s, L, x, ldx, n, d, bandwidth, min_bin_freq, &ns);
    if (rc) return rc;
  } else {
    ns = n;
    B2D_CUDA(cudaMemcpy2DAsync(L.mean, d * sizeof(float), x, ldx * sizeof(float), d * sizeof(float), n,
                               cudaMemcpyDeviceToDevice, s));
  }
  if (ns == 0) {   // no bin reached min_bin_freq: no seed, no centre
    B2D_CUDA(cudaMemsetAsync(labels, 0xff, static_cast<size_t>(n) * sizeof(int32_t), s));
    ms_finish_kernel<<<1, 1, 0, s>>>(L.ctrl, n_centers, n_iter);
    B2D_CUDA(cudaGetLastError());
    return B2D_OK;
  }
  ms_init_kernel<<<ms_grid(ns, 256), 256, 0, s>>>(ns, L.state, L.iters, L.inten);
  B2D_CUDA(cudaGetLastError());

  // 2. the iterations: seeds prepared as x (every iteration), data as y (once); later iterations are no-ops on the
  //    device once no seed is active
  rc = launch_prep<float>(s, L.tc, L.mean, d, 1, ns, x, ldx, 1, n, d, nullptr, nullptr, TC_L2);
  if (rc) return rc;
  rc = ms_clear_nonfinite(s, L.tc, n, d);
  if (rc) return rc;
  for (int it = 0; it <= max_iter; ++it) {
    ProfileScope prof(s);
    if (it > 0) {
      rc = launch_prep<float>(s, L.tc, L.mean, d, 1, ns, nullptr, 0, 1, 0, d, nullptr, nullptr, TC_L2, nullptr, false,
                              run, true);
      if (rc) return rc;
    }
    for (int64_t r0 = 0; r0 < ns; r0 += L.b) {
      const int64_t w = std::min(L.b, ns - r0);
      rc = ms_eps(s, L, r0, w, n, d, e, TC_NO_DIAG, run);
      if (rc) return rc;
      rc = ms_sums(s, L.tc, L.adj, L.ld, w, n, d, L.part, L.part_cnt, run);
      if (rc) return rc;
      ms_update_kernel<<<ms_grid(w, 8), 256, 0, s>>>(run, L.part, L.part_cnt, static_cast<int>(L.nchunks), w, r0, dd,
                                                     L.tc.gmax, thr, max_iter, L.mean, L.state, L.iters, L.inten, L.ctrl);
      B2D_CUDA(cudaGetLastError());
    }
    ms_step_end_kernel<<<1, 1, 0, s>>>(L.ctrl);
    B2D_CUDA(cudaGetLastError());
  }

  // 3. candidates: the survivors in mean order (dropped seeds last), one per run of bitwise-equal means
  ms_survive_kernel<<<ms_grid(ns, 256), 256, 0, s>>>(ns, L.state, L.iters, L.flag, L.ctrl);
  B2D_CUDA(cudaGetLastError());
  rc = km_scan(s, nullptr, L.flag, ns, L.tiles, &L.scan[0]);
  if (rc) return rc;
  ms_iota_kernel<<<ms_grid(ns, 256), 256, 0, s>>>(L.order, ns);
  B2D_CUDA(cudaGetLastError());
  rc = ms_sort(s, L, L.order, ns, MsByMean{L.mean, L.inten, L.state, dd});
  if (rc) return rc;
  ms_unique_kernel<<<ms_grid(ns, 256), 256, 0, s>>>(L.order, &L.scan[0].total, L.mean, dd, L.flag, ns);
  B2D_CUDA(cudaGetLastError());
  rc = km_scan(s, nullptr, L.flag, ns, L.tiles, &L.scan[1]);
  if (rc) return rc;
  ms_compact_kernel<<<ms_grid(ns, 256), 256, 0, s>>>(ns, L.order, L.flag, &L.scan[1].total, L.order2);
  B2D_CUDA(cudaGetLastError());
  unsigned nc = 0;
  rc = ms_read(s, &L.scan[1].total, &nc);
  if (rc) return rc;
  if (nc == 0) {   // no seed had a neighbour
    B2D_CUDA(cudaMemsetAsync(labels, 0xff, static_cast<size_t>(n) * sizeof(int32_t), s));
    ms_finish_kernel<<<1, 1, 0, s>>>(L.ctrl, n_centers, n_iter);
    B2D_CUDA(cudaGetLastError());
    return B2D_OK;
  }
  const int64_t C = nc;
  rc = ms_sort(s, L, L.order2, C, MsByIntensity{L.mean, L.inten, dd});
  if (rc) return rc;
  ms_gather_kernel<<<ms_grid(C, 8), 256, 0, s>>>(L.mean, dd, L.order2, C, L.cand);
  B2D_CUDA(cudaGetLastError());

  // 4. the greedy walk in batches of candidate rows against all candidates (one prepared matrix on both sides)
  rc = launch_prep<float>(s, L.tc, L.cand, d, 1, C, L.cand, d, 1, C, d, nullptr, nullptr, TC_L2);
  if (rc) return rc;
  B2D_CUDA(cudaMemsetAsync(L.status, 0, static_cast<size_t>(C), s));
  for (int64_t r0 = 0; r0 < C; r0 += L.b) {
    const int64_t w = std::min(L.b, C - r0);
    rc = ms_eps(s, L, r0, w, C, d, e, -r0, nullptr);
    if (rc) return rc;
    ms_walk_kernel<<<1, 1024, 0, s>>>(L.adj, L.ld, r0, w, C, L.status, L.kept, L.ctrl);
    B2D_CUDA(cudaGetLastError());
  }
  unsigned nk = 0;
  rc = ms_read(s, &L.ctrl->n_kept, &nk);
  if (rc) return rc;
  ms_gather_kernel<<<ms_grid(nk, 8), 256, 0, s>>>(L.cand, dd, L.kept, nk, centers);
  B2D_CUDA(cudaGetLastError());
  ms_finish_kernel<<<1, 1, 0, s>>>(L.ctrl, n_centers, n_iter);
  B2D_CUDA(cudaGetLastError());

  // 5. labels: the fused arg-min of the data against the kept centres
  rc = launch_prep<float>(s, L.tc, x, ldx, 1, n, centers, d, 1, nk, d, nullptr, nullptr, TC_L2);
  if (rc) return rc;
  minloc_init(s, sl_grid(n), L.keys, n);
  TcParams p{};
  p.m = n; p.n = nk; p.keys = L.keys;
  rc = launch_tc(s, L.tc, p, d, EPI_MINLOC, POST_NONE);
  if (rc) return rc;
  ms_label_kernel<<<ms_grid(n, 256), 256, 0, s>>>(L.keys, n, cluster_all, e, labels);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

int b2d_debug_mean_shift_sums(void* stream, const uint8_t* adj, int64_t ld_adj, int64_t m, const float* x, int64_t ldx,
                              int64_t n, int64_t d, float* part, uint32_t* counts, int32_t* exponent, int64_t* info,
                              void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (m < 1 || n < 1) return fail(B2D_ERR_INVALID_ARG, "m and n must be positive");
  if (m > 0x7fffffffll || n > 0x7fffffffll) return fail(B2D_ERR_INVALID_ARG, "mean_shift: m and n must be below 2^31");
  if (d < 1) return fail(B2D_ERR_INVALID_ARG, "d must be positive");
  if (d > 320) return fail(B2D_ERR_UNSUPPORTED, "mean_shift supports d <= 320 (the whole distance at once)");
  if (!adj || !x || !part || !counts || !exponent || !info)
    return fail(B2D_ERR_INVALID_ARG, "null adj / x / part / counts / exponent / info");
  if (ldx < d) return fail(B2D_ERR_INVALID_ARG, "leading dimension smaller than d");
  if (ld_adj < n || ld_adj % 16 != 0 || reinterpret_cast<uintptr_t>(adj) % 16 != 0)
    return fail(B2D_ERR_INVALID_ARG, "adjacency pitch must be >= n and a multiple of 16, on a 16-byte boundary");
  int rc = check_workspace(workspace, workspace_bytes, ms_layout(nullptr, n, d, m, 0).bytes);
  if (rc) return rc;
  const MsLayout L = ms_layout(workspace, n, d, m, 0);
  unsigned bad = 0;
  B2D_CUDA(cudaMemsetAsync(L.flag, 0, sizeof(unsigned), s));
  ms_adj_check_kernel<<<static_cast<unsigned>(std::min<int64_t>(ms_grid(m * n, 256), 4096)), 256, 0, s>>>(adj, ld_adj, m,
                                                                                                        n, L.flag);
  B2D_CUDA(cudaGetLastError());
  rc = ms_read(s, L.flag, &bad);
  if (rc) return rc;
  if (bad) return fail(B2D_ERR_INVALID_ARG, "adjacency bytes must be 0 or 1");
  // the data side of a fit: prepared, non-finite rows cleared, then the fit's launcher
  rc = launch_prep<float>(s, L.tc, nullptr, 0, 1, 0, x, ldx, 1, n, d, nullptr, nullptr, TC_L2);
  if (rc) return rc;
  rc = ms_clear_nonfinite(s, L.tc, n, d);
  if (rc) return rc;
  MsSumPlan plan{};
  rc = ms_sums(s, L.tc, adj, ld_adj, m, n, d, part, counts, nullptr, &plan);
  if (rc) return rc;
  ms_exponent_kernel<<<1, 1, 0, s>>>(L.tc.gmax, exponent);
  B2D_CUDA(cudaGetLastError());
  unsigned scaled = 0;
  rc = ms_read(s, L.tc.nonuni + 1, &scaled);
  if (rc) return rc;
  const int64_t out[6] = {plan.gsz, plan.ngroups, plan.nchunks, plan.n_items, plan.grid, scaled};
  std::copy(out, out + 6, info);
  return B2D_OK;
}
