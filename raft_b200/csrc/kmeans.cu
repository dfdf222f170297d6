// k-means (kmeans.cuh), and the stable counting sort of rows by label that single linkage and DBSCAN run too.
#include <cuda_runtime.h>
#include <algorithm>
#include <cmath>
#include <string>

#include "host.cuh"
#include "kmeans.cuh"

using namespace b2d;

// ------------------------------------------------------------------------------------------
// k-means (kmeans.cuh): Lloyd's iterations on the exact EPI_MINLOC arg-min, the deterministic centroid update and the
// k-means++ / Random initialisations.  Every call only enqueues work; the loop of a fit runs max_iter conditional
// iterations on the device (run word in KmCtrl).
namespace b2d {
constexpr int64_t kKmHistCap = 1ll << 24;   // histogram words (n_clusters x row blocks) the layout allows

KmSortPlan km_sort_plan(int64_t m, int64_t nc)
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

KmSort km_sort_regions(Carve& c, int64_t m, int64_t nc, bool any_count)
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

int km_scan(cudaStream_t s, const unsigned* run, unsigned* a, int64_t n, unsigned* tiles, KmCtrl* ctrl)
{
  const unsigned ntiles = static_cast<unsigned>((n + kKmScanTile - 1) / kKmScanTile);
  km_scan_tiles_kernel<<<ntiles, kKmThreads, 0, s>>>(run, a, n, tiles);
  km_scan_kernel<<<ntiles, kKmThreads, 0, s>>>(run, a, n, tiles, ctrl);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

int km_sort_count(cudaStream_t s, const KmSort& S, const KmSortPlan& P, const int* labels, int64_t m, int64_t nc)
{
  km_begin_kernel<<<km_grid(P.nhist), 256, 0, s>>>(nullptr, nullptr, 0, nullptr, nullptr, S.hist, P.nhist);
  km_assign_kernel<<<static_cast<unsigned>(P.nblk), kKmThreads, 0, s>>>(nullptr, nullptr, const_cast<int*>(labels), nullptr, m,
                                                                        static_cast<int>(nc), P.rb, P.nblk, S.hist, nullptr);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

int km_sort_scatter(cudaStream_t s, const unsigned* run, const KmSort& S, const KmSortPlan& P, const int* labels,
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

void km_gather_rows(cudaStream_t s, unsigned grid, const float* x, int64_t ldx, int k, const int* idx, int nc, float* out)
{
  km_gather_rows_kernel<int><<<grid, 128, 0, s>>>(x, ldx, k, idx, nc, out);
}
}  // namespace b2d

namespace b2d {
KmLayout km_layout(void* base, int64_t m, int64_t k, int64_t nc)
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

int km_args(const float* x, int64_t ldx, int64_t m, int64_t k, int64_t nc, const void* c)
{
  if (m < 0 || k < 0) return fail(B2D_ERR_INVALID_ARG, "negative extent");
  if (k < 1 || k > (1 << 24)) return fail(B2D_ERR_INVALID_ARG, "k must be in [1, 2^24]");
  if (m > 0x7fffffffll) return fail(B2D_ERR_INVALID_ARG, "m must be below 2^31");
  if (nc < 1 || nc > m) return fail(B2D_ERR_INVALID_ARG, "n_clusters must be in [1, m]");
  if (!x || !c) return fail(B2D_ERR_INVALID_ARG, "null x / centroids");
  if (ldx < k) return fail(B2D_ERR_INVALID_ARG, "leading dimension smaller than k");
  return B2D_OK;
}

// the start of an assignment: keys <- KEY_EMPTY, histogram <- 0, and the centroids prepared again when prep_y
int km_assign_prep(cudaStream_t s, const KmLayout& L, int64_t m, int64_t k, int64_t nc, const float* c, const unsigned* run,
                   bool prep_y, bool hist)
{
  const int64_t nh = hist ? L.P.nhist : 0;
  // (the centroid side's exponent and scale flag are zeroed only where it is prepared again below)
  km_begin_kernel<<<km_grid(std::max(m, nh)), 256, 0, s>>>(run, L.tc.keys, m, prep_y ? L.tc.gmax : nullptr, L.tc.nonuni,
                                                           hist ? L.sort.hist : nullptr, nh);
  B2D_CUDA(cudaGetLastError());
  if (prep_y) {
    int rc = launch_prep<float>(s, L.tc, nullptr, 0, 1, m, c, k, 1, nc, k, nullptr, nullptr, TC_L2, nullptr, true, run);
    if (rc) return rc;
  }
  return B2D_OK;
}

// the end of an assignment: labels from the keys, inertia partials, label histogram (when hist)
int km_assign_labels(cudaStream_t s, const KmLayout& L, int64_t m, int64_t nc, const float* w, int* labels,
                     const unsigned* run, bool hist)
{
  km_assign_kernel<<<static_cast<unsigned>(L.P.nblk), kKmThreads, 0, s>>>(run, L.tc.keys, labels, w, m, static_cast<int>(nc),
                                                                          L.P.rb, L.P.nblk, hist ? L.sort.hist : nullptr,
                                                                          L.ipart);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

// arg-min of every row against the prepared centroids: labels, inertia partials, label histogram (when hist)
int km_assign(cudaStream_t s, const KmLayout& L, int64_t m, int64_t k, int64_t nc, const float* c, const float* w,
              int* labels, const unsigned* run, bool prep_y, bool hist)
{
  int rc = km_assign_prep(s, L, m, k, nc, c, run, prep_y, hist);
  if (rc) return rc;
  TcParams p{};
  p.m = m; p.n = nc; p.keys = L.tc.keys; p.run_flag = run;
  rc = launch_tc(s, L.tc, p, k, EPI_MINLOC, POST_NONE);
  if (rc) return rc;
  return km_assign_labels(s, L, m, nc, w, labels, run, hist);
}

// new centroids from the histogram km_assign (or km_sort_count) left: scan, stable scatter, fp64 sums
int km_update(cudaStream_t s, const KmLayout& L, const float* x, int64_t ldx, int64_t m, int64_t k, int64_t nc,
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
const float* km_weights(cudaStream_t s, const KmLayout& L, const float* w, int64_t m, bool normalize)
{
  if (!w) return nullptr;
  km_wsum_kernel<<<static_cast<unsigned>(L.nb), kKmThreads, 0, s>>>(w, m, L.bs, L.ctrl);
  km_wscale_kernel<<<1, kKmThreads, 0, s>>>(L.bs, L.nb, m, L.ctrl);
  if (!normalize) return w;
  km_wapply_kernel<<<km_grid(m), 256, 0, s>>>(w, L.w, m, L.ctrl);
  return L.w;
}

int km_plus_plus(cudaStream_t s, const KmLayout& L, const float* x, int64_t ldx, const float* w, int64_t m, int64_t k,
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

int km_fit_args(const double* inertia, const int32_t* n_iter, int max_iter, double tol, int init, int n_init)
{
  if (!inertia || !n_iter) return fail(B2D_ERR_INVALID_ARG, "null inertia / n_iter");
  if (max_iter < 0) return fail(B2D_ERR_INVALID_ARG, "max_iter must be >= 0");
  if (!(tol >= 0.0)) return fail(B2D_ERR_INVALID_ARG, "tol must be >= 0");
  if (init != B2D_KMEANS_INIT_PLUS_PLUS && init != B2D_KMEANS_INIT_RANDOM && init != B2D_KMEANS_INIT_ARRAY)
    return fail(B2D_ERR_INVALID_ARG, "unknown init method " + std::to_string(init));
  if (n_init < 1) return fail(B2D_ERR_INVALID_ARG, "n_init must be >= 1");
  return B2D_OK;
}

int km_fit_runs(cudaStream_t s, const KmLayout& L, const float* x, int64_t ldx, const float* w, int64_t m, int64_t k,
                int64_t nc, int max_iter, double tol, int inertia_check, int runs, float* centroids, double* inertia,
                int32_t* n_iter, const std::function<int(int)>& seed_run)
{
  unsigned* run = &L.ctrl->run;
  for (int r = 0; r < runs; ++r) {
    int rc = seed_run(r);
    if (rc) return rc;
    km_fit_begin_kernel<<<1, 1, 0, s>>>(L.ctrl);
    B2D_CUDA(cudaGetLastError());
    if (r == 0) {   // x is prepared once per fit; every iteration prepares the centroids alone
      rc = launch_prep<float>(s, L.tc, x, ldx, 1, m, centroids, k, 1, nc, k, nullptr, nullptr, TC_L2);
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

void km_ctrl_init(cudaStream_t s, KmCtrl* ctrl) { km_ctrl_init_kernel<<<1, 1, 0, s>>>(ctrl); }

void km_par_keys(cudaStream_t s, const long long* fold_keys, float* d2, const float* w, int64_t m, uint64_t seed, int round,
                 float* key)
{
  km_par_keys_kernel<<<static_cast<unsigned>((m + 255) / 256), 256, 0, s>>>(fold_keys, d2, w, m, seed, round, key);
}

void km_par_take(cudaStream_t s, const float* x, int64_t ldx, int k, const int64_t* idx, int n, float* cand, int* ids,
                 float* d2)
{
  km_par_take_kernel<<<static_cast<unsigned>(n), 128, 0, s>>>(x, ldx, k, idx, n, cand, ids, d2);
}
}  // namespace b2d

namespace {
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
  rc = km_fit_args(inertia, n_iter, max_iter, tol, init, n_init);
  if (rc) return rc;
  const int64_t nc = n_clusters;
  rc = check_workspace(workspace, workspace_bytes, km_layout(nullptr, m, k, nc).bytes);
  if (rc) return rc;
  const KmLayout L = km_layout(workspace, m, k, nc);
  km_ctrl_init_kernel<<<1, 1, 0, s>>>(L.ctrl);
  B2D_CUDA(cudaGetLastError());
  const float* w = km_weights(s, L, sample_weight, m, true);
  B2D_CUDA(cudaGetLastError());
  const int runs = init == B2D_KMEANS_INIT_ARRAY ? 1 : n_init;
  return km_fit_runs(s, L, x, ldx, w, m, k, nc, max_iter, tol, inertia_check, runs, centroids, inertia, n_iter,
                     [&](int r) {
                       if (init == B2D_KMEANS_INIT_RANDOM) return km_random(s, L, x, ldx, m, k, nc, seed + r, centroids);
                       if (init == B2D_KMEANS_INIT_PLUS_PLUS) return km_plus_plus(s, L, x, ldx, w, m, k, nc, seed + r, centroids);
                       return static_cast<int>(B2D_OK);
                     });
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
  rc = launch_prep<float>(s, L.tc, x, ldx, 1, m, centroids, k, 1, nc, k, nullptr, nullptr, TC_L2);
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
