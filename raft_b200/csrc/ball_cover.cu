// Random ball cover (raft::neighbors::ball_cover before the move to cuVS): exact kNN and epsilon queries for 2-D and 3-D
// points under the unexpanded L2 distances.  The build samples landmarks, puts every row in the ball of its nearest
// landmark and stores the rows sorted by (ball, s to the landmark); the queries (ball_cover.cuh) walk the balls and skip
// what the triangle inequality rules out, with the rounding margin of ball_cover.cuh.  DESIGN.md K19.
#include <cuda_runtime.h>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <algorithm>
#include <cmath>
#include <string>

#include "ball_cover_build.cuh"
#include "host.cuh"

using namespace b2d;

int64_t b2d::bc_landmarks(int64_t n, int64_t nl)
{
  if (nl > 0) return nl;
  int64_t r = static_cast<int64_t>(std::sqrt(static_cast<double>(n)));
  while (r * r < n) ++r;
  while (r > 1 && (r - 1) * (r - 1) >= n) --r;
  return r;
}

BcLayout b2d::bc_layout(void* base, int64_t n, int64_t d, int64_t nl)
{
  Carve c(base, 256);
  BcLayout L;
  L.ix.lm  = c.take<float>(nl * d);
  L.ix.rhi = c.take<float>(nl);
  L.ix.off = c.take<int>(nl + 2);
  L.ix.pts = c.take<float>(n * d);
  L.ix.ids = c.take<int>(n);
  L.ix.rl  = c.take<float>(n);
  L.bytes  = c.bytes;
  return L;
}

BcBuildLayout b2d::bc_build_layout(void* base, int64_t n)
{
  Carve c(base, 256);
  BcBuildLayout L;
  for (int b = 0; b < 2; ++b) L.keys[b] = c.take<unsigned long long>(n);
  for (int b = 0; b < 2; ++b) L.vals[b] = c.take<int>(n);
  L.tmp_bytes = bc_sort_bytes(n);
  L.tmp       = c.take<char>(L.tmp_bytes);
  L.bytes     = c.bytes;
  return L;
}

namespace {

// The epsilon queries' workspace: the scan's look-back state (at most one 16-byte word per 64 rows), then, for fill,
// the sort's second key buffer [nnz] and its scratch.
struct BcEpsLayout {
  void* scan_tmp;
  size_t scan_bytes;
  long long* alt;
  void* sort_tmp;
  size_t sort_bytes;
  size_t bytes;
};

BcEpsLayout bc_eps_layout(void* base, int64_t m, int64_t nnz)
{
  Carve c(base, 256);
  BcEpsLayout L;
  L.scan_bytes = 16 * static_cast<size_t>(m / 64 + 256);
  L.scan_tmp   = c.take<char>(L.scan_bytes);
  L.alt        = c.take<long long>(nnz);
  L.sort_bytes = nnz > 0 ? kRowSortBytes : 0;
  L.sort_tmp   = c.take<char>(L.sort_bytes);
  L.bytes      = c.bytes;
  return L;
}

// the description of an index every call takes (the values given to the build)
int bc_check_index(const void* index, int64_t n, int64_t d, int metric, int64_t nl)
{
  if (metric != B2D_L2Unexpanded && metric != B2D_L2SqrtUnexpanded)
    return fail(B2D_ERR_UNSUPPORTED, "ball_cover supports L2Unexpanded and L2SqrtUnexpanded, got metric " +
                                         std::to_string(metric));
  if (d != 2 && d != 3) return fail(B2D_ERR_UNSUPPORTED, "ball_cover supports d = 2 and d = 3, got d = " + std::to_string(d));
  if (n < 1) return fail(B2D_ERR_INVALID_ARG, "n must be positive");
  if (n > 0x7fffffffll) return fail(B2D_ERR_INVALID_ARG, "n must be below 2^31");
  if (nl < 0 || nl > n) return fail(B2D_ERR_INVALID_ARG, "n_landmarks must be in [0, n] (0: ceil(sqrt(n)))");
  if (!index) return fail(B2D_ERR_INVALID_ARG, "null index");
  if (reinterpret_cast<uintptr_t>(index) % 256) return fail(B2D_ERR_INVALID_ARG, "index must be 256-byte aligned");
  return B2D_OK;
}

// the queries' arguments besides the index
int bc_check_queries(const float* q, int64_t ldq, int64_t m, int64_t d)
{
  if (m < 0) return fail(B2D_ERR_INVALID_ARG, "negative extent");
  if (m > 0x7fffffffll) return fail(B2D_ERR_INVALID_ARG, "m must be below 2^31");
  if (m > 0 && !q) return fail(B2D_ERR_INVALID_ARG, "null queries");
  if (ldq < d) return fail(B2D_ERR_INVALID_ARG, "ldq smaller than d");
  return B2D_OK;
}

unsigned bc_grid(int64_t items, int sms) { return static_cast<unsigned>(std::max<int64_t>(1, std::min<int64_t>((items + 255) / 256, int64_t(sms) * 16))); }

}  // namespace

template <int D>
int b2d::bc_build(cudaStream_t s, const BcIndex& ix, const BcBuildLayout& W, const float* x, int64_t ldx, int n, int nl,
                  uint64_t seed)
{
  int sms = 0;
  int rc  = device_sms(&sms);
  if (rc) return rc;
  // 1. landmarks: the first nl rows by a seeded hash, finite rows first
  bc_sample_kernel<D><<<bc_grid(n, sms), 256, 0, s>>>(x, ldx, n, seed, W.keys[0]);
  B2D_CUDA(cudaGetLastError());
  cub::DoubleBuffer<unsigned long long> keys(W.keys[0], W.keys[1]);
  size_t need = 0;
  B2D_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, need, keys, n, 0, 64, s));
  if (need > W.tmp_bytes) return fail(B2D_ERR_WORKSPACE, "internal: sort scratch " + std::to_string(need) + " bytes");
  B2D_CUDA(cub::DeviceRadixSort::SortKeys(W.tmp, need, keys, n, 0, 64, s));
  bc_landmark_kernel<D><<<bc_grid(nl, sms), 256, 0, s>>>(x, ldx, keys.Current(), nl, ix.lm);
  B2D_CUDA(cudaGetLastError());
  // 2. every row to its nearest landmark; 3. rows sorted by (landmark, s to it, row)
  unsigned long long* k0 = keys.Current() == W.keys[0] ? W.keys[1] : W.keys[0];
  bc_assign_kernel<D><<<static_cast<unsigned>((n + 255) / 256), 256, 0, s>>>(x, ldx, n, ix.lm, nl, k0, W.vals[0]);
  B2D_CUDA(cudaGetLastError());
  cub::DoubleBuffer<unsigned long long> pk(k0, k0 == W.keys[0] ? W.keys[1] : W.keys[0]);
  cub::DoubleBuffer<int> pv(W.vals[0], W.vals[1]);
  int end_bit = 32;
  while ((int64_t(1) << (end_bit - 32)) <= nl) ++end_bit;   // labels 0 .. nl
  B2D_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, need, pk, pv, n, 0, end_bit, s));
  if (need > W.tmp_bytes) return fail(B2D_ERR_WORKSPACE, "internal: sort scratch " + std::to_string(need) + " bytes");
  B2D_CUDA(cub::DeviceRadixSort::SortPairs(W.tmp, need, pk, pv, n, 0, end_bit, s));
  // 4. offsets, rows in position order, radii
  bc_offsets_kernel<<<bc_grid(int64_t(n) + 1, sms), 256, 0, s>>>(pk.Current(), n, nl, ix.off);
  B2D_CUDA(cudaGetLastError());
  bc_permute_kernel<D><<<bc_grid(n, sms), 256, 0, s>>>(x, ldx, pk.Current(), pv.Current(), n, ix.pts, ix.ids, ix.rl);
  B2D_CUDA(cudaGetLastError());
  bc_radius_kernel<<<bc_grid(nl, sms), 256, 0, s>>>(ix.off, ix.rl, nl, ix.rhi);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}
template int b2d::bc_build<2>(cudaStream_t, const BcIndex&, const BcBuildLayout&, const float*, int64_t, int, int, uint64_t);
template int b2d::bc_build<3>(cudaStream_t, const BcIndex&, const BcBuildLayout&, const float*, int64_t, int, int, uint64_t);

size_t b2d_ball_cover_index_bytes(int64_t n, int64_t d, int64_t n_landmarks)
{
  if (n < 1 || n > 0x7fffffffll || (d != 2 && d != 3) || n_landmarks < 0 || n_landmarks > n) return static_cast<size_t>(-1);
  return bc_layout(nullptr, n, d, bc_landmarks(n, n_landmarks)).bytes;
}

size_t b2d_ball_cover_build_workspace_bytes(int64_t n, int64_t d, int64_t n_landmarks)
{
  if (b2d_ball_cover_index_bytes(n, d, n_landmarks) == static_cast<size_t>(-1)) return static_cast<size_t>(-1);
  return bc_build_layout(nullptr, n).bytes;
}

int b2d_ball_cover_build(void* stream, void* index, const float* x, int64_t ldx, int64_t n, int64_t d, int metric,
                         int64_t n_landmarks, uint64_t seed, void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  int rc         = bc_check_index(index, n, d, metric, n_landmarks);
  if (rc) return rc;
  if (!x) return fail(B2D_ERR_INVALID_ARG, "null x");
  if (ldx < d) return fail(B2D_ERR_INVALID_ARG, "ldx smaller than d");
  rc = check_workspace(workspace, workspace_bytes, bc_build_layout(nullptr, n).bytes);
  if (rc) return rc;
  const int64_t nl          = bc_landmarks(n, n_landmarks);
  const BcIndex ix          = bc_layout(index, n, d, nl).ix;
  const BcBuildLayout W     = bc_build_layout(workspace, n);
  return d == 2 ? bc_build<2>(s, ix, W, x, ldx, static_cast<int>(n), static_cast<int>(nl), seed)
                : bc_build<3>(s, ix, W, x, ldx, static_cast<int>(n), static_cast<int>(nl), seed);
}

int b2d_ball_cover_knn(void* stream, int64_t* out_idx, float* out_dist, const void* index, int64_t n, int64_t d,
                       int metric, int64_t n_landmarks, const float* q, int64_t ldq, int64_t m, int64_t k)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  int rc         = bc_check_index(index, n, d, metric, n_landmarks);
  if (rc) return rc;
  rc = bc_check_queries(q, ldq, m, d);
  if (rc) return rc;
  if (k < 1 || k > n) return fail(B2D_ERR_INVALID_ARG, "k must be in [1, n]");
  if (k > 64) return fail(B2D_ERR_UNSUPPORTED, "k > 64 is not supported");
  if (m > 0 && (!out_idx || !out_dist)) return fail(B2D_ERR_INVALID_ARG, "null out_idx / out_dist");
  if (m == 0) return B2D_OK;
  const int64_t nl = bc_landmarks(n, n_landmarks);
  const BcIndex ix = bc_layout(const_cast<void*>(index), n, d, nl).ix;
  const int root   = metric == B2D_L2SqrtUnexpanded;
  const int ni = static_cast<int>(n), nli = static_cast<int>(nl), mi = static_cast<int>(m), ki = static_cast<int>(k);
  return d == 2 ? bc_walk_launch(s, bc_knn_kernel<2>, m, nl, d, ix, ni, nli, root, q, ldq, mi, ki, out_idx, out_dist)
                : bc_walk_launch(s, bc_knn_kernel<3>, m, nl, d, ix, ni, nli, root, q, ldq, mi, ki, out_idx, out_dist);
}

size_t b2d_ball_cover_eps_workspace_bytes(int64_t m, int64_t nnz)
{
  if (m < 0 || nnz < 0) return static_cast<size_t>(-1);
  return bc_eps_layout(nullptr, m, nnz).bytes;
}

int b2d_ball_cover_eps_count(void* stream, int64_t* indptr, const void* index, int64_t n, int64_t d, int metric,
                             int64_t n_landmarks, const float* q, int64_t ldq, int64_t m, float eps, void* workspace,
                             size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  int rc         = bc_check_index(index, n, d, metric, n_landmarks);
  if (rc) return rc;
  rc = bc_check_queries(q, ldq, m, d);
  if (rc) return rc;
  if (!indptr) return fail(B2D_ERR_INVALID_ARG, "null indptr");
  if (m > 0) {
    rc = check_workspace(workspace, workspace_bytes, bc_eps_layout(nullptr, m, 0).bytes);
    if (rc) return rc;
  }
  if (m == 0 || !(eps >= 0.f)) {   // no pairs (a NaN or negative eps matches nothing)
    B2D_CUDA(cudaMemsetAsync(indptr, 0, static_cast<size_t>(m + 1) * sizeof(int64_t), s));
    return B2D_OK;
  }
  const int64_t nl     = bc_landmarks(n, n_landmarks);
  const BcIndex ix     = bc_layout(const_cast<void*>(index), n, d, nl).ix;
  const BcEpsLayout L  = bc_eps_layout(workspace, m, 0);
  const int root       = metric == B2D_L2SqrtUnexpanded;
  const int ni = static_cast<int>(n), nli = static_cast<int>(nl), mi = static_cast<int>(m);
  rc = d == 2 ? bc_walk_launch(s, bc_eps_kernel<2>, m, nl, d, ix, ni, nli, root, q, ldq, mi, eps, indptr, nullptr, 0)
              : bc_walk_launch(s, bc_eps_kernel<3>, m, nl, d, ix, ni, nli, root, q, ldq, mi, eps, indptr, nullptr, 0);
  if (rc) return rc;
  size_t need = 0;
  B2D_CUDA(cub::DeviceScan::InclusiveSum(nullptr, need, indptr + 1, indptr + 1, m, s));
  if (need > L.scan_bytes) return fail(B2D_ERR_WORKSPACE, "internal: scan scratch " + std::to_string(need) + " bytes");
  B2D_CUDA(cub::DeviceScan::InclusiveSum(L.scan_tmp, need, indptr + 1, indptr + 1, m, s));
  return B2D_OK;
}

int b2d_ball_cover_eps_fill(void* stream, const int64_t* indptr, int64_t nnz, int64_t* indices, float* distances,
                            const void* index, int64_t n, int64_t d, int metric, int64_t n_landmarks, const float* q,
                            int64_t ldq, int64_t m, float eps, void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  int rc         = bc_check_index(index, n, d, metric, n_landmarks);
  if (rc) return rc;
  rc = bc_check_queries(q, ldq, m, d);
  if (rc) return rc;
  if (!indptr) return fail(B2D_ERR_INVALID_ARG, "null indptr");
  if (nnz < 0) return fail(B2D_ERR_INVALID_ARG, "negative nnz");
  if (nnz > 0x7fffffffll)
    return fail(B2D_ERR_UNSUPPORTED, "nnz = " + std::to_string(nnz) +
                                         " exceeds 2^31 - 1 pairs per call: split the queries into smaller batches");
  if (nnz > 0 && (!indices || !distances)) return fail(B2D_ERR_INVALID_ARG, "null indices / distances");
  if (m > 0) {
    rc = check_workspace(workspace, workspace_bytes, bc_eps_layout(nullptr, m, nnz).bytes);
    if (rc) return rc;
  }
  if (m == 0 || nnz == 0 || !(eps >= 0.f)) return B2D_OK;
  const int64_t nl     = bc_landmarks(n, n_landmarks);
  const BcIndex ix     = bc_layout(const_cast<void*>(index), n, d, nl).ix;
  const BcEpsLayout L  = bc_eps_layout(workspace, m, nnz);
  const int root       = metric == B2D_L2SqrtUnexpanded;
  long long* keys      = reinterpret_cast<long long*>(indices);
  int64_t* ip          = const_cast<int64_t*>(indptr);
  const int ni = static_cast<int>(n), nli = static_cast<int>(nl), mi = static_cast<int>(m);
  rc = d == 2 ? bc_walk_launch(s, bc_eps_kernel<2>, m, nl, d, ix, ni, nli, root, q, ldq, mi, eps, ip, keys, nnz)
              : bc_walk_launch(s, bc_eps_kernel<3>, m, nl, d, ix, ni, nli, root, q, ldq, mi, eps, ip, keys, nnz);
  if (rc) return rc;
  return radius_sort_split(s, indptr, m, nnz, indices, distances, L.alt, L.sort_tmp, L.sort_bytes);
}
