// Radius neighbours (sklearn.neighbors.NearestNeighbors.radius_neighbors with sort_results=True): every pair of a query
// row and a dataset row within a radius, as CSR rows in (distance, index) order, without the m x n matrix.  The distance is
// the one b2d_pairwise_distance returns; the tensor kernel's EPI_RADIUS epilogue counts the pairs per row (count call) and
// appends them as packed keys (fill call), and a segmented radix sort orders each row.  (cub::DeviceSegmentedSort would
// copy its segment counts to the host and wait for them once m passes a few hundred rows: neither call may synchronise.)
#include <cuda_runtime.h>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_segmented_radix_sort.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <thrust/iterator/transform_iterator.h>
#include <algorithm>
#include <string>

#include "host.cuh"
#include "radius.cuh"

using namespace b2d;

namespace {

// The workspace of both calls: the tensor path's operands, the row degrees [m + 1] (the last one stays 0, so the exclusive
// scan of m + 1 words ends in nnz), the fill counters [m], the sort's second key buffer [nnz] and the CUB scratch.  CUB
// reports its scratch only with a device present, so the workspace holds a bound that the calls check at run time: the
// scan's look-back state of at most one 16-byte word per 64 rows, and kRowSortBytes for the segmented sort (fill only).
struct RadiusLayout {
  TcWorkspace w;
  unsigned* deg;
  unsigned* fill;
  long long* alt;
  void* scan_tmp;
  size_t scan_bytes;
  void* sort_tmp;
  size_t sort_bytes;
  size_t bytes;
};

RadiusLayout radius_layout(void* base, int64_t m, int64_t n, int64_t k, int64_t nnz)
{
  Carve c(base, 1024);
  RadiusLayout L;
  L.w          = tc_layout(c, m, n, k, false);
  L.deg        = c.take<unsigned>(m + 1);
  L.fill       = c.take<unsigned>(m);
  L.alt        = c.take<long long>(nnz);
  L.scan_bytes = 16 * static_cast<size_t>(m / 64 + 256);
  L.scan_tmp   = c.take<char>(L.scan_bytes);
  L.sort_bytes = nnz > 0 ? kRowSortBytes : 0;
  L.sort_tmp   = c.take<char>(L.sort_bytes);
  L.bytes      = c.bytes;
  return L;
}

// The argument checks both calls share.  *work: there are pairs to look at (m > 0 and n > 0).
int radius_check(int metric, const int64_t* indptr, const float* x, int64_t ldx, const float* y, int64_t ldy, int64_t m,
                 int64_t n, int64_t k, TcMetric* tm, bool* work)
{
  // (the distance of b2d_pairwise_distance)
  if ((metric != B2D_L2Expanded && metric != B2D_L2SqrtExpanded && metric != B2D_CosineExpanded &&
       metric != B2D_CorrelationExpanded) || !tc_metric(metric, k, tm))
    return fail(B2D_ERR_UNSUPPORTED, "radius_neighbors supports L2Expanded, L2SqrtExpanded, CosineExpanded and "
                                     "CorrelationExpanded, got metric " + std::to_string(metric));
  if (m < 0 || n < 0 || k < 0) return fail(B2D_ERR_INVALID_ARG, "negative extent");
  if (m > 0x7fffffffll || n > 0x7fffffffll) return fail(B2D_ERR_INVALID_ARG, "m and n must be below 2^31");
  if (!indptr) return fail(B2D_ERR_INVALID_ARG, "null indptr");
  *work = m > 0 && n > 0;
  if (!*work) return B2D_OK;
  if (k == 0) return fail(B2D_ERR_INVALID_ARG, "k must be positive");
  if (k > 320) return fail(B2D_ERR_UNSUPPORTED, "radius_neighbors supports k <= 320 (the whole distance at once)");
  if (!x || !y) return fail(B2D_ERR_INVALID_ARG, "null x / y");
  if (ldx < k || ldy < k) return fail(B2D_ERR_INVALID_ARG, "leading dimension smaller than k");
  return B2D_OK;
}

// prep and the parameters of an EPI_RADIUS launch, with the self pairs of b2d_pairwise_distance
int radius_prep(cudaStream_t s, const RadiusLayout& L, const TcMetric& tm, const float* x, int64_t ldx, const float* y,
                int64_t ldy, int64_t m, int64_t n, int64_t k, float radius, TcParams* p)
{
  const int rc = launch_prep<float>(s, L.w, x, ldx, 1, m, y, ldy, 1, n, k, nullptr, nullptr, tm);
  if (rc) return rc;
  *p = TcParams{};
  p->m = m; p->n = n; p->eps = radius;
  p->diag_off = tc_self_diag(tm, x, ldx, 1, m, y, ldy, 1, n);
  return B2D_OK;
}

}  // namespace

namespace b2d {

int radius_sort_split(cudaStream_t s, const int64_t* indptr, int64_t m, int64_t nnz, int64_t* indices, float* distances,
                      long long* alt, void* sort_tmp, size_t sort_bytes)
{
  // every row's keys in ascending order (they are distinct: one per column), segments clipped to the nnz slots
  cub::DoubleBuffer<long long> keys(reinterpret_cast<long long*>(indices), alt);
  using RowIt = thrust::counting_iterator<int64_t>;
  const thrust::transform_iterator<RadiusRowStart, RowIt, long long> begin(RowIt(0), RadiusRowStart{indptr, nnz});
  const thrust::transform_iterator<RadiusRowStart, RowIt, long long> end(RowIt(0), RadiusRowStart{indptr + 1, nnz});
  size_t need = 0;
  B2D_CUDA(cub::DeviceSegmentedRadixSort::SortKeys(nullptr, need, keys, static_cast<int>(nnz), static_cast<int>(m), begin, end,
                                                   0, 64, s));
  if (need > sort_bytes) return fail(B2D_ERR_WORKSPACE, "internal: segmented sort scratch " + std::to_string(need) + " bytes");
  B2D_CUDA(cub::DeviceSegmentedRadixSort::SortKeys(sort_tmp, need, keys, static_cast<int>(nnz), static_cast<int>(m), begin,
                                                   end, 0, 64, s));
  int sms = 0;
  const int rc = device_sms(&sms);
  if (rc) return rc;
  const int64_t blocks = std::min<int64_t>((nnz + 255) / 256, static_cast<int64_t>(sms) * 8);
  radius_split_kernel<<<static_cast<unsigned>(blocks), 256, 0, s>>>(keys.Current(), indices, distances, nnz);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

}  // namespace b2d

size_t b2d_radius_neighbors_workspace_bytes(int64_t m, int64_t n, int64_t k, int64_t nnz)
{
  if (m < 0 || n < 0 || k < 0 || nnz < 0) return static_cast<size_t>(-1);
  return radius_layout(nullptr, m, n, k, nnz).bytes;
}

int b2d_radius_neighbors_count(void* stream, int64_t* indptr, int metric, const float* x, int64_t ldx, const float* y,
                               int64_t ldy, int64_t m, int64_t n, int64_t k, float radius, void* workspace,
                               size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  TcMetric tm;
  bool work = false;
  int rc = radius_check(metric, indptr, x, ldx, y, ldy, m, n, k, &tm, &work);
  if (rc) return rc;
  if (work) {
    rc = check_workspace(workspace, workspace_bytes, radius_layout(nullptr, m, n, k, 0).bytes);
    if (rc) return rc;
  }
  if (!work || !(radius >= 0.f)) {   // no pairs (a NaN or negative radius matches nothing)
    B2D_CUDA(cudaMemsetAsync(indptr, 0, static_cast<size_t>(m + 1) * sizeof(int64_t), s));
    return B2D_OK;
  }
  const RadiusLayout L = radius_layout(workspace, m, n, k, 0);
  TcParams p;
  rc = radius_prep(s, L, tm, x, ldx, y, ldy, m, n, k, radius, &p);
  if (rc) return rc;
  B2D_CUDA(cudaMemsetAsync(L.deg, 0, static_cast<size_t>(m + 1) * sizeof(unsigned), s));
  p.knn_cnt  = L.deg;
  p.rad_fill = 0;
  {
    ProfileScope prof(s);
    rc = launch_tc(s, L.w, p, k, EPI_RADIUS, tm.post);
    if (rc) return rc;
  }
  const thrust::transform_iterator<RadiusDeg64, const unsigned*, long long> deg(L.deg, RadiusDeg64{});
  size_t need = 0;
  B2D_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, need, deg, indptr, m + 1, s));
  if (need > L.scan_bytes) return fail(B2D_ERR_WORKSPACE, "internal: scan scratch " + std::to_string(need) + " bytes");
  B2D_CUDA(cub::DeviceScan::ExclusiveSum(L.scan_tmp, need, deg, indptr, m + 1, s));
  return B2D_OK;
}

int b2d_radius_neighbors_fill(void* stream, const int64_t* indptr, int64_t nnz, int64_t* indices, float* distances,
                              int metric, const float* x, int64_t ldx, const float* y, int64_t ldy, int64_t m, int64_t n,
                              int64_t k, float radius, void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  TcMetric tm;
  bool work = false;
  int rc = radius_check(metric, indptr, x, ldx, y, ldy, m, n, k, &tm, &work);
  if (rc) return rc;
  if (nnz < 0) return fail(B2D_ERR_INVALID_ARG, "negative nnz");
  if (nnz > 0x7fffffffll)
    return fail(B2D_ERR_UNSUPPORTED, "nnz = " + std::to_string(nnz) +
                                         " exceeds 2^31 - 1 pairs per call: split the queries into smaller batches");
  if (nnz > 0 && (!indices || !distances)) return fail(B2D_ERR_INVALID_ARG, "null indices / distances");
  if (work) {
    rc = check_workspace(workspace, workspace_bytes, radius_layout(nullptr, m, n, k, nnz).bytes);
    if (rc) return rc;
  }
  if (!work || nnz == 0 || !(radius >= 0.f)) return B2D_OK;
  const RadiusLayout L = radius_layout(workspace, m, n, k, nnz);
  TcParams p;
  rc = radius_prep(s, L, tm, x, ldx, y, ldy, m, n, k, radius, &p);
  if (rc) return rc;
  B2D_CUDA(cudaMemsetAsync(L.fill, 0, static_cast<size_t>(m) * sizeof(unsigned), s));
  p.knn_cnt    = L.fill;
  p.knn_cand   = reinterpret_cast<long long*>(indices);
  p.rad_indptr = reinterpret_cast<const long long*>(indptr);
  p.rad_nnz    = nnz;
  p.rad_fill   = 1;
  {
    ProfileScope prof(s);
    rc = launch_tc(s, L.w, p, k, EPI_RADIUS, tm.post);
    if (rc) return rc;
  }
  return radius_sort_split(s, indptr, m, nnz, indices, distances, L.alt, L.sort_tmp, L.sort_bytes);
}
