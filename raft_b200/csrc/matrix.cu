// Row-wise matrix operations: select_k (select_k.cuh), row_argmin and row_norm.
#include <cuda_runtime.h>
#include <algorithm>
#include <string>
#include <cub/device/device_segmented_radix_sort.cuh>

#include "host.cuh"
#include "select_k.cuh"

namespace b2d {

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
