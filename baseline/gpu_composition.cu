// GPU BASELINE -- measurement infrastructure, NOT part of the product (nothing under raft_b200/ links or loads it;
// only bench.py's `gpu_baselines` leg and tests/test_gpu_baseline.py do).
//
// What the reference's SURVIVING primitives compose to for this path (SURVEY.md 8(d) "GPU baselines", Appendix A
// "Baseline composition recipe"; the fused distance kernels themselves were removed upstream, SURVEY.md section 0):
//   raft::linalg::norm<L2Norm, ALONG_ROWS>     cpp/include/raft/linalg/norm.cuh:118-147          -> bl_row_norm_kernel
//   raft::linalg::gemm (NT) through cuBLASLt   cpp/include/raft/linalg/detail/cublaslt_wrappers.hpp:35-38 (fp32:
//       CUBLAS_COMPUTE_32F, no TF32), :268-313 (cublasLtMatmul with a heuristic-selected algorithm) -> bl_gemm_nt
//   raft::linalg::map_offset elementwise pass  cpp/include/raft/linalg/map.cuh:216-300           -> bl_l2_epilogue_kernel
//   raft::matrix::argmin (cub block ArgMin)    cpp/include/raft/matrix/detail/math.cuh:290-343   -> bl_row_argmin_kernel
// i.e. three passes over the m x n matrix (write, read+write, read) where the engine makes one (or none, for NN).
// Written from the primitives' documented behaviour; no reference source is copied.
#include <cublasLt.h>
#include <cuda_runtime.h>
#include <cfloat>
#include <cstdint>
#include <cstdio>

namespace {

cublasLtHandle_t g_lt = nullptr;
char g_err[256]       = "";

int fail(const char* what, int code)
{
  snprintf(g_err, sizeof(g_err), "%s failed (%d)", what, code);
  return 1;
}

__global__ void bl_row_norm_kernel(float* out, const float* x, int64_t rows, int k)
{
  const int lane  = threadIdx.x & 31;
  const int64_t r = static_cast<int64_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= rows) return;
  const float* row = x + r * k;
  float acc = 0.f;
  for (int t = lane; t < k; t += 32) { const float v = __ldg(row + t); acc = fmaf(v, v, acc); }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) out[r] = acc;
}

// one elementwise pass (read + write), index -> (i, j) like map_offset: d = max(xn_i + yn_j - 2 g, 0) [sqrt]
__global__ void bl_l2_epilogue_kernel(float* d, const float* xn, const float* yn, int64_t m, int64_t n, int do_sqrt)
{
  const int64_t n4    = n >> 2;
  const int64_t total = m * n4;
  for (int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < total;
       t += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t i = t / n4, j = (t - i * n4) << 2;
    float4 g        = *reinterpret_cast<const float4*>(d + i * n + j);
    const float a   = __ldg(xn + i);
    const float4 b  = *reinterpret_cast<const float4*>(yn + j);
    g.x = fmaxf(a + b.x - 2.f * g.x, 0.f); g.y = fmaxf(a + b.y - 2.f * g.y, 0.f);
    g.z = fmaxf(a + b.z - 2.f * g.z, 0.f); g.w = fmaxf(a + b.w - 2.f * g.w, 0.f);
    if (do_sqrt) { g.x = sqrtf(g.x); g.y = sqrtf(g.y); g.z = sqrtf(g.z); g.w = sqrtf(g.w); }
    *reinterpret_cast<float4*>(d + i * n + j) = g;
  }
}

// one block per row: (min value, smallest index holding it), merged into (best_val, best_idx) with index offset
__global__ void __launch_bounds__(256) bl_row_argmin_kernel(const float* d, int64_t n, float* best_val, int* best_idx,
                                                            int idx_offset, int first)
{
  const float* row = d + static_cast<int64_t>(blockIdx.x) * n;
  float v = FLT_MAX;
  int ix  = 0x7fffffff;
  for (int64_t j = threadIdx.x * 4; j < n; j += 256 * 4) {
    const float4 q = *reinterpret_cast<const float4*>(row + j);
    if (q.x < v) { v = q.x; ix = static_cast<int>(j); }
    if (q.y < v) { v = q.y; ix = static_cast<int>(j) + 1; }
    if (q.z < v) { v = q.z; ix = static_cast<int>(j) + 2; }
    if (q.w < v) { v = q.w; ix = static_cast<int>(j) + 3; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi   = __shfl_xor_sync(0xffffffffu, ix, o);
    if (ov < v || (ov == v && oi < ix)) { v = ov; ix = oi; }
  }
  __shared__ float sv[8];
  __shared__ int si[8];
  if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = v; si[threadIdx.x >> 5] = ix; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; ++w)
      if (sv[w] < v || (sv[w] == v && si[w] < ix)) { v = sv[w]; ix = si[w]; }
    ix += idx_offset;
    if (!first) {
      const float bv = best_val[blockIdx.x];
      const int bi   = best_idx[blockIdx.x];
      if (bv < v || (bv == v && bi < ix)) { v = bv; ix = bi; }
    }
    best_val[blockIdx.x] = v;
    best_idx[blockIdx.x] = ix;
  }
}

// g [m,n] row-major = x [m,k] . y [n,k]^T, fp32 in / fp32 compute (CUBLAS_COMPUTE_32F: no TF32) / fp32 out.
// Row-major matrices are the column-major transposes: g^T (n x m, ld n) = y_cm^T (n x k) . x_cm (k x m).
int bl_gemm_nt(cudaStream_t s, float* g, const float* x, const float* y, int64_t m, int64_t n, int64_t k, void* ws,
               size_t ws_bytes)
{
  cublasLtMatmulDesc_t op   = nullptr;
  cublasLtMatrixLayout_t la = nullptr, lb = nullptr, lc = nullptr;
  cublasLtMatmulPreference_t pref = nullptr;
  int rc = 0;
  cublasStatus_t st;
  const cublasOperation_t tn = CUBLAS_OP_T, nn = CUBLAS_OP_N;
  const float alpha = 1.f, beta = 0.f;
  cublasLtMatmulHeuristicResult_t heur;
  int found = 0;
  if ((st = cublasLtMatmulDescCreate(&op, CUBLAS_COMPUTE_32F, CUDA_R_32F)) != CUBLAS_STATUS_SUCCESS) { rc = fail("cublasLtMatmulDescCreate", st); goto done; }
  cublasLtMatmulDescSetAttribute(op, CUBLASLT_MATMUL_DESC_TRANSA, &tn, sizeof(tn));
  cublasLtMatmulDescSetAttribute(op, CUBLASLT_MATMUL_DESC_TRANSB, &nn, sizeof(nn));
  if ((st = cublasLtMatrixLayoutCreate(&la, CUDA_R_32F, k, n, k)) != CUBLAS_STATUS_SUCCESS) { rc = fail("layout A", st); goto done; }
  if ((st = cublasLtMatrixLayoutCreate(&lb, CUDA_R_32F, k, m, k)) != CUBLAS_STATUS_SUCCESS) { rc = fail("layout B", st); goto done; }
  if ((st = cublasLtMatrixLayoutCreate(&lc, CUDA_R_32F, n, m, n)) != CUBLAS_STATUS_SUCCESS) { rc = fail("layout C", st); goto done; }
  if ((st = cublasLtMatmulPreferenceCreate(&pref)) != CUBLAS_STATUS_SUCCESS) { rc = fail("preference", st); goto done; }
  cublasLtMatmulPreferenceSetAttribute(pref, CUBLASLT_MATMUL_PREF_MAX_WORKSPACE_BYTES, &ws_bytes, sizeof(ws_bytes));
  st = cublasLtMatmulAlgoGetHeuristic(g_lt, op, la, lb, lc, lc, pref, 1, &heur, &found);
  if (st != CUBLAS_STATUS_SUCCESS || found == 0) { rc = fail("cublasLtMatmulAlgoGetHeuristic", st); goto done; }
  st = cublasLtMatmul(g_lt, op, &alpha, y, la, x, lb, &beta, g, lc, g, lc, &heur.algo, ws, ws_bytes, s);
  if (st != CUBLAS_STATUS_SUCCESS) rc = fail("cublasLtMatmul", st);
done:
  if (pref) cublasLtMatmulPreferenceDestroy(pref);
  if (lc) cublasLtMatrixLayoutDestroy(lc);
  if (lb) cublasLtMatrixLayoutDestroy(lb);
  if (la) cublasLtMatrixLayoutDestroy(la);
  if (op) cublasLtMatmulDescDestroy(op);
  return rc;
}

}  // namespace

extern "C" {

const char* bl_last_error(void) { return g_err; }

int bl_init(void)
{
  if (g_lt) return 0;
  const cublasStatus_t st = cublasLtCreate(&g_lt);
  return st == CUBLAS_STATUS_SUCCESS ? 0 : fail("cublasLtCreate", st);
}

// dist [m,n] = L2Expanded (do_sqrt: L2SqrtExpanded) of x [m,k], y [n,k]; xn [m], yn [n] scratch; n % 4 == 0.
int bl_pairwise_l2(void* stream, float* dist, const float* x, const float* y, float* xn, float* yn, int64_t m, int64_t n,
                   int64_t k, int do_sqrt, void* ws, size_t ws_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (!g_lt && bl_init()) return 1;
  if (n % 4) return fail("n % 4", 0);
  bl_row_norm_kernel<<<static_cast<unsigned>((m + 7) / 8), 256, 0, s>>>(xn, x, m, static_cast<int>(k));
  bl_row_norm_kernel<<<static_cast<unsigned>((n + 7) / 8), 256, 0, s>>>(yn, y, n, static_cast<int>(k));
  if (bl_gemm_nt(s, dist, x, y, m, n, k, ws, ws_bytes)) return 1;
  bl_l2_epilogue_kernel<<<132 * 16, 256, 0, s>>>(dist, xn, yn, m, n, do_sqrt);
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : fail(cudaGetErrorString(e), e);
}

// fusedL2NN by composition: for every chunk of `chunk_rows` rows of y: the three passes above into `tile`
// [m x chunk_rows] + one row-argmin pass merged into (best_val, best_idx).
int bl_l2_nn(void* stream, float* best_val, int* best_idx, const float* x, const float* y, float* tile, float* xn,
             float* yn, int64_t m, int64_t n, int64_t k, int64_t chunk_rows, void* ws, size_t ws_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (!g_lt && bl_init()) return 1;
  if (chunk_rows % 4 || n % 4) return fail("chunk_rows % 4", 0);
  bl_row_norm_kernel<<<static_cast<unsigned>((m + 7) / 8), 256, 0, s>>>(xn, x, m, static_cast<int>(k));
  for (int64_t j0 = 0; j0 < n; j0 += chunk_rows) {
    const int64_t nc = n - j0 < chunk_rows ? n - j0 : chunk_rows;
    bl_row_norm_kernel<<<static_cast<unsigned>((nc + 7) / 8), 256, 0, s>>>(yn, y + j0 * k, nc, static_cast<int>(k));
    if (bl_gemm_nt(s, tile, x, y + j0 * k, m, nc, k, ws, ws_bytes)) return 1;
    bl_l2_epilogue_kernel<<<132 * 16, 256, 0, s>>>(tile, xn, yn, m, nc, 0);
    bl_row_argmin_kernel<<<static_cast<unsigned>(m), 256, 0, s>>>(tile, nc, best_val, best_idx, static_cast<int>(j0), j0 == 0);
  }
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : fail(cudaGetErrorString(e), e);
}

}  // extern "C"
