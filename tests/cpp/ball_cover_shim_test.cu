// C++ test of the raft::neighbors::ball_cover shim.  Compiled by tests/test_ball_cover.py with and without the mock raft
// headers; on the GPU (tests/test_ball_cover_shim.py) it reads n, m, d, metric, k, eps, the dataset and the queries from
// argv[1] (int64 n, m, d, metric, k; float eps; dataset; queries), builds an index, runs knn_query, all_knn_query (its
// first rows must equal a knn_query of the dataset) and eps_nn_count / eps_nn, checks that mismatched outputs throw, and
// writes the kNN indices and distances and the CSR to argv[2] for the Python test to compare with the Python calls.
#include <cstdint>
#include <cstdio>
#include <vector>
#include <cuda_runtime.h>
#ifdef RAFT_B200_USE_REAL_RAFT
#include <raft/core/device_mdspan.hpp>
// (the mock headers have no 1-d view; real RAFT declares this one in raft/core/device_mdspan.hpp)
namespace raft {
template <typename T, typename IdxT = std::uint32_t, typename Layout = layout_c_contiguous>
using device_vector_view = cuda::std::mdspan<T, cuda::std::extents<IdxT, dynamic_extent>, Layout>;
}
#endif
#include <raft/neighbors/ball_cover.cuh>

namespace bc = raft::neighbors::ball_cover;

int main(int argc, char** argv)
{
  if (argc < 3) { std::printf("usage: ball_cover_shim_test in.bin out.bin\n"); return 2; }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { std::printf("SKIP no gpu\n"); return 0; }
  FILE* f = std::fopen(argv[1], "rb");
  int64_t dims[5];
  float eps;
  if (!f || std::fread(dims, 8, 5, f) != 5 || std::fread(&eps, 4, 1, f) != 1) { std::printf("FAIL input\n"); return 1; }
  const int64_t n = dims[0], m = dims[1], d = dims[2], k = dims[4];
  const auto metric = static_cast<raft::distance::DistanceType>(dims[3]);
  std::vector<float> hx(n * d), hq(m * d);
  if (std::fread(hx.data(), 4, hx.size(), f) != hx.size() || std::fread(hq.data(), 4, hq.size(), f) != hq.size()) {
    std::printf("FAIL input\n");
    return 1;
  }
  std::fclose(f);
  float *x, *q, *dist, *adist;
  int64_t *idx, *aidx, *indptr;
  cudaMalloc(&x, hx.size() * 4); cudaMalloc(&q, hq.size() * 4);
  cudaMalloc(&idx, m * k * 8); cudaMalloc(&dist, m * k * 4); cudaMalloc(&aidx, n * k * 8); cudaMalloc(&adist, n * k * 4);
  cudaMalloc(&indptr, (m + 1) * 8);
  cudaMemcpy(x, hx.data(), hx.size() * 4, cudaMemcpyHostToDevice);
  cudaMemcpy(q, hq.data(), hq.size() * 4, cudaMemcpyHostToDevice);
  cudaStream_t s;
  cudaStreamCreate(&s);
  int bad = 0;
  std::vector<int64_t> hi(m * k), hai(n * k), hp(m + 1), hj;
  std::vector<float> hd(m * k), had(n * k), hdd;
  {
#ifdef RAFT_B200_USE_REAL_RAFT
    raft::resources handle;
    handle.mock_set_stream(s);
#else
    raft::resources handle(s);
#endif
    auto xv = raft::make_device_matrix_view<const float, int64_t>(x, n, d);
    auto qv = raft::make_device_matrix_view<const float, int64_t>(q, m, d);
    bc::BallCoverIndex<int64_t, float> index(handle, xv, metric);
    bc::build_index(handle, index);
    bc::knn_query(handle, index, qv, raft::make_device_matrix_view<int64_t, int64_t>(idx, m, k),
                  raft::make_device_matrix_view<float, int64_t>(dist, m, k));
    bc::all_knn_query(handle, index, raft::make_device_matrix_view<int64_t, int64_t>(aidx, n, k),
                      raft::make_device_matrix_view<float, int64_t>(adist, n, k));
    bool threw = false;
    try {   // dists narrower than inds
      bc::knn_query(handle, index, qv, raft::make_device_matrix_view<int64_t, int64_t>(idx, m, k),
                    raft::make_device_matrix_view<float, int64_t>(dist, m, k - 1));
    } catch (const raft::logic_error&) {
      threw = true;
    }
    if (!threw) ++bad;
    bc::eps_nn_count(handle, index, qv, raft::device_vector_view<int64_t, int64_t>(indptr, m + 1), eps);
    raft::resource::sync_stream(handle);
    cudaMemcpy(hp.data(), indptr, (m + 1) * 8, cudaMemcpyDeviceToHost);
    const int64_t nnz = hp[m];
    int64_t* ja;
    float* dd;
    cudaMalloc(&ja, (nnz + 1) * 8); cudaMalloc(&dd, (nnz + 1) * 4);
    bc::eps_nn(handle, index, qv, raft::device_vector_view<const int64_t, int64_t>(indptr, m + 1),
               raft::device_vector_view<int64_t, int64_t>(ja, nnz), raft::device_vector_view<float, int64_t>(dd, nnz), eps);
    raft::resource::sync_stream(handle);
    hj.resize(nnz); hdd.resize(nnz);
    cudaMemcpy(hj.data(), ja, nnz * 8, cudaMemcpyDeviceToHost);
    cudaMemcpy(hdd.data(), dd, nnz * 4, cudaMemcpyDeviceToHost);
    cudaFree(ja); cudaFree(dd);
  }
  cudaMemcpy(hi.data(), idx, m * k * 8, cudaMemcpyDeviceToHost);
  cudaMemcpy(hd.data(), dist, m * k * 4, cudaMemcpyDeviceToHost);
  cudaMemcpy(hai.data(), aidx, n * k * 8, cudaMemcpyDeviceToHost);
  cudaMemcpy(had.data(), adist, n * k * 4, cudaMemcpyDeviceToHost);
  for (int64_t i = 0; i < n; ++i)   // every row finds itself at distance 0
    if (had[i * k] != 0.f) { ++bad; break; }
  FILE* o = std::fopen(argv[2], "wb");
  std::fwrite(hi.data(), 8, hi.size(), o);
  std::fwrite(hd.data(), 4, hd.size(), o);
  std::fwrite(hai.data(), 8, hai.size(), o);
  std::fwrite(hp.data(), 8, hp.size(), o);
  std::fwrite(hj.data(), 8, hj.size(), o);
  std::fwrite(hdd.data(), 4, hdd.size(), o);
  std::fclose(o);
  cudaStreamDestroy(s);
  cudaFree(x); cudaFree(q); cudaFree(idx); cudaFree(dist); cudaFree(aidx); cudaFree(adist); cudaFree(indptr);
  std::printf(bad ? "FAIL %d\n" : "PASS\n", bad);
  return bad ? 1 : 0;
}
