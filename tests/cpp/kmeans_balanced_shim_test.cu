// C++ test of the raft::cluster::kmeans_balanced shim.  Compiled by tests/test_kmeans_balanced_shim.py with and without
// the mock raft headers; on the GPU it reads argv[1] (int64 m, k, n_clusters; x [m, k]), runs fit_predict with int32
// labels, predict with uint32 labels and fit, checks that a cosine metric throws raft::logic_error, and writes the
// centroids, the fit_predict labels and the predict labels to argv[2] for the Python test to compare.
#include <cstdint>
#include <cstdio>
#include <vector>
#include <cuda_runtime.h>
#ifdef RAFT_B200_USE_REAL_RAFT
#include <raft/core/device_mdspan.hpp>
#endif
#include <raft/cluster/kmeans_balanced.cuh>

namespace kb = raft::cluster::kmeans_balanced;

template <typename T>
auto vec(T* p, int n)
{
#ifdef RAFT_B200_USE_REAL_RAFT
  return cuda::std::mdspan<T, cuda::std::dextents<int, 1>>(p, n);
#else
  return raft::make_device_vector_view<T, int>(p, n);
#endif
}

int main(int argc, char** argv)
{
  if (argc < 3) { std::printf("usage: kmeans_balanced_shim_test in.bin out.bin\n"); return 2; }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { std::printf("SKIP no gpu\n"); return 0; }
  FILE* f = std::fopen(argv[1], "rb");
  int64_t dims[3];
  if (!f || std::fread(dims, 8, 3, f) != 3) { std::printf("FAIL input\n"); return 1; }
  const int m = int(dims[0]), k = int(dims[1]), nc = int(dims[2]);
  std::vector<float> hx(size_t(m) * k);
  if (std::fread(hx.data(), 4, hx.size(), f) != hx.size()) { std::printf("FAIL input\n"); return 1; }
  std::fclose(f);
  float *x, *c, *c2;
  int32_t* lab;
  uint32_t* ulab;
  cudaMalloc(&x, hx.size() * 4); cudaMalloc(&c, size_t(nc) * k * 4); cudaMalloc(&c2, size_t(nc) * k * 4);
  cudaMalloc(&lab, size_t(m) * 4); cudaMalloc(&ulab, size_t(m) * 4);
  cudaMemcpy(x, hx.data(), hx.size() * 4, cudaMemcpyHostToDevice);
  cudaStream_t s;
  cudaStreamCreate(&s);
  std::vector<float> hc(size_t(nc) * k), hc2(hc.size());
  std::vector<int32_t> hl(m);
  std::vector<uint32_t> hu(m);
  bool threw = false;
  {
#ifdef RAFT_B200_USE_REAL_RAFT
    raft::resources handle;
    handle.mock_set_stream(s);
#else
    raft::resources handle(s);
#endif
    auto X = raft::make_device_matrix_view<const float, int>(x, m, k);
    auto C = raft::make_device_matrix_view<float, int>(c, nc, k);
    raft::cluster::kmeans_balanced_params p;
    p.n_iters = 10;
    p.seed = 7;
    kb::fit_predict(handle, p, X, C, vec(lab, m));
    kb::predict(handle, p, X, raft::make_device_matrix_view<const float, int>(c, nc, k),
                vec(ulab, m));
    kb::fit(handle, p, X, raft::make_device_matrix_view<float, int>(c2, nc, k));
    raft::cluster::kmeans_balanced_params q;
    q.metric = raft::distance::DistanceType::CosineExpanded;
    try {
      kb::fit(handle, q, X, C);
    } catch (const raft::logic_error&) {
      threw = true;
    }
    cudaMemcpyAsync(hc.data(), c, hc.size() * 4, cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(hc2.data(), c2, hc2.size() * 4, cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(hl.data(), lab, hl.size() * 4, cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(hu.data(), ulab, hu.size() * 4, cudaMemcpyDeviceToHost, s);
    raft::resource::sync_stream(handle);
  }
  if (!threw) { std::printf("FAIL cosine did not throw\n"); return 1; }
  for (size_t i = 0; i < hc.size(); ++i)
    if (hc[i] != hc2[i]) { std::printf("FAIL fit != fit_predict\n"); return 1; }
  FILE* o = std::fopen(argv[2], "wb");
  std::fwrite(hc.data(), 4, hc.size(), o);
  std::fwrite(hl.data(), 4, hl.size(), o);
  std::fwrite(hu.data(), 4, hu.size(), o);
  std::fclose(o);
  cudaStreamDestroy(s);
  cudaFree(x); cudaFree(c); cudaFree(c2); cudaFree(lab); cudaFree(ulab);
  std::printf("PASS\n");
  return 0;
}
