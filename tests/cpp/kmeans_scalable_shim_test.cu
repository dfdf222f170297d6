// C++ test of the raft::cluster::kmeans shim's k-means|| route.  Compiled by tests/test_kmeans_scalable_shim.py with and
// without the mock raft headers; on the GPU it reads argv[1] (int64 m, k, n_clusters; x [m, k]), runs fit with
// KMeansPlusPlus and oversampling_factor = 2 (k-means||), then with a default-constructed KMeansParams (greedy k-means++),
// and writes both results (centroids, inertia as float, n_iter as int32) to argv[2] for the Python test to compare with
// raft_b200.cluster.fit.
#include <cstdint>
#include <cstdio>
#include <vector>
#include <cuda_runtime.h>
#ifdef RAFT_B200_USE_REAL_RAFT
#include <raft/core/device_mdspan.hpp>
#endif
#include <raft/cluster/kmeans.cuh>

namespace km = raft::cluster::kmeans;

int main(int argc, char** argv)
{
  if (argc < 3) { std::printf("usage: kmeans_scalable_shim_test in.bin out.bin\n"); return 2; }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { std::printf("SKIP no gpu\n"); return 0; }
  FILE* f = std::fopen(argv[1], "rb");
  int64_t dims[3];
  if (!f || std::fread(dims, 8, 3, f) != 3) { std::printf("FAIL input\n"); return 1; }
  const int m = int(dims[0]), k = int(dims[1]), nc = int(dims[2]);
  std::vector<float> hx(size_t(m) * k);
  if (std::fread(hx.data(), 4, hx.size(), f) != hx.size()) { std::printf("FAIL input\n"); return 1; }
  std::fclose(f);
  float *x, *c;
  cudaMalloc(&x, hx.size() * 4); cudaMalloc(&c, size_t(nc) * k * 4);
  cudaMemcpy(x, hx.data(), hx.size() * 4, cudaMemcpyHostToDevice);
  cudaStream_t s;
  cudaStreamCreate(&s);
  std::vector<float> out[2] = {std::vector<float>(size_t(nc) * k), std::vector<float>(size_t(nc) * k)};
  float inertia[2] = {0.f, 0.f};
  int n_iter[2] = {0, 0};
  {
#ifdef RAFT_B200_USE_REAL_RAFT
    raft::resources handle;
    handle.mock_set_stream(s);
#else
    raft::resources handle(s);
#endif
    auto X = raft::make_device_matrix_view<const float, int>(x, m, k);
    auto C = raft::make_device_matrix_view<float, int>(c, nc, k);
    for (int v = 0; v < 2; ++v) {
      km::KMeansParams p;   // v = 1: the defaults (greedy k-means++)
      p.n_clusters = nc;
      p.rng_state.seed = 7;
      if (v == 0) p.oversampling_factor = 2.0;
      km::fit(handle, p, X, static_cast<const float*>(nullptr), C, &inertia[v], &n_iter[v]);
      cudaMemcpyAsync(out[v].data(), c, out[v].size() * 4, cudaMemcpyDeviceToHost, s);
      raft::resource::sync_stream(handle);
    }
  }
  FILE* o = std::fopen(argv[2], "wb");
  for (int v = 0; v < 2; ++v) {
    std::fwrite(out[v].data(), 4, out[v].size(), o);
    std::fwrite(&inertia[v], 4, 1, o);
    std::fwrite(&n_iter[v], 4, 1, o);
  }
  std::fclose(o);
  cudaStreamDestroy(s);
  cudaFree(x); cudaFree(c);
  std::printf("PASS\n");
  return 0;
}
