// C++ test of the raft::cluster::kmeans shim.  Compiled by tests/test_kmeans_shim.py with and without the mock raft
// headers; on the GPU it reads argv[1] (int64 m, k, n_clusters; x [m, k]; initial centroids [n_clusters, k]), runs fit
// with InitMethod::Array, predict and cluster_cost, checks that a wrong centroid shape and a non-L2 metric throw, and
// writes the centroids, labels, inertia (float) and n_iter (int32) to argv[2] for the Python test to compare with
// raft_b200.cluster.
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
  if (argc < 3) { std::printf("usage: kmeans_shim_test in.bin out.bin\n"); return 2; }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { std::printf("SKIP no gpu\n"); return 0; }
  FILE* f = std::fopen(argv[1], "rb");
  int64_t dims[3];
  if (!f || std::fread(dims, 8, 3, f) != 3) { std::printf("FAIL input\n"); return 1; }
  const int m = int(dims[0]), k = int(dims[1]), nc = int(dims[2]);
  std::vector<float> hx(size_t(m) * k), hc(size_t(nc) * k);
  if (std::fread(hx.data(), 4, hx.size(), f) != hx.size() || std::fread(hc.data(), 4, hc.size(), f) != hc.size()) {
    std::printf("FAIL input\n");
    return 1;
  }
  std::fclose(f);
  float *x, *c;
  int32_t* lab;
  cudaMalloc(&x, hx.size() * 4); cudaMalloc(&c, hc.size() * 4); cudaMalloc(&lab, size_t(m) * 4);
  cudaMemcpy(x, hx.data(), hx.size() * 4, cudaMemcpyHostToDevice);
  cudaMemcpy(c, hc.data(), hc.size() * 4, cudaMemcpyHostToDevice);
  cudaStream_t s;
  cudaStreamCreate(&s);
  int bad = 0;
  float inertia = 0.f, pred_inertia = 0.f, cost = 0.f;
  int n_iter = 0;
  std::vector<int32_t> hl(m);
  {
#ifdef RAFT_B200_USE_REAL_RAFT
    raft::resources handle;
    handle.mock_set_stream(s);
#else
    raft::resources handle(s);
#endif
    km::KMeansParams p;
    p.n_clusters = nc;
    p.init = km::InitMethod::Array;
    p.max_iter = 25;
    p.tol = 1e-4;
    auto X = raft::make_device_matrix_view<const float, int>(x, m, k);
    km::fit(handle, p, X, static_cast<const float*>(nullptr), raft::make_device_matrix_view<float, int>(c, nc, k), &inertia,
            &n_iter);
    auto C = raft::make_device_matrix_view<const float, int>(c, nc, k);
    km::predict(handle, p, X, static_cast<const float*>(nullptr), C, lab, true, &pred_inertia);
    km::cluster_cost(handle, X, C, &cost);
    if (pred_inertia != inertia || cost != inertia) ++bad;
    bool threw = false;
    try {
      km::fit(handle, p, X, static_cast<const float*>(nullptr), raft::make_device_matrix_view<float, int>(c, nc - 1, k),
              &inertia, &n_iter);
    } catch (const raft::logic_error&) {
      threw = true;
    }
    if (!threw) ++bad;
    threw = false;
    try {
      km::KMeansParams q = p;
      q.metric = raft::distance::DistanceType::CosineExpanded;
      km::predict(handle, q, X, static_cast<const float*>(nullptr), C, lab, true, &pred_inertia);
    } catch (const raft::logic_error&) {
      threw = true;
    }
    if (!threw) ++bad;
    cudaMemcpyAsync(hc.data(), c, hc.size() * 4, cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(hl.data(), lab, hl.size() * 4, cudaMemcpyDeviceToHost, s);
    raft::resource::sync_stream(handle);
  }
  FILE* o = std::fopen(argv[2], "wb");
  std::fwrite(hc.data(), 4, hc.size(), o);
  std::fwrite(hl.data(), 4, hl.size(), o);
  std::fwrite(&inertia, 4, 1, o);
  std::fwrite(&n_iter, 4, 1, o);
  std::fclose(o);
  cudaStreamDestroy(s);
  cudaFree(x); cudaFree(c); cudaFree(lab);
  std::printf(bad ? "FAIL %d\n" : "PASS\n", bad);
  return bad ? 1 : 0;
}
