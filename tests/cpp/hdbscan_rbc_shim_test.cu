// C++ test of the raft::cluster::hdbscan shim (include/raft/cluster/hdbscan.cuh).  Compiled by
// tests/test_hdbscan_rbc_shim.py with and without the mock raft headers; on the GPU it reads argv[1] (int64 m, d,
// min_cluster_size, min_samples; x [m, d] with d = 2 or 3), runs the mdspan form (L2SqrtExpanded, taken as
// L2SqrtUnexpanded) and the pointer form (L2SqrtUnexpanded), which must agree, checks that a wrong labels extent and
// d = 4 throw, and writes n_clusters, the labels and the probabilities (int32 / int32 [m] / fp32 [m]) to argv[2] for the
// Python test to compare with raft_b200.cluster.hdbscan.
#include <cstdint>
#include <cstdio>
#include <vector>
#include <cuda_runtime.h>
#ifdef RAFT_B200_USE_REAL_RAFT
#include <raft/core/device_mdspan.hpp>
#endif
#include <raft/cluster/hdbscan.cuh>

namespace hd = raft::cluster::hdbscan;

template <typename T>
struct vec_view {   // a 1-d view: what the mdspan form reads of raft::device_vector_view
  T* p;
  int n;
  T* data_handle() const { return p; }
  int extent(int) const { return n; }
};

int main(int argc, char** argv)
{
  if (argc < 3) { std::printf("usage: hdbscan_rbc_shim_test in.bin out.bin\n"); return 2; }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { std::printf("SKIP no gpu\n"); return 0; }
  FILE* f = std::fopen(argv[1], "rb");
  int64_t dims[4];
  if (!f || std::fread(dims, 8, 4, f) != 4) { std::printf("FAIL input\n"); return 1; }
  const int m = int(dims[0]), d = int(dims[1]);
  std::vector<float> hx(size_t(m) * d);
  if (std::fread(hx.data(), 4, hx.size(), f) != hx.size()) { std::printf("FAIL input\n"); return 1; }
  std::fclose(f);
  float *x, *prob, *prob2;
  int *lab, *lab2;
  cudaMalloc(&x, hx.size() * 4);
  cudaMalloc(&lab, size_t(m) * 4); cudaMalloc(&lab2, size_t(m) * 4);
  cudaMalloc(&prob, size_t(m) * 4); cudaMalloc(&prob2, size_t(m) * 4);
  cudaMemcpy(x, hx.data(), hx.size() * 4, cudaMemcpyHostToDevice);
  cudaStream_t s;
  cudaStreamCreate(&s);
  int bad = 0, nc = 0, nc2 = 0;
  std::vector<int32_t> hlab(m), hlab2(m);
  std::vector<float> hprob(m), hprob2(m);
  {
#ifdef RAFT_B200_USE_REAL_RAFT
    raft::resources handle;
    handle.mock_set_stream(s);
#else
    raft::resources handle(s);
#endif
    using raft::distance::DistanceType;
    hd::params p;
    p.min_cluster_size = int(dims[2]);
    p.min_samples      = int(dims[3]);
    auto X = raft::make_device_matrix_view<const float, int>(x, m, d);
    nc = hd::fit(handle, X, vec_view<int>{lab, m}, vec_view<float>{prob, m}, p, DistanceType::L2SqrtExpanded);
    p.n_landmarks = 5;
    p.seed        = 9;
    nc2 = hd::fit(handle, x, m, d, DistanceType::L2SqrtUnexpanded, p, lab2, prob2);
    auto throws = [&](auto&& call) {
      try {
        call();
      } catch (const raft::logic_error&) {
        return true;
      }
      return false;
    };
    if (!throws([&] { hd::fit(handle, X, vec_view<int>{lab, m - 1}, vec_view<float>{prob, m}, p); })) ++bad;
    auto X4 = raft::make_device_matrix_view<const float, int>(x, m / 2, 4);
    if (!throws([&] { hd::fit(handle, X4, vec_view<int>{lab, m / 2}, vec_view<float>{prob, m / 2}, p); })) ++bad;
    cudaMemcpyAsync(hlab.data(), lab, size_t(m) * 4, cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(hlab2.data(), lab2, size_t(m) * 4, cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(hprob.data(), prob, size_t(m) * 4, cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(hprob2.data(), prob2, size_t(m) * 4, cudaMemcpyDeviceToHost, s);
    raft::resource::sync_stream(handle);
  }
  if (hlab != hlab2 || hprob != hprob2 || nc != nc2) ++bad;
  FILE* o = std::fopen(argv[2], "wb");
  std::fwrite(&nc, 4, 1, o);
  std::fwrite(hlab.data(), 4, m, o);
  std::fwrite(hprob.data(), 4, m, o);
  std::fclose(o);
  cudaStreamDestroy(s);
  cudaFree(x); cudaFree(lab); cudaFree(lab2); cudaFree(prob); cudaFree(prob2);
  std::printf(bad ? "FAIL %d\n" : "PASS\n", bad);
  return bad ? 1 : 0;
}
