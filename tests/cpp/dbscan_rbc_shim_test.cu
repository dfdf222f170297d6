// C++ test of the EpsNnMethod::RBC forms of the raft::cluster::dbscan shim.  Compiled by tests/test_dbscan_rbc.py with and
// without the mock raft headers; on the GPU (tests/test_dbscan_rbc_gpu.py) it reads argv[1] (int64 m, d, min_samples,
// n_landmarks; float eps; x [m, d]), runs the mdspan form (with core sample indices, L2SqrtUnexpanded by default) and the
// pointer form (with and without them, n_landmarks and seed given), which must agree, checks that a wrong labels extent
// and a batch size with RBC throw and that the BRUTE_FORCE method reaches the brute fit, and writes the labels and
// core_sample_indices (int32 [m] each) to argv[2] for the Python test to compare with
// raft_b200.cluster.dbscan(algorithm="rbc").
#include <cstdint>
#include <cstdio>
#include <optional>
#include <vector>
#include <cuda_runtime.h>
#ifdef RAFT_B200_USE_REAL_RAFT
#include <raft/core/device_mdspan.hpp>
#endif
#include <raft/cluster/dbscan.cuh>

namespace db = raft::cluster::dbscan;

template <typename T>
struct vec_view {   // a 1-d view: what the mdspan form reads of raft::device_vector_view
  T* p;
  int n;
  T* data_handle() const { return p; }
  int extent(int) const { return n; }
};

int main(int argc, char** argv)
{
  if (argc < 3) { std::printf("usage: dbscan_rbc_shim_test in.bin out.bin\n"); return 2; }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { std::printf("SKIP no gpu\n"); return 0; }
  FILE* f = std::fopen(argv[1], "rb");
  int64_t dims[4];
  float eps = 0.f;
  if (!f || std::fread(dims, 8, 4, f) != 4 || std::fread(&eps, 4, 1, f) != 1) { std::printf("FAIL input\n"); return 1; }
  const int m = int(dims[0]), d = int(dims[1]), ms = int(dims[2]);
  const int64_t nl = dims[3];
  std::vector<float> hx(size_t(m) * d);
  if (std::fread(hx.data(), 4, hx.size(), f) != hx.size()) { std::printf("FAIL input\n"); return 1; }
  std::fclose(f);
  float* x;
  int *lab, *core, *lab2, *core2, *lab3, *lab4;
  cudaMalloc(&x, hx.size() * 4);
  cudaMalloc(&lab, size_t(m) * 4); cudaMalloc(&core, size_t(m) * 4);
  cudaMalloc(&lab2, size_t(m) * 4); cudaMalloc(&core2, size_t(m) * 4); cudaMalloc(&lab3, size_t(m) * 4);
  cudaMalloc(&lab4, size_t(m) * 4);
  cudaMemcpy(x, hx.data(), hx.size() * 4, cudaMemcpyHostToDevice);
  cudaStream_t s;
  cudaStreamCreate(&s);
  int bad = 0;
  std::vector<int32_t> hlab(m), hcore(m), hlab2(m), hcore2(m), hlab3(m), hlab4(m);
  {
#ifdef RAFT_B200_USE_REAL_RAFT
    raft::resources handle;
    handle.mock_set_stream(s);
#else
    raft::resources handle(s);
#endif
    const auto rbc = db::EpsNnMethod::RBC;
    const auto sqrt_unexp = raft::distance::DistanceType::L2SqrtUnexpanded;
    auto X = raft::make_device_matrix_view<const float, int>(x, m, d);
    db::fit(handle, X, vec_view<int>{lab, m}, eps, ms, rbc, sqrt_unexp, std::make_optional(vec_view<int>{core, m}));
    db::fit(handle, x, m, d, eps, ms, sqrt_unexp, lab2, core2, 0, rbc, nl, 12345);
    db::fit(handle, x, m, d, eps, ms, sqrt_unexp, lab3, nullptr, 0, rbc);
    // the brute fit through the method parameter: the expanded metric
    db::fit(handle, x, m, d, eps, ms, raft::distance::DistanceType::L2SqrtExpanded, lab4, nullptr, 0,
            db::EpsNnMethod::BRUTE_FORCE);
    bool threw = false;
    try {
      db::fit(handle, X, vec_view<int>{lab, m - 1}, eps, ms, rbc);
    } catch (const raft::logic_error&) {
      threw = true;
    }
    if (!threw) ++bad;
    threw = false;
    try {
      db::fit(handle, x, m, d, eps, ms, sqrt_unexp, lab3, nullptr, 1 << 20, rbc);
    } catch (const raft::logic_error&) {
      threw = true;
    }
    if (!threw) ++bad;
    cudaMemcpyAsync(hlab.data(), lab, size_t(m) * 4, cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(hcore.data(), core, size_t(m) * 4, cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(hlab2.data(), lab2, size_t(m) * 4, cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(hcore2.data(), core2, size_t(m) * 4, cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(hlab3.data(), lab3, size_t(m) * 4, cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(hlab4.data(), lab4, size_t(m) * 4, cudaMemcpyDeviceToHost, s);
    raft::resource::sync_stream(handle);
  }
  if (hlab != hlab2 || hlab != hlab3 || hcore != hcore2) ++bad;
  FILE* o = std::fopen(argv[2], "wb");
  std::fwrite(hlab.data(), 4, hlab.size(), o);
  std::fwrite(hcore.data(), 4, hcore.size(), o);
  std::fwrite(hlab4.data(), 4, hlab4.size(), o);
  std::fclose(o);
  cudaStreamDestroy(s);
  cudaFree(x); cudaFree(lab); cudaFree(core); cudaFree(lab2); cudaFree(core2); cudaFree(lab3); cudaFree(lab4);
  std::printf(bad ? "FAIL %d\n" : "PASS\n", bad);
  return bad ? 1 : 0;
}
