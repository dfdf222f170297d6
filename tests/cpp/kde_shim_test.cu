// C++ test of the raft::neighbors::kernel_density shim.  Compiled by tests/test_kde.py with and without the mock raft
// headers; on the GPU (tests/test_kde_shim.py) it reads the problem from argv[1] (int64 m, n, d, kernel, weighted; double
// bandwidth; queries; dataset; weights when weighted), runs score_samples twice (the second result must be the same
// bytes), checks that an output of the wrong length throws, and writes the log densities to argv[2] for the Python test to
// compare with kernel_density.
#include <cstdint>
#include <cstdio>
#include <cstring>
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
#include <raft/neighbors/kernel_density.cuh>

namespace kd = raft::neighbors::kernel_density;

int main(int argc, char** argv)
{
  if (argc < 3) { std::printf("usage: kde_shim_test in.bin out.bin\n"); return 2; }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { std::printf("SKIP no gpu\n"); return 0; }
  FILE* f = std::fopen(argv[1], "rb");
  int64_t hdr[5];
  double h;
  if (!f || std::fread(hdr, 8, 5, f) != 5 || std::fread(&h, 8, 1, f) != 1) { std::printf("FAIL input\n"); return 1; }
  const int64_t m = hdr[0], n = hdr[1], d = hdr[2];
  const bool weighted = hdr[4] != 0;
  std::vector<float> hq(m * d), hx(n * d), hw(weighted ? n : 0);
  if (std::fread(hq.data(), 4, hq.size(), f) != hq.size() || std::fread(hx.data(), 4, hx.size(), f) != hx.size() ||
      std::fread(hw.data(), 4, hw.size(), f) != hw.size()) {
    std::printf("FAIL input\n");
    return 1;
  }
  std::fclose(f);
  float *q, *x, *w = nullptr;
  double* out;
  cudaMalloc(&q, hq.size() * 4); cudaMalloc(&x, hx.size() * 4); cudaMalloc(&out, m * 8);
  cudaMemcpy(q, hq.data(), hq.size() * 4, cudaMemcpyHostToDevice);
  cudaMemcpy(x, hx.data(), hx.size() * 4, cudaMemcpyHostToDevice);
  if (weighted) {
    cudaMalloc(&w, n * 4);
    cudaMemcpy(w, hw.data(), n * 4, cudaMemcpyHostToDevice);
  }
  cudaStream_t s;
  cudaStreamCreate(&s);
  int bad = 0;
  std::vector<double> ho[2];
  {
#ifdef RAFT_B200_USE_REAL_RAFT
    raft::resources handle;
    handle.mock_set_stream(s);
#else
    raft::resources handle(s);
#endif
    auto qv = raft::make_device_matrix_view<const float, int64_t>(q, m, d);
    auto xv = raft::make_device_matrix_view<const float, int64_t>(x, n, d);
    std::optional<raft::device_vector_view<const float, int64_t>> wv;
    if (weighted) wv = raft::device_vector_view<const float, int64_t>(w, n);
    kd::KdeParams params;
    params.kernel    = static_cast<kd::KernelType>(hdr[3]);
    params.bandwidth = h;
    for (int rep = 0; rep < 2; ++rep) {
      params.batch_cols = rep ? 256 : 0;   // the slab width changes no bit
      kd::score_samples<int64_t>(handle, xv, qv, wv, raft::device_vector_view<double, int64_t>(out, m), params);
      raft::resource::sync_stream(handle);
      ho[rep].resize(m);
      cudaMemcpy(ho[rep].data(), out, m * 8, cudaMemcpyDeviceToHost);
    }
    bool threw = false;
    try {   // one output short
      kd::score_samples<int64_t>(handle, xv, qv, wv, raft::device_vector_view<double, int64_t>(out, m - 1), params);
    } catch (const raft::logic_error&) {
      threw = true;
    }
    if (!threw) ++bad;
  }
  for (int64_t i = 0; i < m; ++i)
    if (std::memcmp(&ho[0][i], &ho[1][i], 8) != 0) ++bad;
  FILE* o = std::fopen(argv[2], "wb");
  std::fwrite(ho[0].data(), 8, m, o);
  std::fclose(o);
  cudaStreamDestroy(s);
  cudaFree(q); cudaFree(x); cudaFree(out); cudaFree(w);
  std::printf(bad ? "FAIL %d\n" : "PASS\n", bad);
  return bad ? 1 : 0;
}
