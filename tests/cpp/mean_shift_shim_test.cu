// C++ test of the raft::cluster::mean_shift shim.  Compiled by tests/test_mean_shift.py with and without the mock raft
// headers; on the GPU (tests/test_mean_shift_shim.py) it reads the problem from argv[1] (int64 m, d, s, bin_seeding;
// double bandwidth; x; seeds when s > 0), fits twice (the second time with 128-seed batches: the result must be the
// same bytes), checks that labels of the wrong length throw, and writes (n_centers, n_iter, centers, labels) to argv[2]
// for the Python test to compare with mean_shift.
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
#include <raft/cluster/mean_shift.cuh>

namespace ms = raft::cluster::mean_shift;

int main(int argc, char** argv)
{
  if (argc < 3) { std::printf("usage: mean_shift_shim_test in.bin out.bin\n"); return 2; }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { std::printf("SKIP no gpu\n"); return 0; }
  FILE* f = std::fopen(argv[1], "rb");
  int64_t hdr[4];
  double h;
  if (!f || std::fread(hdr, 8, 4, f) != 4 || std::fread(&h, 8, 1, f) != 1) { std::printf("FAIL input\n"); return 1; }
  const int64_t m = hdr[0], d = hdr[1], s = hdr[2];
  std::vector<float> hx(m * d), hs(s * d);
  if (std::fread(hx.data(), 4, hx.size(), f) != hx.size() || std::fread(hs.data(), 4, hs.size(), f) != hs.size()) {
    std::printf("FAIL input\n");
    return 1;
  }
  std::fclose(f);
  const int64_t cap = s > 0 ? s : m;
  float *x, *sd = nullptr, *c;
  int* lab;
  cudaMalloc(&x, hx.size() * 4); cudaMalloc(&c, cap * d * 4); cudaMalloc(&lab, m * 4);
  cudaMemcpy(x, hx.data(), hx.size() * 4, cudaMemcpyHostToDevice);
  if (s > 0) {
    cudaMalloc(&sd, hs.size() * 4);
    cudaMemcpy(sd, hs.data(), hs.size() * 4, cudaMemcpyHostToDevice);
  }
  cudaStream_t st;
  cudaStreamCreate(&st);
  int bad = 0;
  std::vector<float> hc[2];
  std::vector<int> hl[2];
  int nc[2] = {0, 0}, it[2] = {0, 0};
  {
#ifdef RAFT_B200_USE_REAL_RAFT
    raft::resources handle;
    handle.mock_set_stream(st);
#else
    raft::resources handle(st);
#endif
    auto xv = raft::make_device_matrix_view<const float, int64_t>(x, m, d);
    std::optional<raft::device_matrix_view<const float, int64_t, raft::row_major>> sv;
    if (s > 0) sv = raft::make_device_matrix_view<const float, int64_t>(sd, s, d);
    auto cv = raft::make_device_matrix_view<float, int64_t>(c, cap, d);
    ms::MeanShiftParams params;
    params.bandwidth   = h;
    params.bin_seeding = hdr[3] != 0;
    for (int rep = 0; rep < 2; ++rep) {
      params.max_bytes_per_batch = rep ? 1 : 0;   // 128 seeds per batch changes no bit
      ms::fit(handle, params, xv, sv, cv, raft::device_vector_view<int, int64_t>(lab, m), nc[rep], it[rep]);
      hc[rep].resize(nc[rep] * d);
      hl[rep].resize(m);
      cudaMemcpy(hc[rep].data(), c, hc[rep].size() * 4, cudaMemcpyDeviceToHost);
      cudaMemcpy(hl[rep].data(), lab, m * 4, cudaMemcpyDeviceToHost);
    }
    bool threw = false;
    try {   // one label short
      ms::fit(handle, params, xv, sv, cv, raft::device_vector_view<int, int64_t>(lab, m - 1), nc[1], it[1]);
    } catch (const raft::logic_error&) {
      threw = true;
    }
    if (!threw) ++bad;
  }
  if (nc[0] != nc[1] || it[0] != it[1] || hc[0].size() != hc[1].size() ||
      std::memcmp(hc[0].data(), hc[1].data(), hc[0].size() * 4) != 0 || hl[0] != hl[1])
    ++bad;
  FILE* o = std::fopen(argv[2], "wb");
  const int32_t head[2] = {nc[0], it[0]};
  std::fwrite(head, 4, 2, o);
  std::fwrite(hc[0].data(), 4, hc[0].size(), o);
  std::fwrite(hl[0].data(), 4, m, o);
  std::fclose(o);
  cudaStreamDestroy(st);
  cudaFree(x); cudaFree(c); cudaFree(lab); cudaFree(sd);
  std::printf(bad ? "FAIL %d\n" : "PASS\n", bad);
  return bad ? 1 : 0;
}
