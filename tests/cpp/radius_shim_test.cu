// C++ test of the raft::neighbors radius_neighbors shim.  Compiled by tests/test_radius_neighbors.py with and without the
// mock raft headers; on the GPU (tests/test_radius_neighbors_shim.py) it reads the metric, the radius, queries and dataset
// from argv[1] (int64 m, n, d, metric; float radius; queries; dataset), runs count and fill twice (the second result must
// be the same bytes), checks that a fill with too short outputs throws, and writes indptr, indices and distances to
// argv[2] for the Python test to compare with radius_neighbors.
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
#include <raft/neighbors/radius_neighbors.cuh>

namespace rn = raft::neighbors;

int main(int argc, char** argv)
{
  if (argc < 3) { std::printf("usage: radius_shim_test in.bin out.bin\n"); return 2; }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { std::printf("SKIP no gpu\n"); return 0; }
  FILE* f = std::fopen(argv[1], "rb");
  int64_t dims[4];
  float radius;
  if (!f || std::fread(dims, 8, 4, f) != 4 || std::fread(&radius, 4, 1, f) != 1) { std::printf("FAIL input\n"); return 1; }
  const int64_t m = dims[0], n = dims[1], d = dims[2];
  const auto metric = static_cast<raft::distance::DistanceType>(dims[3]);
  std::vector<float> hq(m * d), hx(n * d);
  if (std::fread(hq.data(), 4, hq.size(), f) != hq.size() || std::fread(hx.data(), 4, hx.size(), f) != hx.size()) {
    std::printf("FAIL input\n");
    return 1;
  }
  std::fclose(f);
  float *q, *x;
  int64_t* indptr;
  cudaMalloc(&q, hq.size() * 4); cudaMalloc(&x, hx.size() * 4); cudaMalloc(&indptr, (m + 1) * 8);
  cudaMemcpy(q, hq.data(), hq.size() * 4, cudaMemcpyHostToDevice);
  cudaMemcpy(x, hx.data(), hx.size() * 4, cudaMemcpyHostToDevice);
  cudaStream_t s;
  cudaStreamCreate(&s);
  int bad = 0;
  std::vector<int64_t> hp[2], hi[2];
  std::vector<float> hd[2];
  {
#ifdef RAFT_B200_USE_REAL_RAFT
    raft::resources handle;
    handle.mock_set_stream(s);
#else
    raft::resources handle(s);
#endif
    auto qv = raft::make_device_matrix_view<const float, int64_t>(q, m, d);
    auto xv = raft::make_device_matrix_view<const float, int64_t>(x, n, d);
    for (int rep = 0; rep < 2; ++rep) {
      rn::radius_neighbors_count<int64_t>(handle, qv, xv, raft::device_vector_view<int64_t, int64_t>(indptr, m + 1), radius,
                                          metric);
      int64_t nnz = 0;
      cudaMemcpyAsync(&nnz, indptr + m, 8, cudaMemcpyDeviceToHost, s);
      raft::resource::sync_stream(handle);
      int64_t* idx;
      float* dist;
      cudaMalloc(&idx, (nnz + 1) * 8); cudaMalloc(&dist, (nnz + 1) * 4);
      rn::radius_neighbors_fill<int64_t>(handle, qv, xv, raft::device_vector_view<const int64_t, int64_t>(indptr, m + 1),
                                         raft::device_vector_view<int64_t, int64_t>(idx, nnz),
                                         raft::device_vector_view<float, int64_t>(dist, nnz), radius, metric);
      bool threw = false;
      try {   // distances shorter than indices
        rn::radius_neighbors_fill<int64_t>(handle, qv, xv, raft::device_vector_view<const int64_t, int64_t>(indptr, m + 1),
                                           raft::device_vector_view<int64_t, int64_t>(idx, nnz + 1),
                                           raft::device_vector_view<float, int64_t>(dist, nnz), radius, metric);
      } catch (const raft::logic_error&) {
        threw = true;
      }
      if (!threw) ++bad;
      raft::resource::sync_stream(handle);
      hp[rep].resize(m + 1); hi[rep].resize(nnz); hd[rep].resize(nnz);
      cudaMemcpy(hp[rep].data(), indptr, (m + 1) * 8, cudaMemcpyDeviceToHost);
      cudaMemcpy(hi[rep].data(), idx, nnz * 8, cudaMemcpyDeviceToHost);
      cudaMemcpy(hd[rep].data(), dist, nnz * 4, cudaMemcpyDeviceToHost);
      cudaFree(idx); cudaFree(dist);
    }
  }
  if (hp[0] != hp[1] || hi[0] != hi[1] || hd[0] != hd[1]) ++bad;
  FILE* o = std::fopen(argv[2], "wb");
  std::fwrite(hp[0].data(), 8, hp[0].size(), o);
  std::fwrite(hi[0].data(), 8, hi[0].size(), o);
  std::fwrite(hd[0].data(), 4, hd[0].size(), o);
  std::fclose(o);
  cudaStreamDestroy(s);
  cudaFree(q); cudaFree(x); cudaFree(indptr);
  std::printf(bad ? "FAIL %d\n" : "PASS\n", bad);
  return bad ? 1 : 0;
}
