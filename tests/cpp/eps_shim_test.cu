// C++ test of the raft::neighbors::epsilon_neighborhood shim, both forms, int and int64 degrees.  Compiled by
// tests/test_eps_neighborhood.py with and without the mock raft headers; on the GPU it reads x, y and eps from argv[1]
// (int64 m, n, k; float eps; x; y), checks that the four calls agree and that a second call adds to vd, and writes the
// adjacency bytes and the int64 degrees to argv[2] for the Python test to compare with eps_neighbors_l2sq.
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
#include <raft/neighbors/epsilon_neighborhood.cuh>

namespace en = raft::neighbors::epsilon_neighborhood;

template <typename idx_t>
static std::vector<int64_t> fetch(const idx_t* d, int64_t n)
{
  std::vector<idx_t> h(n);
  cudaMemcpy(h.data(), d, n * sizeof(idx_t), cudaMemcpyDeviceToHost);
  return std::vector<int64_t>(h.begin(), h.end());
}

int main(int argc, char** argv)
{
  if (argc < 3) { std::printf("usage: eps_shim_test in.bin out.bin\n"); return 2; }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { std::printf("SKIP no gpu\n"); return 0; }
  FILE* f = std::fopen(argv[1], "rb");
  int64_t dims[3];
  float eps;
  if (!f || std::fread(dims, 8, 3, f) != 3 || std::fread(&eps, 4, 1, f) != 1) { std::printf("FAIL input\n"); return 1; }
  const int64_t m = dims[0], n = dims[1], k = dims[2];
  std::vector<float> hx(m * k), hy(n * k);
  if (std::fread(hx.data(), 4, hx.size(), f) != hx.size() || std::fread(hy.data(), 4, hy.size(), f) != hy.size()) {
    std::printf("FAIL input\n");
    return 1;
  }
  std::fclose(f);
  float *x, *y;
  bool *adj[4];
  int* v32[2];
  int64_t* v64[2];
  cudaMalloc(&x, hx.size() * 4); cudaMalloc(&y, hy.size() * 4);
  cudaMemcpy(x, hx.data(), hx.size() * 4, cudaMemcpyHostToDevice);
  cudaMemcpy(y, hy.data(), hy.size() * 4, cudaMemcpyHostToDevice);
  for (auto& a : adj) cudaMalloc(&a, m * n);
  for (int i = 0; i < 2; ++i) {
    cudaMalloc(&v32[i], (n + 1) * 4); cudaMemset(v32[i], 0, (n + 1) * 4);
    cudaMalloc(&v64[i], (n + 1) * 8); cudaMemset(v64[i], 0, (n + 1) * 8);
  }
  cudaStream_t s;
  cudaStreamCreate(&s);
  int bad = 0;
  {
#ifdef RAFT_B200_USE_REAL_RAFT
    raft::resources handle;
    handle.mock_set_stream(s);
#else
    raft::resources handle(s);
#endif
    // pointer form, int and int64 (the int form twice: it adds)
    en::epsUnexpL2SqNeighborhood<float, int>(adj[0], v32[0], x, y, int(m), int(n), int(k), eps, s);
    en::epsUnexpL2SqNeighborhood<float, int>(adj[0], v32[0], x, y, int(m), int(n), int(k), eps, s);
    en::epsUnexpL2SqNeighborhood<float, int64_t>(adj[1], v64[0], x, y, m, n, k, eps, s);
    // mdspan form, int and int64
    auto xv = raft::make_device_matrix_view<const float, int64_t>(x, m, k);
    auto yv = raft::make_device_matrix_view<const float, int64_t>(y, n, k);
    en::eps_neighbors_l2sq<float, int, int64_t>(handle, xv, yv, raft::make_device_matrix_view<bool, int64_t>(adj[2], m, n),
                                                raft::device_vector_view<int, int64_t>(v32[1], n + 1), eps);
    en::eps_neighbors_l2sq<float, int64_t, int64_t>(handle, xv, yv,
                                                    raft::make_device_matrix_view<bool, int64_t>(adj[3], m, n),
                                                    raft::device_vector_view<int64_t, int64_t>(v64[1], n + 1), eps);
    bool threw = false;
    try {
      en::eps_neighbors_l2sq<float, int64_t, int64_t>(handle, xv, yv,
                                                      raft::make_device_matrix_view<bool, int64_t>(adj[3], m, n),
                                                      raft::device_vector_view<int64_t, int64_t>(v64[1], n), eps);
    } catch (const raft::logic_error&) {
      threw = true;
    }
    if (!threw) ++bad;
    raft::resource::sync_stream(handle);
  }
  std::vector<uint8_t> ha[4];
  for (int i = 0; i < 4; ++i) {
    ha[i].resize(m * n);
    cudaMemcpy(ha[i].data(), adj[i], m * n, cudaMemcpyDeviceToHost);
    if (i && ha[i] != ha[0]) ++bad;
  }
  const std::vector<int64_t> a = fetch(v32[0], n + 1), b = fetch(v64[0], n + 1), c = fetch(v32[1], n + 1),
                             d = fetch(v64[1], n + 1);
  for (int64_t j = 0; j <= n; ++j)
    if (a[j] != 2 * b[j] || c[j] != b[j] || d[j] != b[j]) ++bad;
  FILE* o = std::fopen(argv[2], "wb");
  std::fwrite(ha[0].data(), 1, ha[0].size(), o);
  std::fwrite(b.data(), 8, b.size(), o);
  std::fclose(o);
  cudaStreamDestroy(s);
  cudaFree(x); cudaFree(y);
  for (auto a2 : adj) cudaFree(a2);
  for (int i = 0; i < 2; ++i) { cudaFree(v32[i]); cudaFree(v64[i]); }
  std::printf(bad ? "FAIL %d\n" : "PASS\n", bad);
  return bad ? 1 : 0;
}
