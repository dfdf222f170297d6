// C++ test of the raft::distance::kernels shim: every kernel through KernelFactory, both forms (mdspan and the legacy
// pointer evaluate), row- and column-major.  Compiled by tests/test_gram.py with and without the mock raft headers; on
// the GPU it reads x and y from argv[1] (int64 m, n, k; x; y), checks that the forms and layouts agree bit for bit and
// that a bad shape throws, and writes the four row-major [m, n] matrices to argv[2] for the Python test to compare with
// gram_matrix.
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <memory>
#include <vector>
#include <cuda_runtime.h>
#ifdef RAFT_B200_USE_REAL_RAFT
#include <raft/core/device_mdspan.hpp>
#endif
#include <raft/distance/kernels.cuh>

namespace kn = raft::distance::kernels;

int main(int argc, char** argv)
{
  if (argc < 3) { std::printf("usage: gram_shim_test in.bin out.bin\n"); return 2; }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { std::printf("SKIP no gpu\n"); return 0; }
  FILE* f = std::fopen(argv[1], "rb");
  int64_t dims[3];
  if (!f || std::fread(dims, 8, 3, f) != 3) { std::printf("FAIL input\n"); return 1; }
  const int m = int(dims[0]), n = int(dims[1]), k = int(dims[2]);
  std::vector<float> hx(size_t(m) * k), hy(size_t(n) * k);
  if (std::fread(hx.data(), 4, hx.size(), f) != hx.size() || std::fread(hy.data(), 4, hy.size(), f) != hy.size()) {
    std::printf("FAIL input\n");
    return 1;
  }
  std::fclose(f);
  // column-major copies of x and y
  std::vector<float> cx(hx.size()), cy(hy.size());
  for (int i = 0; i < m; ++i)
    for (int t = 0; t < k; ++t) cx[size_t(t) * m + i] = hx[size_t(i) * k + t];
  for (int j = 0; j < n; ++j)
    for (int t = 0; t < k; ++t) cy[size_t(t) * n + j] = hy[size_t(j) * k + t];
  float *x, *y, *xc, *yc, *d1, *d2, *d3;
  cudaMalloc(&x, hx.size() * 4); cudaMalloc(&y, hy.size() * 4);
  cudaMalloc(&xc, cx.size() * 4); cudaMalloc(&yc, cy.size() * 4);
  cudaMalloc(&d1, size_t(m) * n * 4); cudaMalloc(&d2, size_t(m) * n * 4); cudaMalloc(&d3, size_t(m) * n * 4);
  cudaMemcpy(x, hx.data(), hx.size() * 4, cudaMemcpyHostToDevice);
  cudaMemcpy(y, hy.data(), hy.size() * 4, cudaMemcpyHostToDevice);
  cudaMemcpy(xc, cx.data(), cx.size() * 4, cudaMemcpyHostToDevice);
  cudaMemcpy(yc, cy.data(), cy.size() * 4, cudaMemcpyHostToDevice);
  cudaStream_t s;
  cudaStreamCreate(&s);
  int bad = 0;
  const kn::KernelParams params[4] = {{kn::LINEAR, 0, 1.0, 0.0}, {kn::POLYNOMIAL, 3, 0.05, 1.0}, {kn::RBF, 0, 0.02, 0.0},
                                      {kn::TANH, 0, 0.03, -0.5}};
  FILE* o = std::fopen(argv[2], "wb");
  {
#ifdef RAFT_B200_USE_REAL_RAFT
    raft::resources handle;
    handle.mock_set_stream(s);
#else
    raft::resources handle(s);
#endif
    std::vector<float> h1(size_t(m) * n), h2(h1.size()), h3(h1.size());
    for (const kn::KernelParams& kp : params) {
      std::unique_ptr<kn::GramMatrixBase<float>> kernel(kn::KernelFactory<float>::create(kp));
      // mdspan, row-major; legacy pointer form, row-major; mdspan, column-major
      (*kernel)(handle, raft::make_device_matrix_view<const float, int>(x, m, k),
                raft::make_device_matrix_view<const float, int>(y, n, k), raft::make_device_matrix_view<float, int>(d1, m, n));
      kernel->evaluate(x, m, k, y, n, d2, true, s, k, k, n);
      (*kernel)(handle, raft::make_device_matrix_view<const float, int, raft::col_major>(xc, m, k),
                raft::make_device_matrix_view<const float, int, raft::col_major>(yc, n, k),
                raft::make_device_matrix_view<float, int, raft::col_major>(d3, m, n));
      bool threw = false;
      try {
        (*kernel)(handle, raft::make_device_matrix_view<const float, int>(x, m, k),
                  raft::make_device_matrix_view<const float, int>(y, n, k),
                  raft::make_device_matrix_view<float, int>(d1, m, n - 1));
      } catch (const raft::logic_error&) {
        threw = true;
      }
      if (!threw) ++bad;
      cudaMemcpyAsync(h1.data(), d1, h1.size() * 4, cudaMemcpyDeviceToHost, s);
      cudaMemcpyAsync(h2.data(), d2, h2.size() * 4, cudaMemcpyDeviceToHost, s);
      cudaMemcpyAsync(h3.data(), d3, h3.size() * 4, cudaMemcpyDeviceToHost, s);
      raft::resource::sync_stream(handle);
      if (h1 != h2) ++bad;
      // column-major: the same kernel values up to the operand roles (K(x, y) = K(y, x) computed the other way round)
      for (int i = 0; i < m; ++i)
        for (int j = 0; j < n; ++j) {
          const float a = h1[size_t(i) * n + j], b = h3[size_t(j) * m + i];
          if (!(std::fabs(a - b) <= 1e-4f * std::fmax(1.f, std::fabs(a)))) ++bad;
        }
      std::fwrite(h1.data(), 4, h1.size(), o);
    }
  }
  std::fclose(o);
  cudaStreamDestroy(s);
  cudaFree(x); cudaFree(y); cudaFree(xc); cudaFree(yc); cudaFree(d1); cudaFree(d2); cudaFree(d3);
  std::printf(bad ? "FAIL %d\n" : "PASS\n", bad);
  return bad ? 1 : 0;
}
