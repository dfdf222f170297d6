// Dependency-free C++ test of the raft::matrix::select_k shim.  Compiled by tests/test_select_k.py with and without the
// mock raft headers; runs on the GPU box, compiles (and links) everywhere.
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <numeric>
#include <vector>
#include <cuda_runtime.h>
#include <raft/matrix/select_k.cuh>

// the selection order restated on the host: -0.0 == +0.0, NaN above +inf, ties to the smaller column
static unsigned host_key(float v)
{
  unsigned b;
  std::memcpy(&b, &v, 4);
  if ((b & 0x7fffffffu) > 0x7f800000u) return 0xffffffffu;
  if (b == 0x80000000u) b = 0;
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

int main()
{
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { std::printf("SKIP no gpu\n"); return 0; }
  const int64_t rows = 5, len = 3000, k = 37;
  std::vector<float> hv(rows * len);
  std::vector<int64_t> hp(rows * len);
  for (int64_t i = 0; i < rows * len; ++i) {
    hv[i] = static_cast<float>((i * 7919) % 1013) * 0.25f - 100.f;   // repeated values: ties
    hp[i] = 1000000 + i;
  }
  float *v, *ov;
  int64_t *p, *oi;
  cudaMalloc(&v, hv.size() * 4); cudaMalloc(&p, hp.size() * 8);
  cudaMalloc(&ov, rows * k * 4); cudaMalloc(&oi, rows * k * 8);
  cudaMemcpy(v, hv.data(), hv.size() * 4, cudaMemcpyHostToDevice);
  cudaMemcpy(p, hp.data(), hp.size() * 8, cudaMemcpyHostToDevice);
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
    auto inv  = raft::make_device_matrix_view<const float, int64_t>(v, rows, len);
    auto inp  = raft::make_device_matrix_view<const int64_t, int64_t>(p, rows, len);
    auto outv = raft::make_device_matrix_view<float, int64_t>(ov, rows, k);
    auto outi = raft::make_device_matrix_view<int64_t, int64_t>(oi, rows, k);
    for (int sel_min = 0; sel_min < 2; ++sel_min) {
      for (int with_idx = 0; with_idx < 2; ++with_idx) {
        raft::matrix::select_k<float, int64_t>(
          handle, inv, with_idx ? std::make_optional(inp) : std::nullopt, outv, outi, sel_min == 1, true,
          raft::matrix::SelectAlgo::kRadix11bits);
        std::vector<float> gv(rows * k);
        std::vector<int64_t> gi(rows * k);
        cudaMemcpyAsync(gv.data(), ov, gv.size() * 4, cudaMemcpyDeviceToHost, s);
        cudaMemcpyAsync(gi.data(), oi, gi.size() * 8, cudaMemcpyDeviceToHost, s);
        raft::resource::sync_stream(handle);
        for (int64_t r = 0; r < rows; ++r) {
          std::vector<int64_t> col(len);
          std::iota(col.begin(), col.end(), 0);
          auto key = [&](int64_t c) { unsigned kk = host_key(hv[r * len + c]); return sel_min ? kk : ~kk; };
          std::stable_sort(col.begin(), col.end(), [&](int64_t a, int64_t b) { return key(a) < key(b); });
          for (int64_t j = 0; j < k; ++j) {
            const int64_t want = with_idx ? hp[r * len + col[j]] : col[j];
            if (gi[r * k + j] != want || gv[r * k + j] != hv[r * len + col[j]]) ++bad;
          }
        }
      }
    }
    bool threw = false;
    try {
      auto big = raft::make_device_matrix_view<float, int64_t>(ov, 1, len + 1);
      auto bigi = raft::make_device_matrix_view<int64_t, int64_t>(oi, 1, len + 1);
      auto one = raft::make_device_matrix_view<const float, int64_t>(v, 1, len);
      raft::matrix::select_k<float, int64_t>(handle, one, std::nullopt, big, bigi, true);
    } catch (const raft::logic_error&) {
      threw = true;
    }
    if (!threw) ++bad;
  }
  cudaStreamDestroy(s);
  cudaFree(v); cudaFree(p); cudaFree(ov); cudaFree(oi);
  std::printf(bad ? "FAIL %d\n" : "PASS\n", bad);
  return bad ? 1 : 0;
}
