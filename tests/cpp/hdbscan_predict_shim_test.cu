// C++ test of raft::cluster::hdbscan's prediction_model, its fit overload and approximate_predict
// (include/raft/cluster/hdbscan.cuh).  Compiled by tests/test_hdbscan_predict_shim.py with and without the mock raft
// headers; on the GPU it reads argv[1] (int64 m, d, min_cluster_size, min_samples, nq; x [m, d]; queries [nq, d]), fits
// with a model (the labels must equal those of the fit without one), checks that queries of another width and a model
// that was never fitted throw, predicts, and writes the predicted labels and probabilities (int32 [nq] / fp32 [nq]) to
// argv[2] for the Python test to compare with raft_b200.cluster.approximate_predict.
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
struct vec_view {
  T* p;
  int n;
  T* data_handle() const { return p; }
  int extent(int) const { return n; }
};

int main(int argc, char** argv)
{
  if (argc < 3) { std::printf("usage: hdbscan_predict_shim_test in.bin out.bin\n"); return 2; }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { std::printf("SKIP no gpu\n"); return 0; }
  FILE* f = std::fopen(argv[1], "rb");
  int64_t dims[5];
  if (!f || std::fread(dims, 8, 5, f) != 5) { std::printf("FAIL input\n"); return 1; }
  const int m = int(dims[0]), d = int(dims[1]), nq = int(dims[4]);
  std::vector<float> hx(size_t(m) * d), hq(size_t(nq) * d);
  if (std::fread(hx.data(), 4, hx.size(), f) != hx.size() || std::fread(hq.data(), 4, hq.size(), f) != hq.size()) {
    std::printf("FAIL input\n");
    return 1;
  }
  std::fclose(f);
  float *x, *q, *prob, *prob2, *qprob;
  int *lab, *lab2, *qlab;
  cudaMalloc(&x, hx.size() * 4);
  cudaMalloc(&q, hq.size() * 4);
  cudaMalloc(&lab, size_t(m) * 4); cudaMalloc(&lab2, size_t(m) * 4);
  cudaMalloc(&prob, size_t(m) * 4); cudaMalloc(&prob2, size_t(m) * 4);
  cudaMalloc(&qlab, size_t(nq) * 4); cudaMalloc(&qprob, size_t(nq) * 4);
  cudaMemcpy(x, hx.data(), hx.size() * 4, cudaMemcpyHostToDevice);
  cudaMemcpy(q, hq.data(), hq.size() * 4, cudaMemcpyHostToDevice);
  cudaStream_t s;
  cudaStreamCreate(&s);
  int bad = 0;
  std::vector<int32_t> hlab(m), hlab2(m), hqlab(nq);
  std::vector<float> hprob(m), hprob2(m), hqprob(nq);
  {
#ifdef RAFT_B200_USE_REAL_RAFT
    raft::resources handle;
    handle.mock_set_stream(s);
#else
    raft::resources handle(s);
#endif
    hd::params p;
    p.min_cluster_size = int(dims[2]);
    p.min_samples      = int(dims[3]);
    auto X = raft::make_device_matrix_view<const float, int>(x, m, d);
    auto Q = raft::make_device_matrix_view<const float, int>(q, nq, d);
    auto throws = [&](auto&& call) {
      try {
        call();
      } catch (const raft::logic_error&) {
        return true;
      }
      return false;
    };
    hd::prediction_model model;
    if (!throws([&] { hd::approximate_predict(handle, model, Q, vec_view<int>{qlab, nq}, vec_view<float>{qprob, nq}); }))
      ++bad;
    const int nc  = hd::fit(handle, X, vec_view<int>{lab, m}, vec_view<float>{prob, m}, p);
    const int nc2 = hd::fit(handle, X, vec_view<int>{lab2, m}, vec_view<float>{prob2, m}, model, p);
    if (nc != nc2 || !model.is_fitted() || model.n_rows() != m || model.n_cols() != d) ++bad;
    auto Qw = raft::make_device_matrix_view<const float, int>(q, nq / 4, 4);
    if (!throws([&] { hd::approximate_predict(handle, model, Qw, vec_view<int>{qlab, nq / 4}, vec_view<float>{qprob, nq / 4}); }))
      ++bad;
    hd::approximate_predict(handle, model, Q, vec_view<int>{qlab, nq}, vec_view<float>{qprob, nq});
    cudaMemcpyAsync(hlab.data(), lab, size_t(m) * 4, cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(hlab2.data(), lab2, size_t(m) * 4, cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(hprob.data(), prob, size_t(m) * 4, cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(hprob2.data(), prob2, size_t(m) * 4, cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(hqlab.data(), qlab, size_t(nq) * 4, cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(hqprob.data(), qprob, size_t(nq) * 4, cudaMemcpyDeviceToHost, s);
    raft::resource::sync_stream(handle);
  }
  if (hlab != hlab2 || hprob != hprob2) ++bad;
  FILE* o = std::fopen(argv[2], "wb");
  std::fwrite(hqlab.data(), 4, nq, o);
  std::fwrite(hqprob.data(), 4, nq, o);
  std::fclose(o);
  cudaStreamDestroy(s);
  cudaFree(x); cudaFree(q); cudaFree(lab); cudaFree(lab2); cudaFree(prob); cudaFree(prob2); cudaFree(qlab);
  cudaFree(qprob);
  std::printf(bad ? "FAIL %d\n" : "PASS\n", bad);
  return bad ? 1 : 0;
}
