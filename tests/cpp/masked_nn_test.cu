// Test of the masked_l2_nn header shim (include/raft/distance/masked_nn.cuh).  Compiled by tests/test_masked_nn.py;
// runs on the GPU box (tests/test_masked_nn_gpu.py), compiles and links everywhere.  The reference is a host brute force.
#include <cfloat>
#include <cmath>
#include <cstdio>
#include <vector>
#include <cuda_runtime.h>
#include <raft/distance/masked_nn.cuh>

int main()
{
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { std::printf("SKIP no gpu\n"); return 0; }
  const int m = 300, n = 500, k = 24, G = 7;
  const int hg[G] = {40, 40, 170, 171, 300, 420, 470};   // an empty group; rows 470.. are in no group
  std::vector<float> hx(m * k), hy(n * k), hxn(m), hyn(n);
  for (int i = 0; i < m * k; ++i) hx[i] = std::sin(0.37f * i) * 3.f;
  for (int i = 0; i < n * k; ++i) hy[i] = std::cos(0.11f * i) * 3.f;
  for (int i = 0; i < m; ++i) { float s = 0; for (int t = 0; t < k; ++t) s += hx[i * k + t] * hx[i * k + t]; hxn[i] = s; }
  for (int j = 0; j < n; ++j) { float s = 0; for (int t = 0; t < k; ++t) s += hy[j * k + t] * hy[j * k + t]; hyn[j] = s; }
  bool hadj[m * G];
  for (int i = 0; i < m; ++i)
    for (int g = 0; g < G; ++g) hadj[i * G + g] = i >= 250 ? false : ((i * 7 + g * 3) % 5) < 2;   // rows 250..: none
  // host brute force (fp64): best index and value per row, -1 without a candidate
  std::vector<int> ri(m, -1);
  std::vector<double> rv(m, 0.0);
  for (int i = 0; i < m; ++i) {
    int lo = 0;
    for (int g = 0; g < G; ++g) {
      for (int j = lo; j < hg[g]; ++j) {
        if (!hadj[i * G + g]) continue;
        double d = 0;
        for (int t = 0; t < k; ++t) { const double e = double(hx[i * k + t]) - hy[j * k + t]; d += e * e; }
        if (ri[i] < 0 || d < rv[i]) { ri[i] = j; rv[i] = d; }
      }
      lo = hg[g];
    }
  }
  float *x, *y, *xn, *yn, *fout;
  bool* adj;
  int* gidx;
  raft::KeyValuePair<int, float>* kout;
  cudaMalloc(&x, hx.size() * 4); cudaMalloc(&y, hy.size() * 4); cudaMalloc(&xn, m * 4); cudaMalloc(&yn, n * 4);
  cudaMalloc(&adj, sizeof(hadj)); cudaMalloc(&gidx, sizeof(hg)); cudaMalloc(&kout, m * sizeof(*kout)); cudaMalloc(&fout, m * 4);
  cudaMemcpy(x, hx.data(), hx.size() * 4, cudaMemcpyHostToDevice);
  cudaMemcpy(y, hy.data(), hy.size() * 4, cudaMemcpyHostToDevice);
  cudaMemcpy(xn, hxn.data(), m * 4, cudaMemcpyHostToDevice);
  cudaMemcpy(yn, hyn.data(), n * 4, cudaMemcpyHostToDevice);
  cudaMemcpy(adj, hadj, sizeof(hadj), cudaMemcpyHostToDevice);
  cudaMemcpy(gidx, hg, sizeof(hg), cudaMemcpyHostToDevice);
  cudaStream_t s;
  cudaStreamCreate(&s);
  raft::resources handle(s);
  auto xv  = raft::make_device_matrix_view<const float, int>(x, m, k);
  auto yv  = raft::make_device_matrix_view<const float, int>(y, n, k);
  auto xnv = raft::make_device_vector_view<const float, int>(xn, m);
  auto ynv = raft::make_device_vector_view<const float, int>(yn, n);
  auto av  = raft::make_device_matrix_view<const bool, int>(adj, m, G);
  auto gv  = raft::make_device_vector_view<const int, int>(gidx, G);
  using KVP = raft::KeyValuePair<int, float>;
  using Red = raft::distance::MinAndDistanceReduceOp<int, float>;
  using Pair = raft::distance::KVPMinReduce<int, float>;
  int bad = 0;
  auto close = [](double got, double ref) { return std::fabs(got - ref) <= 1e-4 * std::fmax(ref, 1.0) + 1e-3; };
  // 1. KVP output, initOutBuffer = true
  raft::distance::masked_l2_nn<float, KVP, int, Red, Pair>(handle, {Red{}, Pair{}, false, true}, xv, yv, xnv, ynv, av, gv,
                                                            raft::make_device_vector_view<KVP, int>(kout, m));
  std::vector<KVP> hk(m);
  cudaMemcpyAsync(hk.data(), kout, m * sizeof(KVP), cudaMemcpyDeviceToHost, s);
  cudaStreamSynchronize(s);
  for (int i = 0; i < m; ++i) {
    if (ri[i] < 0) { if (hk[i].value != FLT_MAX) ++bad; continue; }
    if (hk[i].key != ri[i] && !close(hk[i].value, rv[i])) ++bad;
    if (!close(hk[i].value, rv[i])) ++bad;
  }
  if (bad) std::printf("kvp: %d\n", bad);
  // 2. float output (MinReduceOp), sqrt
  using RedF = raft::distance::MinReduceOp<int, float>;
  raft::distance::masked_l2_nn<float, float, int, RedF, Pair>(handle, {RedF{}, Pair{}, true, true}, xv, yv, xnv, ynv, av, gv,
                                                               raft::make_device_vector_view<float, int>(fout, m));
  std::vector<float> hf(m);
  cudaMemcpyAsync(hf.data(), fout, m * 4, cudaMemcpyDeviceToHost, s);
  cudaStreamSynchronize(s);
  for (int i = 0; i < m; ++i) {
    if (ri[i] < 0) { if (hf[i] != FLT_MAX) ++bad; continue; }
    if (!close(hf[i], std::sqrt(rv[i]))) ++bad;
  }
  if (bad) std::printf("float: %d\n", bad);
  // 3. initOutBuffer = false: the caller's {-5, 1e30} survives where there is no candidate, loses elsewhere
  for (auto& e : hk) { e.key = -5; e.value = 1e30f; }
  cudaMemcpyAsync(kout, hk.data(), m * sizeof(KVP), cudaMemcpyHostToDevice, s);
  raft::distance::masked_l2_nn<float, KVP, int, Red, Pair>(handle, {Red{}, Pair{}, false, false}, xv, yv, xnv, ynv, av, gv,
                                                            raft::make_device_vector_view<KVP, int>(kout, m));
  cudaMemcpyAsync(hk.data(), kout, m * sizeof(KVP), cudaMemcpyDeviceToHost, s);
  cudaStreamSynchronize(s);
  for (int i = 0; i < m; ++i) {
    if (ri[i] < 0) { if (hk[i].key != -5 || hk[i].value != 1e30f) ++bad; continue; }
    if (!close(hk[i].value, rv[i])) ++bad;
  }
  if (cudaGetLastError() != cudaSuccess) ++bad;
  std::printf(bad ? "FAIL %d\n" : "PASS\n", bad);
  return bad ? 1 : 0;
}
