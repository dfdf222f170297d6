// C++ test of the LinkageDistance::PAIRWISE forms of the raft::cluster::single_linkage shim.  Compiled by
// tests/test_single_linkage_rbc_shim.py with and without the mock raft headers; on the GPU it reads argv[1] (int64 m, d,
// n_clusters; x [m, d] with d = 2 or 3), runs the mdspan form (L2SqrtExpanded, taken as L2SqrtUnexpanded) and the
// pointer form (L2SqrtUnexpanded, with deltas and sizes), which must agree, checks that PAIRWISE at d = 4, a metric
// outside the L2 ones and a wrong dendrogram shape throw, and writes the children, labels, deltas, sizes and
// n_connected_components (int32 / fp32) to argv[2] for the Python test to compare with
// raft_b200.cluster.single_linkage(linkage="pairwise").
#include <cstdint>
#include <cstdio>
#include <vector>
#include <cuda_runtime.h>
#ifdef RAFT_B200_USE_REAL_RAFT
#include <raft/core/device_mdspan.hpp>
#endif
#include <raft/cluster/single_linkage.cuh>

namespace rc = raft::cluster;

template <typename T>
struct vec_view {   // a 1-d view: what the mdspan form reads of raft::device_vector_view
  T* p;
  int n;
  T* data_handle() const { return p; }
  int extent(int) const { return n; }
};

int main(int argc, char** argv)
{
  if (argc < 3) { std::printf("usage: single_linkage_rbc_shim_test in.bin out.bin\n"); return 2; }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { std::printf("SKIP no gpu\n"); return 0; }
  FILE* f = std::fopen(argv[1], "rb");
  int64_t dims[3];
  if (!f || std::fread(dims, 8, 3, f) != 3) { std::printf("FAIL input\n"); return 1; }
  const int m = int(dims[0]), d = int(dims[1]), nc = int(dims[2]);
  std::vector<float> hx(size_t(m) * d);
  if (std::fread(hx.data(), 4, hx.size(), f) != hx.size()) { std::printf("FAIL input\n"); return 1; }
  std::fclose(f);
  float *x, *deltas;
  int *ch, *lab, *ch2, *lab2, *sizes;
  cudaMalloc(&x, hx.size() * 4);
  cudaMalloc(&ch, size_t(m) * 8); cudaMalloc(&ch2, size_t(m) * 8);
  cudaMalloc(&lab, size_t(m) * 4); cudaMalloc(&lab2, size_t(m) * 4);
  cudaMalloc(&deltas, size_t(m) * 4); cudaMalloc(&sizes, size_t(m) * 4);
  cudaMemcpy(x, hx.data(), hx.size() * 4, cudaMemcpyHostToDevice);
  cudaStream_t s;
  cudaStreamCreate(&s);
  int bad = 0;
  std::vector<int32_t> hch(size_t(m - 1) * 2), hlab(m), hch2(hch.size()), hlab2(m), hsz(m - 1);
  std::vector<float> hde(m - 1);
  rc::linkage_output<int> out;
  {
#ifdef RAFT_B200_USE_REAL_RAFT
    raft::resources handle;
    handle.mock_set_stream(s);
#else
    raft::resources handle(s);
#endif
    using raft::distance::DistanceType;
    auto X = raft::make_device_matrix_view<const float, int>(x, m, d);
    rc::single_linkage<int, float, rc::LinkageDistance::PAIRWISE>(
      handle, X, raft::make_device_matrix_view<int, int>(ch, m - 1, 2), vec_view<int>{lab, m},
      DistanceType::L2SqrtExpanded, size_t(nc));
    out.children = ch2;
    out.labels   = lab2;
    rc::single_linkage<int, float, rc::LinkageDistance::PAIRWISE>(handle, x, size_t(m), size_t(d),
                                                                  DistanceType::L2SqrtUnexpanded, &out, 15, size_t(nc),
                                                                  deltas, sizes);
    if (out.m != m || out.n_clusters != nc || out.n_connected_components != 1) ++bad;
    auto throws = [&](auto&& call) {
      try {
        call();
      } catch (const raft::logic_error&) {
        return true;
      }
      return false;
    };
    auto X4 = raft::make_device_matrix_view<const float, int>(x, m / 2, 4);
    if (!throws([&] {
          rc::single_linkage<int, float, rc::LinkageDistance::PAIRWISE>(
            handle, X4, raft::make_device_matrix_view<int, int>(ch, m / 2 - 1, 2), vec_view<int>{lab, m / 2},
            DistanceType::L2SqrtExpanded, size_t(1));
        }))
      ++bad;
    if (!throws([&] {
          rc::single_linkage<int, float, rc::LinkageDistance::PAIRWISE>(
            handle, X, raft::make_device_matrix_view<int, int>(ch, m - 1, 2), vec_view<int>{lab, m},
            DistanceType::CosineExpanded, size_t(nc));
        }))
      ++bad;
    if (!throws([&] {
          rc::single_linkage<int, float, rc::LinkageDistance::PAIRWISE>(
            handle, X, raft::make_device_matrix_view<int, int>(ch, m - 2, 2), vec_view<int>{lab, m},
            DistanceType::L2SqrtExpanded, size_t(nc));
        }))
      ++bad;
    cudaMemcpyAsync(hch.data(), ch, hch.size() * 4, cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(hlab.data(), lab, hlab.size() * 4, cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(hch2.data(), ch2, hch2.size() * 4, cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(hlab2.data(), lab2, hlab2.size() * 4, cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(hde.data(), deltas, hde.size() * 4, cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(hsz.data(), sizes, hsz.size() * 4, cudaMemcpyDeviceToHost, s);
    raft::resource::sync_stream(handle);
  }
  if (hch != hch2 || hlab != hlab2) ++bad;
  FILE* o = std::fopen(argv[2], "wb");
  std::fwrite(hch.data(), 4, hch.size(), o);
  std::fwrite(hlab.data(), 4, hlab.size(), o);
  std::fwrite(hde.data(), 4, hde.size(), o);
  std::fwrite(hsz.data(), 4, hsz.size(), o);
  std::fwrite(&out.n_connected_components, 4, 1, o);
  std::fclose(o);
  cudaStreamDestroy(s);
  cudaFree(x); cudaFree(ch); cudaFree(ch2); cudaFree(lab); cudaFree(lab2); cudaFree(deltas); cudaFree(sizes);
  std::printf(bad ? "FAIL %d\n" : "PASS\n", bad);
  return bad ? 1 : 0;
}
