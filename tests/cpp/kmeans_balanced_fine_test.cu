// C++ test of the assignment step of balanced k-means' stage 1 (b2d_debug_kmeans_balanced_fine_assign: the adjacency
// bits written from the groups' row ranges, the tile classes, one EPI_MINLOC_MASKED launch) against a host brute force
// per group in fp64.  Every row of a group with centroids must get a centroid of its group whose distance is the group's
// minimum within the rounding of the fp32-grade expanded form; rows in no group, or in a group without centroids, get
// -1.  Two shapes: n_clusters over several 256-column blocks with uneven, empty and centroid-less groups, and
// ceil(m / 32) * num_groups above 2^24 adjacency words (2200003 rows, 256 groups, 65536 centroids).  Compiled by
// tests/test_kmeans_balanced_fine.py; prints PASS, or FAIL with the first bad row.
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <random>
#include <vector>
#include <cuda_runtime.h>

#include "raft_b200.h"

static int run(const char* name, int64_t m, int64_t k, int nc, const std::vector<int>& E, const std::vector<int>& F,
               uint32_t seed)
{
  const int64_t G = static_cast<int64_t>(E.size());
  std::mt19937 rng(seed);
  std::normal_distribution<float> nd(0.f, 1.f);
  std::vector<float> x(static_cast<size_t>(m) * k), c(static_cast<size_t>(nc) * k);
  std::vector<float> centre(static_cast<size_t>(G) * k);
  for (auto& v : centre) v = 10.f * nd(rng);
  auto group_of = [&](const std::vector<int>& ends, int64_t i) {
    int64_t g = 0;
    while (g < G && ends[g] <= i) ++g;
    return g;   // G: in no group
  };
  for (int64_t i = 0, g = 0; i < m; ++i) {
    while (g < G && E[g] <= i) ++g;
    for (int64_t t = 0; t < k; ++t) x[i * k + t] = (g < G ? centre[g * k + t] : 0.f) + nd(rng);
  }
  for (int64_t j = 0, g = 0; j < nc; ++j) {
    while (g < G && F[g] <= j) ++g;
    for (int64_t t = 0; t < k; ++t) c[j * k + t] = (g < G ? centre[g * k + t] : 0.f) + 0.7f * nd(rng);
  }
  float *dx, *dc;
  int *dE, *dF, *dl;
  void* ws;
  const size_t bytes = b2d_kmeans_balanced_workspace_bytes(m, k, nc);
  if (cudaMalloc(&dx, x.size() * 4) || cudaMalloc(&dc, c.size() * 4) || cudaMalloc(&dE, G * 4) || cudaMalloc(&dF, G * 4) ||
      cudaMalloc(&dl, m * 4) || cudaMalloc(&ws, bytes)) {
    std::printf("FAIL %s: allocation\n", name);
    return 1;
  }
  cudaMemcpy(dx, x.data(), x.size() * 4, cudaMemcpyHostToDevice);
  cudaMemcpy(dc, c.data(), c.size() * 4, cudaMemcpyHostToDevice);
  cudaMemcpy(dE, E.data(), G * 4, cudaMemcpyHostToDevice);
  cudaMemcpy(dF, F.data(), G * 4, cudaMemcpyHostToDevice);
  cudaMemset(ws, 0xA5, bytes);   // stale workspace: every table the step reads must be written by it
  int rc = b2d_debug_kmeans_balanced_fine_assign(nullptr, dx, k, m, k, dE, dc, nc, dF, G, dl, ws, bytes);
  if (rc != B2D_OK) { std::printf("FAIL %s: rc %d %s\n", name, rc, b2d_last_error()); return 1; }
  std::vector<int> lab(m);
  if (cudaMemcpy(lab.data(), dl, m * 4, cudaMemcpyDeviceToHost) != cudaSuccess) {
    std::printf("FAIL %s: %s\n", name, cudaGetErrorString(cudaGetLastError()));
    return 1;
  }
  cudaFree(dx); cudaFree(dc); cudaFree(dE); cudaFree(dF); cudaFree(dl); cudaFree(ws);
  int64_t exact = 0, checked = 0;
  for (int64_t i = 0; i < m; ++i) {
    const int64_t g = group_of(E, i);
    const int64_t c0 = g < G ? (g > 0 ? F[g - 1] : 0) : 0, c1 = g < G ? F[g] : 0;
    if (c1 <= c0) {
      if (lab[i] != -1) { std::printf("FAIL %s: row %lld in no group / a group without centroids got %d\n", name, (long long)i, lab[i]); return 1; }
      continue;
    }
    double best = INFINITY, xn = 0.0;
    int64_t bj = -1;
    for (int64_t t = 0; t < k; ++t) xn += double(x[i * k + t]) * x[i * k + t];
    auto d2 = [&](int64_t j) {
      double s = 0.0;
      for (int64_t t = 0; t < k; ++t) { const double e = double(x[i * k + t]) - c[j * k + t]; s += e * e; }
      return s;
    };
    for (int64_t j = c0; j < c1; ++j) {
      const double d = d2(j);
      if (d < best) { best = d; bj = j; }
    }
    const int l = lab[i];
    if (l < c0 || l >= c1) {
      std::printf("FAIL %s: row %lld of group %lld got %d, outside [%lld, %lld)\n", name, (long long)i, (long long)g, l,
                  (long long)c0, (long long)c1);
      return 1;
    }
    double cn = 0.0;
    for (int64_t t = 0; t < k; ++t) cn += double(c[l * k + t]) * c[l * k + t];
    if (d2(l) > best + 1e-5 * (xn + cn)) {
      std::printf("FAIL %s: row %lld got %d at %.9g, the group's minimum is %lld at %.9g\n", name, (long long)i, l, d2(l),
                  (long long)bj, best);
      return 1;
    }
    exact += l == bj;
    ++checked;
  }
  std::printf("%s: %lld rows checked, %lld on the exact fp64 arg-min\n", name, (long long)checked, (long long)exact);
  return 0;
}

int main()
{
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { std::printf("SKIP no gpu\n"); return 0; }
  // 1000 centroids (4 column blocks) in 8 groups of uneven size; group 2 has no centroids, group 5 no rows, and the
  // last 37 rows are in no group
  const std::vector<int> E1 = {3000, 7100, 7600, 12000, 12900, 12900, 17000, 19974};
  const std::vector<int> F1 = {100, 400, 400, 650, 651, 700, 990, 1000};
  if (run("several column blocks", 20011, 32, 1000, E1, F1, 1)) return 1;
  // 2200003 rows in 256 groups, 256 centroids each: 68751 * 256 adjacency words > 2^24
  const int64_t m = 2200003;
  std::vector<int> E2(256), F2(256);
  for (int g = 0; g < 256; ++g) {
    E2[g] = static_cast<int>(m * (g + 1) / 256);
    F2[g] = 256 * (g + 1);
  }
  if (run("more than 2^24 adjacency words", m, 4, 65536, E2, F2, 2)) return 1;
  std::printf("PASS\n");
  return 0;
}
