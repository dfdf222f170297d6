// Host-only test of HDBSCAN's tree stages (raft_b200/csrc/hdbscan_tree.cuh), compiled on its own by
// tests/test_hdbscan_rbc.py.  argv[1] holds cases, each int64 m, min_cluster_size, leaf, allow_single_cluster, then fp64
// cluster_selection_epsilon, then the m - 1 edges as int32 src [m - 1], int32 dst [m - 1], fp32 w [m - 1]; for every
// case argv[2] receives int32 n_clusters, int32 labels [m] and fp32 probabilities [m].
#include <cstdint>
#include <cstdio>
#include <vector>

#include "../../raft_b200/csrc/hdbscan_tree.cuh"

int main(int argc, char** argv)
{
  if (argc < 3) { std::printf("usage: hdbscan_tree_test in.bin out.bin\n"); return 2; }
  FILE* f = std::fopen(argv[1], "rb");
  FILE* o = std::fopen(argv[2], "wb");
  if (!f || !o) { std::printf("FAIL open\n"); return 1; }
  int64_t h[4];
  int cases = 0;
  while (std::fread(h, 8, 4, f) == 4) {
    double eps;
    const int64_t m = h[0], e = m - 1;
    std::vector<int> src(e), dst(e), lab(m);
    std::vector<float> w(e), prob(m);
    if (std::fread(&eps, 8, 1, f) != 1 || std::fread(src.data(), 4, e, f) != size_t(e) ||
        std::fread(dst.data(), 4, e, f) != size_t(e) || std::fread(w.data(), 4, e, f) != size_t(e)) {
      std::printf("FAIL input\n");
      return 1;
    }
    const b2d::HdbTreeParams p{int(h[1]), eps, h[2] != 0, h[3] != 0};
    const int nc = b2d::hdbscan_tree(m, src.data(), dst.data(), w.data(), p, lab.data(), prob.data());
    std::fwrite(&nc, 4, 1, o);
    std::fwrite(lab.data(), 4, m, o);
    std::fwrite(prob.data(), 4, m, o);
    ++cases;
  }
  std::fclose(f);
  std::fclose(o);
  std::printf("PASS %d cases\n", cases);
  return 0;
}
