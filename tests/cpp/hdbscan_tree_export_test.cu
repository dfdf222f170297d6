// Host-only test of the tree export of HDBSCAN's tree stages (raft_b200/csrc/hdbscan_tree.cuh, HdbTreeExport),
// compiled on its own by tests/test_hdbscan_predict.py.  argv[1] holds cases in the format of hdbscan_tree_test.cu
// (int64 m, min_cluster_size, leaf, allow_single_cluster, fp64 cluster_selection_epsilon, int32 src [m - 1], int32 dst
// [m - 1], fp32 w [m - 1]).  For every case argv[2] receives int32 n_clusters, labels [m], fp32 probabilities [m] (with
// the export asked for), then int32 nc, single_root, fp64 thr, int32 row_parent [m], fp64 row_lambda [m], int32 parent,
// owner, label [nc], fp64 birth, death [nc].  FAIL when the labels or probabilities differ from those of the call
// without the export.
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include "../../raft_b200/csrc/hdbscan_tree.cuh"

int main(int argc, char** argv)
{
  if (argc < 3) { std::printf("usage: hdbscan_tree_export_test in.bin out.bin\n"); return 2; }
  FILE* f = std::fopen(argv[1], "rb");
  FILE* o = std::fopen(argv[2], "wb");
  if (!f || !o) { std::printf("FAIL open\n"); return 1; }
  int64_t h[4];
  int cases = 0;
  while (std::fread(h, 8, 4, f) == 4) {
    double eps;
    const int64_t m = h[0], e = m - 1;
    std::vector<int> src(e), dst(e), lab(m), lab0(m);
    std::vector<float> w(e), prob(m), prob0(m);
    if (std::fread(&eps, 8, 1, f) != 1 || std::fread(src.data(), 4, e, f) != size_t(e) ||
        std::fread(dst.data(), 4, e, f) != size_t(e) || std::fread(w.data(), 4, e, f) != size_t(e)) {
      std::printf("FAIL input\n");
      return 1;
    }
    const b2d::HdbTreeParams p{int(h[1]), eps, h[2] != 0, h[3] != 0};
    b2d::HdbTreeExport ex;
    const int nc0 = b2d::hdbscan_tree(m, src.data(), dst.data(), w.data(), p, lab0.data(), prob0.data());
    const int nc  = b2d::hdbscan_tree(m, src.data(), dst.data(), w.data(), p, lab.data(), prob.data(), &ex);
    if (nc != nc0 || lab != lab0 || std::memcmp(prob.data(), prob0.data(), 4 * m) != 0) {
      std::printf("FAIL the export changed the labels of case %d\n", cases);
      return 1;
    }
    const int ncl = static_cast<int>(ex.parent.size()), single = ex.single_root;
    std::fwrite(&nc, 4, 1, o);
    std::fwrite(lab.data(), 4, m, o);
    std::fwrite(prob.data(), 4, m, o);
    std::fwrite(&ncl, 4, 1, o);
    std::fwrite(&single, 4, 1, o);
    std::fwrite(&ex.thr, 8, 1, o);
    std::fwrite(ex.row_parent.data(), 4, m, o);
    std::fwrite(ex.row_lambda.data(), 8, m, o);
    std::fwrite(ex.parent.data(), 4, ncl, o);
    std::fwrite(ex.owner.data(), 4, ncl, o);
    std::fwrite(ex.label.data(), 4, ncl, o);
    std::fwrite(ex.birth.data(), 8, ncl, o);
    std::fwrite(ex.death.data(), 8, ncl, o);
    ++cases;
  }
  std::fclose(f);
  std::fclose(o);
  std::printf("PASS %d cases\n", cases);
  return 0;
}
