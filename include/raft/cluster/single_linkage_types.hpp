// raft::cluster linkage types -- shim of the removed raft/cluster/single_linkage_types.hpp ([RECALLED], <= 25.12).
#pragma once

namespace raft {
namespace cluster {

// How the graph the MST is built on is formed: KNN_GRAPH (include/raft_b200.h, b2d_single_linkage) or, for d = 2 and 3,
// PAIRWISE, the complete graph (b2d_single_linkage_rbc).
enum LinkageDistance { PAIRWISE = 0, KNN_GRAPH = 1 };

// The dendrogram and flat labels of a linkage ([RECALLED] raft::cluster::linkage_output): device pointers owned by the
// caller: children [m - 1][2], labels [m].  The merge distances and sizes are not members; the pointer form of
// single_linkage takes them as optional outputs.
template <typename idx_t>
class linkage_output {
 public:
  idx_t m;
  idx_t n_clusters;
  idx_t n_leaves;
  idx_t n_connected_components;
  idx_t* labels;     // [m]
  idx_t* children;   // [m - 1][2]
};

}  // namespace cluster
}  // namespace raft
