// raft::cluster::kmeans_balanced_params -- shim of the removed raft/cluster/kmeans_balanced_types.hpp ([RECALLED],
// <= 25.12): the parameters of hierarchical balanced k-means (include/raft/cluster/kmeans_balanced.cuh).
#pragma once
#include <cstdint>

#include "../distance/distance.cuh"

namespace raft {
namespace cluster {

struct kmeans_base_params {
  raft::distance::DistanceType metric = raft::distance::DistanceType::L2Expanded;   // the only metric supported
};

struct kmeans_balanced_params : kmeans_base_params {
  uint32_t n_iters = 20;   // balanced-EM iterations of the mesocluster and fine stages (final pass: max(n_iters / 10, 2))
  uint64_t seed    = 0;    // keys the Philox draws of the adjust step (a project addition: the reference had no seed)
};

}  // namespace cluster
}  // namespace raft
