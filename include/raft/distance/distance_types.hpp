// raft::distance::DistanceType -- enum of the removed raft/distance/distance_types.hpp
// (type name proven by cpp/include/raft/stats/silhouette_score.cuh:45 and
// cpp/include/raft/stats/detail/trustworthiness_score.cuh:80; values SURVEY.md 8(a1)).
#pragma once
namespace raft {
namespace distance {
enum DistanceType : unsigned short {
  L2Expanded          = 0,
  L2SqrtExpanded      = 1,
  CosineExpanded      = 2,
  L1                  = 3,
  L2Unexpanded        = 4,
  L2SqrtUnexpanded    = 5,
  InnerProduct        = 6,
  Linf                = 7,
  Canberra            = 8,
  LpUnexpanded        = 9,
  CorrelationExpanded = 10,
  JaccardExpanded     = 11,
  HellingerExpanded   = 12,
  Haversine           = 13,
  BrayCurtis          = 14,
  JensenShannon       = 15,
  HammingUnexpanded   = 16,
  KLDivergence        = 17,
  RusselRaoExpanded   = 18,
  DiceExpanded        = 19,
  Precomputed         = 100
};

namespace kernels {
// raft::distance::kernels::KernelType / KernelParams ([RECALLED] raft/distance/distance_types.hpp, <= 25.12): the kernel
// of a Gram matrix (raft/distance/kernels.cuh) and its parameters, gamma the gain and coef0 the offset
enum KernelType { LINEAR, POLYNOMIAL, RBF, TANH };

struct KernelParams {
  KernelType kernel;
  int degree;
  double gamma;
  double coef0;
};
}  // namespace kernels
}  // namespace distance
}  // namespace raft
