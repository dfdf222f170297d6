from raft_b200.distance import (DISTANCE_TYPES, SUPPORTED_DISTANCES, DistanceType, distance,  # noqa: F401
                                fused_distance_nn, fused_l2_nn_argmin, gram_matrix, pairwise_distance)
