"""Mirror of the removed ``pylibraft.distance`` package (SURVEY.md 8(b))."""
from .distance_type import DISTANCE_TYPES, SUPPORTED_DISTANCES, DistanceType  # noqa: F401
from .fused_l2_nn import (fused_distance_nn, fused_l2_nn, fused_l2_nn_argmin, fused_l2_nn_sharded,  # noqa: F401
                          shard_bounds)
from .gram_matrix import KERNEL_TYPES, gram_matrix  # noqa: F401
from .masked_nn import masked_l2_nn  # noqa: F401
from .pairwise_distance import distance, pairwise_distance, pairwise_distance_raw  # noqa: F401
from .host_api import HostPairwise, pairwise_distance_host  # noqa: F401
