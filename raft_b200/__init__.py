"""raft_b200 -- Blackwell-native pairwise-distance / fusedL2NN engine behind the RAFT distance API.

Host-side mirror of the (removed) ``pylibraft.distance`` package over the C ABI in
``include/raft_b200.h``.  PyTorch is used for device memory and streams only.
"""
from . import cluster, common, distance, neighbors, stats  # noqa: F401
from ._lib import CudaError, LogicError, RaftB200Error  # noqa: F401

__version__ = "0.1.0"
