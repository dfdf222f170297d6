"""Drop-in alias: the subset of the ``pylibraft`` namespace that covers the distance path, served by
raft_b200 (the reference removed ``pylibraft.distance`` in 26.02; README.md:135-148 sends users to
cuVS).  ``from pylibraft.distance import pairwise_distance`` keeps working unchanged."""
from . import cluster, common, config, distance, matrix, neighbors, stats  # noqa: F401
