from raft_b200.cluster.kmeans import (  # noqa: F401
    FitOutput, KMeansParams, cluster_cost, compute_new_centroids, fit, init_plus_plus, init_scalable, predict,
)
