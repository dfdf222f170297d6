from .kmeans import (  # noqa: F401
    FitOutput, KMeansParams, cluster_cost, compute_new_centroids, fit, init_plus_plus, predict,
)
from .dbscan import DbscanOutput, dbscan  # noqa: F401
from .single_linkage import LinkageOutput, MstOutput, mst, single_linkage  # noqa: F401
