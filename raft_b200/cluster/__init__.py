from .kmeans import (  # noqa: F401
    FitOutput, KMeansParams, cluster_cost, compute_new_centroids, fit, init_plus_plus, init_scalable, predict,
)
from . import kmeans_balanced  # noqa: F401  (a module: its fit / predict are not k-means')
from .dbscan import DbscanOutput, dbscan  # noqa: F401
from .mean_shift import MeanShiftOutput, estimate_bandwidth, mean_shift  # noqa: F401
from .single_linkage import LinkageOutput, MstOutput, mst, single_linkage  # noqa: F401
