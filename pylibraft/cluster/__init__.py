from . import kmeans, single_linkage  # noqa: F401
