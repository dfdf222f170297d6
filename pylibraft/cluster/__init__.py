from . import kmeans  # noqa: F401
