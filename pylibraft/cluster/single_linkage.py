from raft_b200.cluster.single_linkage import LinkageOutput, mst, single_linkage  # noqa: F401
