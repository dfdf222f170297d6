from raft_b200.cluster.single_linkage import EmstOutput, LinkageOutput, emst, mst, single_linkage  # noqa: F401
