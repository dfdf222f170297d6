from raft_b200.matrix import select_k  # noqa: F401
