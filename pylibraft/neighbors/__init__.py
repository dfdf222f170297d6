from raft_b200.neighbors import brute_force, epsilon_neighborhood  # noqa: F401
from raft_b200.neighbors.epsilon_neighborhood import eps_neighbors_l2sq  # noqa: F401
