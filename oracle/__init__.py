"""TEST INFRASTRUCTURE ONLY -- CPU oracle for the pairwise-distance / fusedL2NN hot path.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
may import this package.  The product (raft_b200) never does.

PARITY UNPINNED: the reference snapshot (raft 26.06) no longer contains
raft::distance (removed upstream in 26.02, CHANGELOG.md:59), so no reference test pins
results at this boundary.  The oracle restates the metric definitions (identical to
scipy.spatial.distance.cdist) in fp64 and is pinned against
  * scipy cdist fixtures (tests/golden/make_golden.py),
  * the adjacent reference pins that still exist:
      raft::argmin_op tie-break      cpp/tests/core/operators_host.cpp:134-152
      matrix::argmin known answer    cpp/tests/matrix/argmin.cu:71-75
      CompareApprox semantics        cpp/tests/test_utils.h:31-45
      rowNorm L2 vs naive            cpp/tests/linalg/norm.cu:42-77
"""
from .oracle import *  # noqa: F401,F403
