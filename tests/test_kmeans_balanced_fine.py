"""The assignment step of balanced k-means' stage 1 (include/raft_b200.h: b2d_debug_kmeans_balanced_fine_assign) against
a host brute force per group (tests/cpp/kmeans_balanced_fine_test.cu): compiled on the CPU tier, run on the GPU at
several column blocks and above 2^24 adjacency words; and its argument checks."""
import os
import subprocess

import pytest

import cpp_build
from raft_b200 import _lib

P = 1 << 12
E = _lib.B2D_ERR_INVALID_ARG


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return cpp_build.build("kmeans_balanced_fine_test.cu", str(tmp_path_factory.mktemp("kb_fine") / "kb_fine_test"))


def test_compiles(exe):
    assert os.path.exists(exe)


def test_argument_errors():
    def call(m=100, k=8, nc=16, G=4, ends=P, labels=P):
        rc = _lib.lib().b2d_debug_kmeans_balanced_fine_assign(None, P, k, m, k, ends, P, nc, ends, G, labels, P * 256,
                                                              1 << 40)
        return rc, _lib.lib().b2d_last_error().decode()
    assert call(nc=101) == (E, "n_clusters must be in [1, m]")
    for G in (0, 5):
        assert call(G=G) == (E, "num_groups must be in [1, round(sqrt(n_clusters))]")
    assert call(ends=None) == (E, "null row_ends / centroid_ends / labels")
    assert call(labels=None) == (E, "null row_ends / centroid_ends / labels")


@pytest.mark.gpu
def test_fine_assignment_is_the_arg_min_within_each_group(exe):
    res = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    print(res.stdout)
    assert res.returncode == 0 and "PASS" in res.stdout, res.stdout + res.stderr
