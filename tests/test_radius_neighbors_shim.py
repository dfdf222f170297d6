"""The C++ shim of radius_neighbors (include/raft/neighbors/radius_neighbors.cuh) on the GPU, built with and without the
mock raft headers: both calls through mdspan views and the handle's workspace, compared with the Python call."""
import os
import subprocess

import numpy as np
import pytest
import torch

import cpp_build
import oracle
from radius_ref import METRIC_IDS


@pytest.fixture(scope="module")
def build_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("radius_cpp"))


@pytest.mark.gpu
@pytest.mark.parametrize("metric", ["sqeuclidean", "cosine"])
@pytest.mark.parametrize("mock_raft", [False, True])
def test_shim_runs_on_gpu_and_matches_python(build_dir, mock_raft, metric):
    from raft_b200.neighbors import radius_neighbors
    exe = cpp_build.build("radius_shim_test.cu", os.path.join(build_dir, "radius_shim_%d" % mock_raft), mock_raft)
    q, _, c = oracle.make_blobs(1000, 24, seed=51)
    x, _, _ = oracle.make_blobs(1030, 24, seed=52, centers=c)
    radius = np.float32(30.0 if metric == "sqeuclidean" else 0.1)
    m, n, d = q.shape[0], x.shape[0], q.shape[1]
    inp, out = os.path.join(build_dir, "in.bin"), os.path.join(build_dir, "out.bin")
    with open(inp, "wb") as f:
        f.write(np.array([m, n, d, METRIC_IDS[metric]], np.int64).tobytes() + radius.tobytes() + q.tobytes() + x.tobytes())
    res = subprocess.run([exe, inp, out], capture_output=True, text=True, timeout=120)
    assert res.returncode == 0 and "PASS" in res.stdout, res.stdout + res.stderr
    raw = np.fromfile(out, np.uint8)
    indptr = raw[:8 * (m + 1)].view(np.int64)
    nnz = int(indptr[-1])
    indices = raw[8 * (m + 1):8 * (m + 1 + nnz)].view(np.int64)
    dists = raw[8 * (m + 1 + nnz):].view(np.float32)
    p, i, dd = radius_neighbors(torch.from_numpy(x).cuda(), torch.from_numpy(q).cuda(), float(radius), metric=metric)
    assert nnz > m
    assert np.array_equal(indptr, p.cpu().numpy()) and np.array_equal(indices, i.cpu().numpy())
    assert np.array_equal(dists.view(np.int32), dd.cpu().numpy().view(np.int32))
