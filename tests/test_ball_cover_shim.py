"""The C++ shim of the ball cover (include/raft/neighbors/ball_cover.cuh) on the GPU, built with and without the mock raft
headers: build, knn_query, all_knn_query and the two eps_nn calls through mdspan views and the handle's workspace,
compared with the Python calls byte for byte."""
import os
import subprocess

import numpy as np
import pytest
import torch

import cpp_build
from ball_cover_ref import METRIC_IDS


@pytest.fixture(scope="module")
def build_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("ball_cover_cpp"))


@pytest.mark.gpu
@pytest.mark.parametrize("metric", ["sqeuclidean", "euclidean"])
@pytest.mark.parametrize("mock_raft", [False, True])
def test_shim_runs_on_gpu_and_matches_python(build_dir, mock_raft, metric):
    from raft_b200.neighbors import ball_cover
    exe = cpp_build.build("ball_cover_shim_test.cu", os.path.join(build_dir, "bc_shim_%d" % mock_raft), mock_raft)
    r = np.random.default_rng(61)
    n, m, d, k = 3000, 500, 3, 24
    x = r.random((n, d), dtype=np.float32)
    q = r.random((m, d), dtype=np.float32)
    eps = np.float32(0.01 if metric == "sqeuclidean" else 0.1)
    inp, out = os.path.join(build_dir, "in.bin"), os.path.join(build_dir, "out.bin")
    with open(inp, "wb") as f:
        f.write(np.array([n, m, d, METRIC_IDS[metric], k], np.int64).tobytes() + eps.tobytes() + x.tobytes() + q.tobytes())
    res = subprocess.run([exe, inp, out], capture_output=True, text=True, timeout=120)
    assert res.returncode == 0 and "PASS" in res.stdout, res.stdout + res.stderr
    raw = np.fromfile(out, np.uint8)
    parts, at = [], 0
    for count, dt in ((m * k, np.int64), (m * k, np.float32), (n * k, np.int64), (m + 1, np.int64)):
        nb = count * np.dtype(dt).itemsize
        parts.append(raw[at:at + nb].view(dt))
        at += nb
    nnz = int(parts[3][-1])
    parts.append(raw[at:at + 8 * nnz].view(np.int64))
    parts.append(raw[at + 8 * nnz:].view(np.float32))
    xd, qd = torch.from_numpy(x).cuda(), torch.from_numpy(q).cuda()
    index = ball_cover.build_index(xd, metric=metric)
    dist, idx = ball_cover.knn_query(index, qd, k)
    _, aidx = ball_cover.all_knn_query(index, k)
    want = [idx, dist, aidx] + list(ball_cover.eps_nn(index, qd, float(eps)))
    assert nnz > m
    for got, w in zip(parts, want):
        w = w.cpu().numpy().reshape(-1)
        assert got.dtype == w.dtype and np.array_equal(got.view(np.uint8), w.view(np.uint8))
