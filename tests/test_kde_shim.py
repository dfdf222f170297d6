"""The C++ shim of kernel_density (include/raft/neighbors/kernel_density.cuh) on the GPU, built with and without the mock
raft headers: score_samples through mdspan views and the handle's workspace, compared with the Python call."""
import os
import subprocess

import numpy as np
import pytest
import torch

import cpp_build
import oracle


@pytest.fixture(scope="module")
def build_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("kde_cpp"))


@pytest.mark.gpu
@pytest.mark.parametrize("kernel,weighted", [(0, False), (2, True), (5, True)])
@pytest.mark.parametrize("mock_raft", [False, True])
def test_shim_runs_on_gpu_and_matches_python(build_dir, mock_raft, kernel, weighted):
    from raft_b200.neighbors import kernel_density
    from raft_b200.neighbors.kernel_density import KERNELS
    exe = cpp_build.build("kde_shim_test.cu", os.path.join(build_dir, "kde_shim_%d" % mock_raft), mock_raft)
    q, _, c = oracle.make_blobs(1000, 24, seed=61)
    x, _, _ = oracle.make_blobs(1030, 24, seed=62, centers=c)
    w = np.random.default_rng(4).uniform(0, 2, 1030).astype(np.float32)
    h = 8.0   # (about the distance between rows of one blob)
    m, n, d = q.shape[0], x.shape[0], q.shape[1]
    inp, out = os.path.join(build_dir, "in.bin"), os.path.join(build_dir, "out.bin")
    with open(inp, "wb") as f:
        f.write(np.array([m, n, d, kernel, int(weighted)], np.int64).tobytes() + np.float64(h).tobytes() + q.tobytes() +
                x.tobytes() + (w.tobytes() if weighted else b""))
    res = subprocess.run([exe, inp, out], capture_output=True, text=True, timeout=120)
    assert res.returncode == 0 and "PASS" in res.stdout, res.stdout + res.stderr
    got = np.fromfile(out, np.float64)
    want = kernel_density(torch.from_numpy(x).cuda(), torch.from_numpy(q).cuda(), bandwidth=h, kernel=KERNELS[kernel],
                          sample_weight=torch.from_numpy(w).cuda() if weighted else None).cpu().numpy()
    assert np.isfinite(got).sum() > m // 2
    assert np.array_equal(got.view(np.int64), want.view(np.int64))
