"""The raft::cluster::hdbscan C++ shim (include/raft/cluster/hdbscan.cuh): compiled with and without the mock raft
headers on the CPU tier; on the GPU its labels, probabilities and cluster count equal raft_b200.cluster.hdbscan's bit for
bit."""
import os
import subprocess

import numpy as np
import pytest

import cpp_build


@pytest.fixture(scope="module")
def build_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("hdbscan_rbc_cpp"))


def compile_shim(build_dir, mock_raft):
    exe = os.path.join(build_dir, "hdb_shim_mockraft" if mock_raft else "hdb_shim")
    return cpp_build.build("hdbscan_rbc_shim_test.cu", exe, mock_raft)


@pytest.mark.parametrize("mock_raft", [False, True])
def test_shim_compiles(build_dir, mock_raft):
    assert os.path.exists(compile_shim(build_dir, mock_raft))


@pytest.mark.gpu
@pytest.mark.parametrize("mock_raft", [False, True])
def test_shim_runs_on_gpu_and_matches_python(build_dir, mock_raft):
    import torch
    from raft_b200.cluster import hdbscan
    exe = compile_shim(build_dir, mock_raft)
    m, d, mcs, ms = 5000, 3, 25, 7
    rng = np.random.default_rng(8)
    x = (rng.uniform(-40, 40, (6, d))[rng.integers(0, 6, m)] + rng.standard_normal((m, d))).astype(np.float32)
    inp, out = os.path.join(build_dir, "in.bin"), os.path.join(build_dir, "out.bin")
    with open(inp, "wb") as f:
        f.write(np.array([m, d, mcs, ms], np.int64).tobytes() + x.tobytes())
    res = subprocess.run([exe, inp, out], capture_output=True, text=True, timeout=120)
    assert res.returncode == 0 and "PASS" in res.stdout, res.stdout + res.stderr
    raw = np.fromfile(out, np.uint8)
    nc = int(raw[:4].view(np.int32)[0])
    lab = raw[4:4 + 4 * m].view(np.int32)
    prob = raw[4 + 4 * m:].view(np.float32)
    o = hdbscan(torch.from_numpy(x).cuda(), min_cluster_size=mcs, min_samples=ms)
    assert lab.tobytes() == o.labels.cpu().numpy().tobytes()
    assert prob.tobytes() == o.probabilities.cpu().numpy().tobytes()
    assert nc == o.n_clusters and nc >= 2
