"""raft::cluster::hdbscan's prediction_model and approximate_predict (include/raft/cluster/hdbscan.cuh): compiled with and
without the mock raft headers on the CPU tier; on the GPU its predicted labels and probabilities equal
raft_b200.cluster.approximate_predict's bit for bit."""
import os
import subprocess

import numpy as np
import pytest

import cpp_build


@pytest.fixture(scope="module")
def build_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("hdbscan_predict_cpp"))


def compile_shim(build_dir, mock_raft):
    exe = os.path.join(build_dir, "hdb_predict_shim_mockraft" if mock_raft else "hdb_predict_shim")
    return cpp_build.build("hdbscan_predict_shim_test.cu", exe, mock_raft)


@pytest.mark.parametrize("mock_raft", [False, True])
def test_shim_compiles(build_dir, mock_raft):
    assert os.path.exists(compile_shim(build_dir, mock_raft))


@pytest.mark.gpu
@pytest.mark.parametrize("mock_raft", [False, True])
def test_shim_runs_on_gpu_and_matches_python(build_dir, mock_raft):
    import torch
    from raft_b200.cluster import approximate_predict, hdbscan_model
    exe = compile_shim(build_dir, mock_raft)
    m, d, mcs, ms, nq = 5000, 3, 25, 7, 2000
    rng = np.random.default_rng(8)
    c = rng.uniform(-40, 40, (6, d))
    x = (c[rng.integers(0, 6, m)] + rng.standard_normal((m, d))).astype(np.float32)
    q = (c[rng.integers(0, 6, nq)] + 2 * rng.standard_normal((nq, d))).astype(np.float32)
    inp, out = os.path.join(build_dir, "in.bin"), os.path.join(build_dir, "out.bin")
    with open(inp, "wb") as f:
        f.write(np.array([m, d, mcs, ms, nq], np.int64).tobytes() + x.tobytes() + q.tobytes())
    res = subprocess.run([exe, inp, out], capture_output=True, text=True, timeout=120)
    assert res.returncode == 0 and "PASS" in res.stdout, res.stdout + res.stderr
    raw = np.fromfile(out, np.uint8)
    lab, prob = raw[:4 * nq].view(np.int32), raw[4 * nq:].view(np.float32)
    model = hdbscan_model(torch.from_numpy(x).cuda(), min_cluster_size=mcs, min_samples=ms)
    p = approximate_predict(model, torch.from_numpy(q).cuda())
    assert lab.tobytes() == p.labels.cpu().numpy().tobytes()
    assert prob.tobytes() == p.probabilities.cpu().numpy().tobytes()
    assert len(set(lab.tolist()) - {-1}) >= 2
