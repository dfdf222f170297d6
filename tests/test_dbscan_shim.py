"""The C++ raft::cluster::dbscan shim (include/raft/cluster/dbscan.cuh): compiled with and without the mock raft headers
on the CPU tier; on the GPU both its forms give the labels and core sample indices of the Python call, bit for bit."""
import os
import subprocess

import numpy as np
import pytest

import cpp_build


@pytest.fixture(scope="module")
def build_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("dbscan_cpp"))


def compile_shim(build_dir, mock_raft):
    exe = os.path.join(build_dir, "db_shim_mockraft" if mock_raft else "db_shim")
    return cpp_build.build("dbscan_shim_test.cu", exe, mock_raft)


@pytest.mark.parametrize("mock_raft", [False, True])
def test_shim_compiles(build_dir, mock_raft):
    assert os.path.exists(compile_shim(build_dir, mock_raft))


@pytest.mark.gpu
@pytest.mark.parametrize("mock_raft", [False, True])
def test_shim_runs_on_gpu_and_matches_python(build_dir, mock_raft):
    import torch
    from raft_b200.cluster import dbscan
    exe = compile_shim(build_dir, mock_raft)
    m, d, ms, eps = 3000, 12, 10, np.float32(4.0)
    rng = np.random.default_rng(8)
    x = (rng.uniform(-15, 15, (20, d))[rng.integers(0, 20, m)] + rng.standard_normal((m, d))).astype(np.float32)
    x[rng.random(m) < 0.1] = rng.uniform(-16, 16, d).astype(np.float32)
    inp, out = os.path.join(build_dir, "in.bin"), os.path.join(build_dir, "out.bin")
    with open(inp, "wb") as f:
        f.write(np.array([m, d, ms], np.int64).tobytes() + eps.tobytes() + x.tobytes())
    res = subprocess.run([exe, inp, out], capture_output=True, text=True, timeout=120)
    assert res.returncode == 0 and "PASS" in res.stdout, res.stdout + res.stderr
    raw = np.fromfile(out, np.int32)
    o = dbscan(torch.from_numpy(x).cuda(), float(eps), min_samples=ms)
    lab = o.labels.cpu().numpy()
    assert raw[:m].tobytes() == lab.tobytes()
    n = o.core_sample_indices.numel()
    assert raw[m:m + n].tobytes() == o.core_sample_indices.cpu().numpy().tobytes() and (raw[m + n:] == -1).all()
    assert o.n_clusters > 1 and (lab == -1).any()
