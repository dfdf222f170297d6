"""The LinkageDistance::PAIRWISE forms of the C++ raft::cluster::single_linkage shim
(include/raft/cluster/single_linkage.cuh): compiled with and without the mock raft headers on the CPU tier; on the GPU
its dendrogram, labels, merge distances and sizes equal single_linkage(linkage="pairwise")'s bit for bit."""
import os
import subprocess

import numpy as np
import pytest

import cpp_build


@pytest.fixture(scope="module")
def build_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("single_linkage_rbc_cpp"))


def compile_shim(build_dir, mock_raft):
    exe = os.path.join(build_dir, "slr_shim_mockraft" if mock_raft else "slr_shim")
    return cpp_build.build("single_linkage_rbc_shim_test.cu", exe, mock_raft)


@pytest.mark.parametrize("mock_raft", [False, True])
def test_shim_compiles(build_dir, mock_raft):
    assert os.path.exists(compile_shim(build_dir, mock_raft))


@pytest.mark.gpu
@pytest.mark.parametrize("mock_raft", [False, True])
def test_shim_runs_on_gpu_and_matches_python(build_dir, mock_raft):
    import torch
    from raft_b200.cluster import single_linkage
    exe = compile_shim(build_dir, mock_raft)
    m, d, nc = 5000, 3, 7
    rng = np.random.default_rng(8)
    x = (rng.uniform(-40, 40, (nc, d))[rng.integers(0, nc, m)] + rng.standard_normal((m, d))).astype(np.float32)
    inp, out = os.path.join(build_dir, "in.bin"), os.path.join(build_dir, "out.bin")
    with open(inp, "wb") as f:
        f.write(np.array([m, d, nc], np.int64).tobytes() + x.tobytes())
    res = subprocess.run([exe, inp, out], capture_output=True, text=True, timeout=120)
    assert res.returncode == 0 and "PASS" in res.stdout, res.stdout + res.stderr
    raw = np.fromfile(out, np.uint8)
    n_ch = (m - 1) * 2 * 4
    got_ch = raw[:n_ch].view(np.int32).reshape(m - 1, 2)
    got_lab = raw[n_ch:n_ch + m * 4].view(np.int32)
    got_de = raw[n_ch + m * 4:n_ch + m * 4 + (m - 1) * 4].view(np.float32)
    got_sz = raw[n_ch + m * 4 + (m - 1) * 4:n_ch + m * 4 + 2 * (m - 1) * 4].view(np.int32)
    got_nc = raw[n_ch + m * 4 + 2 * (m - 1) * 4:].view(np.int32)[0]
    o = single_linkage(torch.from_numpy(x).cuda(), nc, linkage="pairwise")
    assert got_ch.tobytes() == o.children.cpu().numpy().tobytes()
    assert got_lab.tobytes() == o.labels.cpu().numpy().tobytes()
    assert got_de.tobytes() == o.deltas.cpu().numpy().tobytes()
    assert got_sz.tobytes() == o.sizes.cpu().numpy().tobytes()
    assert got_nc == o.n_connected_components == 1
    assert len(np.unique(got_lab)) == nc
