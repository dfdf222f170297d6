"""The C++ raft::cluster::kmeans shim (include/raft/cluster/kmeans.cuh): compiled with and without the mock raft headers
on the CPU tier; on the GPU its fit / predict / cluster_cost results equal the Python calls bit for bit."""
import os
import subprocess

import numpy as np
import pytest

import cpp_build
import kmeans_ref



@pytest.fixture(scope="module")
def build_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("kmeans_cpp"))


def compile_shim(build_dir, mock_raft):
    exe = os.path.join(build_dir, "kmeans_shim_mockraft" if mock_raft else "kmeans_shim")
    return cpp_build.build("kmeans_shim_test.cu", exe, mock_raft)


@pytest.mark.parametrize("mock_raft", [False, True])
def test_shim_compiles(build_dir, mock_raft):
    assert os.path.exists(compile_shim(build_dir, mock_raft))


@pytest.mark.gpu
@pytest.mark.parametrize("mock_raft", [False, True])
def test_shim_runs_on_gpu_and_matches_python(build_dir, mock_raft):
    import torch
    from raft_b200.cluster import KMeansParams, fit, predict
    exe = compile_shim(build_dir, mock_raft)
    m, k, nc = 20000, 48, 13
    x, _, _ = kmeans_ref.blobs(m, k, nc, seed=31, spread=0.3)
    c0 = x[np.random.default_rng(5).choice(m, nc, replace=False)]
    inp, out = os.path.join(build_dir, "in.bin"), os.path.join(build_dir, "out.bin")
    with open(inp, "wb") as f:
        f.write(np.array([m, k, nc], np.int64).tobytes() + x.tobytes() + c0.tobytes())
    res = subprocess.run([exe, inp, out], capture_output=True, text=True, timeout=120)
    assert res.returncode == 0 and "PASS" in res.stdout, res.stdout + res.stderr
    raw = np.fromfile(out, np.uint8)
    got_c = raw[:nc * k * 4].view(np.float32).reshape(nc, k)
    got_l = raw[nc * k * 4:nc * k * 4 + m * 4].view(np.int32)
    got_in = raw[nc * k * 4 + m * 4:][:4].view(np.float32)[0]
    got_it = raw[nc * k * 4 + m * 4 + 4:][:4].view(np.int32)[0]
    c = torch.from_numpy(c0.copy()).cuda()
    xd = torch.from_numpy(x).cuda()
    o = fit(KMeansParams(n_clusters=nc, max_iter=25, tol=1e-4, init_method="Array"), xd, c)
    assert got_c.tobytes() == c.cpu().numpy().tobytes()
    assert got_it == o.n_iter and got_in == np.float32(o.inertia)
    labels, _ = predict(KMeansParams(n_clusters=nc), xd, c)
    assert (got_l == torch.as_tensor(labels, device="cuda").cpu().numpy()).all()
