"""The C++ raft::cluster::kmeans shim's k-means|| route (include/raft/cluster/kmeans.cuh): compiled with and without the
mock raft headers on the CPU tier; on the GPU a fit with oversampling_factor = 2 equals the Python k-means|| fit bit for
bit, and a default-constructed KMeansParams equals the Python greedy fit."""
import os
import subprocess

import numpy as np
import pytest

import cpp_build
import kmeans_ref


@pytest.fixture(scope="module")
def build_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("kmeans_scalable_cpp"))


def compile_shim(build_dir, mock_raft):
    exe = os.path.join(build_dir, "kmeans_scalable_shim_mockraft" if mock_raft else "kmeans_scalable_shim")
    return cpp_build.build("kmeans_scalable_shim_test.cu", exe, mock_raft)


@pytest.mark.parametrize("mock_raft", [False, True])
def test_shim_compiles(build_dir, mock_raft):
    assert os.path.exists(compile_shim(build_dir, mock_raft))


@pytest.mark.gpu
@pytest.mark.parametrize("mock_raft", [False, True])
def test_shim_runs_on_gpu_and_matches_python(build_dir, mock_raft):
    import torch
    from raft_b200.cluster import KMeansParams, fit
    exe = compile_shim(build_dir, mock_raft)
    m, k, nc = 20000, 48, 13
    x, _, _ = kmeans_ref.blobs(m, k, nc, seed=33, spread=0.3)
    inp, out = os.path.join(build_dir, "in.bin"), os.path.join(build_dir, "out.bin")
    with open(inp, "wb") as f:
        f.write(np.array([m, k, nc], np.int64).tobytes() + x.tobytes())
    res = subprocess.run([exe, inp, out], capture_output=True, text=True, timeout=120)
    assert res.returncode == 0 and "PASS" in res.stdout, res.stdout + res.stderr
    raw = np.fromfile(out, np.uint8)
    xd = torch.from_numpy(x).cuda()
    step = nc * k * 4 + 8
    for v, f in enumerate((2.0, None)):
        got = raw[v * step:(v + 1) * step]
        got_c = got[:nc * k * 4].view(np.float32).reshape(nc, k)
        got_in = got[nc * k * 4:][:4].view(np.float32)[0]
        got_it = got[nc * k * 4 + 4:][:4].view(np.int32)[0]
        o = fit(KMeansParams(n_clusters=nc, seed=7, oversampling_factor=f), xd)
        assert got_c.tobytes() == torch.as_tensor(o.centroids, device="cuda").cpu().numpy().tobytes(), f
        assert got_it == o.n_iter and got_in == np.float32(o.inertia), f
