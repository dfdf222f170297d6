"""The C++ raft::cluster::kmeans_balanced shim (include/raft/cluster/kmeans_balanced.cuh): compiled with and without the
mock raft headers on the CPU tier; on the GPU its fit_predict equals the Python fit_predict bit for bit, its uint32
predict equals the Python predict, and a cosine metric throws raft::logic_error."""
import os
import subprocess

import numpy as np
import pytest

import cpp_build
import kmeans_ref


@pytest.fixture(scope="module")
def build_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("kmeans_balanced_cpp"))


def compile_shim(build_dir, mock_raft):
    exe = os.path.join(build_dir, "kmeans_balanced_shim_mockraft" if mock_raft else "kmeans_balanced_shim")
    return cpp_build.build("kmeans_balanced_shim_test.cu", exe, mock_raft)


@pytest.mark.parametrize("mock_raft", [False, True])
def test_shim_compiles(build_dir, mock_raft):
    assert os.path.exists(compile_shim(build_dir, mock_raft))


@pytest.mark.gpu
@pytest.mark.parametrize("mock_raft", [False, True])
def test_shim_runs_on_gpu_and_matches_python(build_dir, mock_raft):
    import torch
    from raft_b200.cluster import kmeans_balanced as kb
    exe = compile_shim(build_dir, mock_raft)
    m, k, nc = 20000, 48, 100
    x, _, _ = kmeans_ref.blobs(m, k, 30, seed=33, spread=0.3)
    inp, out = os.path.join(build_dir, "in.bin"), os.path.join(build_dir, "out.bin")
    with open(inp, "wb") as f:
        f.write(np.array([m, k, nc], np.int64).tobytes() + x.tobytes())
    res = subprocess.run([exe, inp, out], capture_output=True, text=True, timeout=120)
    assert res.returncode == 0 and "PASS" in res.stdout, res.stdout + res.stderr
    raw = np.fromfile(out, np.uint8)
    got_c = raw[:nc * k * 4].view(np.float32).reshape(nc, k)
    got_l = raw[nc * k * 4:nc * k * 4 + m * 4].view(np.int32)
    got_u = raw[nc * k * 4 + m * 4:].view(np.uint32)
    p = kb.KMeansBalancedParams(n_iters=10, seed=7)
    xd = torch.from_numpy(x).cuda()
    c, lab, _ = kb.fit_predict(p, xd, nc)
    c = torch.as_tensor(c, device="cuda")
    assert got_c.tobytes() == c.cpu().numpy().tobytes()
    assert got_l.tobytes() == torch.as_tensor(lab, device="cuda").cpu().numpy().tobytes()
    pl = torch.as_tensor(kb.predict(p, xd, c), device="cuda").cpu().numpy()
    assert got_u.tobytes() == pl.astype(np.uint32).tobytes()
