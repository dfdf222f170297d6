"""The C++ shim of mean_shift (include/raft/cluster/mean_shift.cuh) on the GPU, built with and without the mock raft
headers: fit through mdspan views and the handle's workspace, compared with the Python call."""
import os
import subprocess

import numpy as np
import pytest
import torch

import cpp_build
from test_mean_shift_gpu import blobs


@pytest.fixture(scope="module")
def build_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("mean_shift_cpp"))


@pytest.mark.gpu
@pytest.mark.parametrize("seeding", ["rows", "bins", "seeds"])
@pytest.mark.parametrize("mock_raft", [False, True])
def test_shim_runs_on_gpu_and_matches_python(build_dir, mock_raft, seeding):
    from raft_b200.cluster import mean_shift
    exe = cpp_build.build("mean_shift_shim_test.cu", os.path.join(build_dir, "ms_shim_%d" % mock_raft), mock_raft)
    x = blobs(1500, 12, 5, 1.0, seed=21)
    seeds = x[::7].copy() if seeding == "seeds" else np.zeros((0, 12), np.float32)
    h = 1.0
    m, d = x.shape
    inp, out = os.path.join(build_dir, "in.bin"), os.path.join(build_dir, "out.bin")
    with open(inp, "wb") as f:
        f.write(np.array([m, d, len(seeds), int(seeding == "bins")], np.int64).tobytes() + np.float64(h).tobytes() +
                x.tobytes() + seeds.tobytes())
    res = subprocess.run([exe, inp, out], capture_output=True, text=True, timeout=120)
    assert res.returncode == 0 and "PASS" in res.stdout, res.stdout + res.stderr
    raw = np.fromfile(out, np.int32)
    nc, it = int(raw[0]), int(raw[1])
    got_c = raw[2:2 + nc * d].view(np.float32).reshape(nc, d)
    got_l = raw[2 + nc * d:]
    want = mean_shift(torch.from_numpy(x).cuda(), bandwidth=h, bin_seeding=seeding == "bins",
                      seeds=torch.from_numpy(seeds).cuda() if seeding == "seeds" else None)
    assert it == want.n_iter
    assert got_c.tobytes() == want.cluster_centers.cpu().numpy().tobytes()
    assert (got_l == want.labels.cpu().numpy()).all()
