"""eps_neighbors_l2sq without a GPU: the workspace query, every argument check of the C ABI, B2D_ERR_CUDA without a
device, the fp64 reference of the GPU tier (tests/eps_ref.py) checked against scipy, and the C++ shim's compile (its run
on the GPU is marked gpu)."""
import os
import subprocess

import numpy as np
import pytest
import torch
from scipy.spatial.distance import cdist

import cpp_build
from eps_ref import ref_eps
from raft_b200 import _lib


SIZE_MAX = 2 ** 64 - 1
P = 1 << 12   # a non-null pointer that is never dereferenced (every call below fails before any work)


def call(adj=P, ld_adj=100, vd=P, vd64=1, init=1, x=P, ldx=8, y=P, ldy=8, m=10, n=100, k=8, eps=1.0, ws=P * 256,
         wsb=1 << 40):
    return _lib.lib().b2d_eps_neighbors_l2sq(None, adj, ld_adj, vd, vd64, init, x, ldx, y, ldy, m, n, k, eps, ws, wsb)


def test_workspace_query():
    L = _lib.lib()
    assert L.b2d_eps_neighbors_l2sq_workspace_bytes(-1, 5, 3) == SIZE_MAX
    assert L.b2d_eps_neighbors_l2sq_workspace_bytes(5, -1, 3) == SIZE_MAX
    assert L.b2d_eps_neighbors_l2sq_workspace_bytes(5, 5, -3) == SIZE_MAX
    for m, n, k in ((1000, 2000, 32), (100000, 100000, 128), (7, 9, 320)):
        assert L.b2d_eps_neighbors_l2sq_workspace_bytes(m, n, k) == L.b2d_pairwise_workspace_bytes(0, _lib.B2D_F32, m, n, k)


def test_argument_errors():
    E = _lib.B2D_ERR_INVALID_ARG
    assert call(k=321) == _lib.B2D_ERR_UNSUPPORTED
    assert call(adj=None, vd=None) == E
    assert call(ld_adj=99) == E
    assert call(x=None) == E
    assert call(y=None) == E
    assert call(ldx=7) == E and call(ldy=7) == E
    assert call(k=0) == E
    assert call(m=-1) == E and call(n=-1) == E
    assert call(m=2 ** 31) == E and call(n=2 ** 31, ld_adj=2 ** 31) == E
    assert call(wsb=10) == _lib.B2D_ERR_WORKSPACE
    assert call(ws=None) == _lib.B2D_ERR_WORKSPACE
    assert call(ws=P * 256 + 16) == E
    # count-only and adjacency-only pass the checks that the adjacency pitch needs only when adj is given
    assert call(adj=None, ld_adj=0, init=0, wsb=10) == _lib.B2D_ERR_WORKSPACE
    # nothing to do: OK without touching anything
    assert call(m=0, x=None, y=None, init=0) == _lib.B2D_OK
    with pytest.raises(_lib.LogicError):
        _lib.check(call(k=321))


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the error without a device")
def test_cuda_error_without_device():
    assert call(m=0, init=1) == _lib.B2D_ERR_CUDA        # zeroing vd is the only work
    assert call() == _lib.B2D_ERR_CUDA


def test_reference_matches_scipy():
    rng = np.random.default_rng(3)
    x = rng.normal(size=(70, 13)).astype(np.float32)
    y = rng.normal(size=(90, 13)).astype(np.float32)
    d = cdist(x.astype(np.float64), y.astype(np.float64), "sqeuclidean")
    eps = float(np.quantile(d, 0.1))
    adj, vd, clear = ref_eps(x, y, eps)
    assert 0 < clear.sum() < clear.size or clear.all()
    assert (adj[clear] == (d <= eps)[clear]).all()
    cols = clear.all(0)   # columns without a pair in the band: their counts are exact
    assert cols.sum() > 40
    assert (vd[:-1][cols] == (d <= eps).sum(0)[cols]).all()
    assert vd[-1] == adj.sum() and len(vd) == 91


@pytest.fixture(scope="module")
def build_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("eps_cpp"))


def compile_shim(build_dir, mock_raft):
    exe = os.path.join(build_dir, "eps_shim_mockraft" if mock_raft else "eps_shim")
    return cpp_build.build("eps_shim_test.cu", exe, mock_raft)


@pytest.mark.parametrize("mock_raft", [False, True])
def test_shim_compiles(build_dir, mock_raft):
    assert os.path.exists(compile_shim(build_dir, mock_raft))


@pytest.mark.gpu
@pytest.mark.parametrize("mock_raft", [False, True])
def test_shim_runs_on_gpu_and_matches_python(build_dir, mock_raft):
    from raft_b200.neighbors import eps_neighbors_l2sq
    exe = compile_shim(build_dir, mock_raft)
    rng = np.random.default_rng(17)
    m, n, k = 1000, 1030, 24
    x = rng.normal(size=(m, k)).astype(np.float32)
    y = rng.normal(size=(n, k)).astype(np.float32)
    eps = np.float32(30.0)
    inp, out = os.path.join(build_dir, "in.bin"), os.path.join(build_dir, "out.bin")
    with open(inp, "wb") as f:
        f.write(np.array([m, n, k], np.int64).tobytes() + eps.tobytes() + x.tobytes() + y.tobytes())
    res = subprocess.run([exe, inp, out], capture_output=True, text=True, timeout=120)
    assert res.returncode == 0 and "PASS" in res.stdout, res.stdout + res.stderr
    raw = np.fromfile(out, np.uint8)
    adj_c, vd_c = raw[:m * n].reshape(m, n), raw[m * n:].view(np.int64)
    adj, vd = eps_neighbors_l2sq(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), float(eps))
    assert (adj_c.astype(bool) == adj.cpu().numpy()).all()
    assert (vd_c == vd.cpu().numpy()).all()
