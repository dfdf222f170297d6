"""mean_shift without a GPU: the fp64 model of the GPU tier (tests/mean_shift_ref.py) pinned to sklearn.cluster.MeanShift,
every argument check of the C call with its status and message, the workspace query and its recorded contract
(tests/golden/mean_shift_workspace_contract.json), and B2D_ERR_CUDA without a device."""
import numpy as np
import pytest
import torch
from sklearn.cluster import MeanShift

import mean_shift_ref as R
from raft_b200 import _lib
from test_workspace_contract import load, replay_bytes, replay_errors

SIZE_MAX = 2 ** 64 - 1
P = 1 << 12   # a non-null pointer that is never dereferenced (every call below fails before any work)
E, U, W = _lib.B2D_ERR_INVALID_ARG, _lib.B2D_ERR_UNSUPPORTED, _lib.B2D_ERR_WORKSPACE
CONTRACT = "mean_shift_workspace_contract.json"


def fit(x=P, ldx=8, n=100, d=8, h=1.0, seeds=None, lds=8, ns=0, bins=0, mbf=1, call=1, max_iter=300, mb=0, c=P, nc=P,
        lab=P, it=P, ws=P * 256, wsb=1 << 40):
    return _lib.lib().b2d_mean_shift_fit(None, x, ldx, n, d, h, seeds, lds, ns, bins, mbf, call, max_iter, mb, c, nc, lab,
                                         it, ws, wsb)


def status(rc):
    return rc, _lib.lib().b2d_last_error().decode()


# ---------------------------------------------------------------------------------------------------------------- model
def blobs(seed, n_per=30, d=2, centres=((0, 0), (6, 0), (0, 6)), std=0.4, dup=0):
    rng = np.random.default_rng(seed)
    c = np.asarray(centres, np.float64)[:, :d]
    x = np.concatenate([ci + std * rng.normal(size=(n_per, d)) for ci in c]).astype(np.float32)
    if dup:
        x = np.concatenate([x, x[:dup]])
    return x


def sk(x, h, **kw):
    ms = MeanShift(bandwidth=h, **kw).fit(x.astype(np.float64))
    return ms.cluster_centers_, ms.labels_, ms.n_iter_


def model(x, h, **kw):
    return R.mean_shift(x, h, R.exact_within(h), R.exact_d2, h2=h * h, **kw)


CASES = [
    ("every row a seed", blobs(0), 2.0, {}),
    ("bin seeding", blobs(1, n_per=60), 1.5, {"bin_seeding": True}),
    ("bin seeding min_bin_freq=5", blobs(2, n_per=60), 1.5, {"bin_seeding": True, "min_bin_freq": 5}),
    ("explicit seeds", blobs(3), 2.0, {"seeds": np.array([[0.5, 0.5], [5.5, 0.2], [0.1, 6.3], [3, 3]], np.float32)}),
    ("cluster_all=False", blobs(4, centres=((0, 0), (6, 0), (0, 6), (30, 30))), 2.0, {"cluster_all": False}),
    ("dropped seeds", blobs(5), 2.0, {"seeds": np.array([[0.2, 0.1], [100, 100], [6, 0.3], [-50, 4]], np.float32)}),
    ("duplicate rows", blobs(6, dup=20), 2.0, {}),
    ("max_iter=0", blobs(7), 2.0, {"max_iter": 0}),
    ("max_iter=1", blobs(8), 2.0, {"max_iter": 1}),
    ("d=3", blobs(9, d=3, centres=((0, 0, 0), (6, 0, 1), (0, 6, 2))), 2.0, {}),
]


@pytest.mark.parametrize("name,x,h,kw", CASES, ids=[c[0] for c in CASES])
def test_model_matches_sklearn(name, x, h, kw):
    sc, sl, si = sk(x, h, **{k: v for k, v in kw.items()})
    mc, ml, mi = model(x, h, **kw)
    assert mi == si
    assert mc.shape == sc.shape
    np.testing.assert_allclose(mc, sc, rtol=0, atol=1e-5)
    assert (ml == sl).all()


def test_model_no_neighbour_error():
    x = blobs(10)
    seeds = np.array([[100, 100], [-100, 3]], np.float32)
    with pytest.raises(ValueError, match="No point was within bandwidth"):
        sk(x, 1.0, seeds=seeds)
    with pytest.raises(ValueError, match="No point was within bandwidth"):
        model(x, 1.0, seeds=seeds)


def test_bin_seeds_match_sklearn():
    from sklearn.cluster import get_bin_seeds
    x = blobs(11, n_per=80)
    for h, f in ((1.0, 1), (1.0, 4), (0.3, 2), (1e-3, 1)):
        got = R.bin_seeds(x, h, f)
        want = get_bin_seeds(x.astype(np.float64), h, f)
        assert {tuple(r) for r in np.asarray(got, np.float64)} == {tuple(r) for r in np.asarray(want, np.float64)}


def test_model_seed_order_free():
    x = blobs(12)
    rng = np.random.default_rng(0)
    seeds = x[rng.permutation(len(x))[:40]]
    a = model(x, 2.0, seeds=seeds)
    b = model(x, 2.0, seeds=seeds[::-1].copy())
    assert a[2] == b[2] and (a[0] == b[0]).all() and (a[1] == b[1]).all()


# ------------------------------------------------------------------------------------------------------------- C ABI
def test_workspace_query():
    L = _lib.lib()
    for args in ((-1, 5, 0, 0), (5, -1, 0, 0), (5, 5, -1, 0), (5, 5, 0, -1)):
        assert L.b2d_mean_shift_fit_workspace_bytes(*args) == SIZE_MAX
    # seeds given: no bin-seeding regions; the batch bound shrinks the adjacency
    n, d = 100000, 32
    assert L.b2d_mean_shift_fit_workspace_bytes(n, d, 1000, 0) < L.b2d_mean_shift_fit_workspace_bytes(n, d, 0, 0)
    small = L.b2d_mean_shift_fit_workspace_bytes(n, d, 0, 128 * n)
    big = L.b2d_mean_shift_fit_workspace_bytes(n, d, 0, 256 * n)
    assert 128 * n <= big - small < 128 * n + 128 * 49 * (d * 4 + 4) + 8192
    # a bound below one 128-seed batch still forms 128 seeds at once
    assert L.b2d_mean_shift_fit_workspace_bytes(n, d, 0, 1) == small


def test_workspace_contract_bytes():
    rows = replay_bytes(load(CONTRACT), "b2d_mean_shift_fit_workspace_bytes")
    assert len(rows) >= 100
    for *args, want in rows:
        assert (want == SIZE_MAX) == (min(args) < 0), args


def test_workspace_contract_errors():
    assert replay_errors(load(CONTRACT)) == 12


def test_argument_errors():
    for kw in ({"n": -1}, {"d": -1}, {"ns": -1}, {"mb": -1}):
        assert status(fit(**kw)) == (E, "negative extent, seed count or batch size")
    assert status(fit(n=2 ** 31)) == (E, "mean_shift: n and n_seeds must be below 2^31")
    assert status(fit(ns=2 ** 31, seeds=P)) == (E, "mean_shift: n and n_seeds must be below 2^31")
    assert status(fit(d=0)) == (E, "d must be positive")
    assert status(fit(d=321, ldx=321, lds=321)) == (U, "mean_shift supports d <= 320 (the whole distance at once)")
    for h in (0.0, -1.0, float("inf"), float("nan")):
        assert status(fit(h=h)) == (E, "bandwidth must be finite and > 0")
    assert status(fit(h=1e20)) == (E, "bandwidth^2 is not finite in fp32")
    assert status(fit(max_iter=-1)) == (E, "max_iter must be >= 0")
    assert status(fit(seeds=P)) == (E, "seeds and n_seeds: both or neither")
    assert status(fit(ns=3)) == (E, "seeds and n_seeds: both or neither")
    assert status(fit(seeds=P, ns=3, lds=7)) == (E, "seeds leading dimension smaller than d")
    assert status(fit(bins=1, mbf=0)) == (E, "min_bin_freq must be >= 1")
    assert status(fit(n=0)) == (E, "n must be positive")
    for kw in ({"x": None}, {"c": None}, {"lab": None}, {"nc": None}):
        assert status(fit(**kw)) == (E, "null x / centers / labels / n_centers")
    assert status(fit(ldx=7)) == (E, "leading dimension smaller than d")
    assert status(fit(wsb=10))[0] == W
    assert status(fit(ws=None))[0] == W
    assert status(fit(ws=P * 256 + 16))[0] == E
    with pytest.raises(_lib.LogicError):
        _lib.check(fit(d=0))


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the error without a device")
def test_cuda_error_without_device():
    assert fit() == _lib.B2D_ERR_CUDA
    assert fit(bins=1, mbf=3) == _lib.B2D_ERR_CUDA
    assert fit(seeds=P, ns=10, it=None) == _lib.B2D_ERR_CUDA


def test_shim_compiles(tmp_path):
    import os

    import cpp_build
    for mock in (False, True):
        exe = str(tmp_path / ("mean_shift_shim_mockraft" if mock else "mean_shift_shim"))
        assert os.path.exists(cpp_build.build("mean_shift_shim_test.cu", exe, mock))
