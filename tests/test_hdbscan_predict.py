"""HDBSCAN's approximate_predict without a GPU: the oracle (tests/hdbscan_predict_ref.py) against the fit's oracle and on
hand-built cases, the host tree export (raft_b200/csrc/hdbscan_tree.cuh, compiled on its own) against the oracle, the
ABI declarations, every argument check of b2d_hdbscan_rbc_fit_model and b2d_hdbscan_rbc_approximate_predict with its
status and message, B2D_ERR_CUDA without a device, the recorded model-size contract
(tests/golden/hdbscan_predict_model_contract.json) and the Python argument errors and signatures.  The GPU tier is in
tests/test_hdbscan_predict_gpu.py."""
import inspect
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import cpp_build
import hdbscan_predict_ref as R
import hdbscan_ref as H
from raft_b200 import _lib
from test_hdbscan_rbc import SELECTIONS, FakeCuda, data, fit
from test_workspace_contract import SIZE_MAX, load, replay_bytes, replay_errors

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 1 << 12
E, U, W = _lib.B2D_ERR_INVALID_ARG, _lib.B2D_ERR_UNSUPPORTED, _lib.B2D_ERR_WORKSPACE
L2, L2SQRT = 4, 5
NEW = ["b2d_hdbscan_rbc_model_bytes", "b2d_hdbscan_rbc_fit_model", "b2d_hdbscan_rbc_approximate_predict"]


def L():
    return _lib.lib()


# ------------------------------------------------------------------------------------------------------------------
# the oracle


@pytest.mark.parametrize("kind,m,d,seed", [("uniform", 150, 2, 1), ("blobs", 240, 2, 2), ("blobs", 200, 3, 3),
                                           ("duplicates", 120, 2, 7), ("uniform", 7, 3, 4), ("uniform", 1, 2, 5)])
@pytest.mark.parametrize("mcs,ms", [(5, 1), (5, 4), (12, 2), (40, 7)])
def test_oracle_fit_labels_equal_tree_labels(kind, m, d, seed, mcs, ms):
    """the restated selection and label rule give hdbscan_ref.tree_labels' labels and probabilities on every case"""
    x = data(kind, m, d, seed)
    ms = min(ms, m)
    for metric in ("euclidean", "sqeuclidean"):
        src, dst, w, _ = H.mr_tree(x, ms, metric)
        for method, single, eps in SELECTIONS + [("eom", True, 1e30), ("leaf", True, 1e-30)]:
            e = R.export(src, dst, w, m, mcs, method, single, eps)
            lab, prob, _ = H.tree_labels(src, dst, w, m, mcs, method, single, eps)
            assert (e["labels"] == lab).all(), (metric, method, single, eps)
            assert e["prob"].tobytes() == prob.tobytes(), (metric, method, single, eps)


@pytest.mark.parametrize("kind,m,d,seed", [("uniform", 150, 2, 11), ("blobs", 240, 2, 12), ("blobs", 200, 3, 13)])
@pytest.mark.parametrize("mcs,ms", [(5, 1), (5, 4), (12, 2), (40, 7)])
def test_oracle_identity_property(kind, m, d, seed, mcs, ms):
    """without duplicate rows, predicting the fitted rows gives the fit's labels and probabilities and the rows
    themselves as neighbours at their core distance"""
    x = data(kind, m, d, seed)
    assert len(np.unique(x, axis=0)) == m
    for metric in ("euclidean", "sqeuclidean"):
        for method, single, eps in SELECTIONS:
            model = R.fit(x, mcs, ms, method, single, eps if metric == "euclidean" else eps * eps, metric)
            lab, prob, nn, ww = R.predict(model, x)
            assert (nn == np.arange(m)).all()
            core = model["core"] if metric == "sqeuclidean" else np.sqrt(model["core"], dtype=np.float32)
            assert ww.tobytes() == core.tobytes()
            assert (lab == model["labels"]).all(), (metric, method, single, eps)
            assert prob.tobytes() == model["prob"].astype(np.float32).tobytes(), (metric, method, single, eps)


def two_blobs():
    """two 11 x 11 lattices of spacing 1/8 centred at (-10, 0) and (10, 0): every interior row has the same core distance
    and leaves its blob at the blob's largest lambda"""
    g = np.stack(np.meshgrid(np.arange(-5, 6), np.arange(-5, 6), indexing="ij"), -1).reshape(-1, 2) * 0.125
    return np.concatenate([g + [-10, 0], g + [10, 0]]).astype(np.float32)


def test_oracle_hand_built_cases():
    """two far blobs: a query at each blob's centre takes that blob's label with probability 1; a query far from both
    is placed at the root (noise); a non-finite query is noise with no neighbour"""
    x = two_blobs()
    model = R.fit(x, 20, 5, metric="euclidean")
    assert set(model["labels"].tolist()) == {0, 1}
    q = np.array([[-10, 0], [10, 0], [0, 500], [np.nan, 0], [np.inf, 1]], np.float32)
    lab, prob, nn, ww = R.predict(model, q)
    assert lab.tolist() == [0, 1, -1, -1, -1]
    assert prob.tolist() == [1.0, 1.0, 0.0, 0.0, 0.0]
    assert nn[3] == nn[4] == -1 and np.isinf(ww[3:]).all()
    assert nn[0] < 121 <= nn[1]
    # the far point leaves the tree at lambda 1 / W, below every cluster's birth, so it climbs to the root
    assert 1.0 / float(ww[2]) < model["birth"][1:].min()
    # allow_single_cluster: one blob and one far point, a query near the blob takes the root's label
    x1 = np.concatenate([x[:121], [[300, 300]]]).astype(np.float32)
    m1 = R.fit(x1, 20, 5, "eom", True, 0.0, "euclidean")
    assert m1["single_root"] and m1["labels"][:121].max() == 0 and m1["labels"][121] == -1
    lab1, _, _, _ = R.predict(m1, np.array([[-10, 0], [300, 300]], np.float32))
    assert lab1.tolist() == [0, -1]


def test_oracle_order_breaks_ties_on_w_by_s():
    """rows 1 to 4 all weigh the query's core distance (its s to row 0): the neighbour is the nearest of them (row 4),
    not the smallest row"""
    x = np.array([[0, 0], [1, 0], [2, 0], [3, 0], [4, 0], [5, 0]], np.float32)
    model = R.fit(x, 2, 6, metric="sqeuclidean")
    j, W = R.neighbour(model, np.array([4.1, 0], np.float32))
    assert j == 4 and W == np.float32(4.1) * np.float32(4.1)


# ------------------------------------------------------------------------------------------------------------------
# the host tree export


@pytest.fixture(scope="module")
def export_exe(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("hdbscan_tree_export"))
    return cpp_build.build("hdbscan_tree_export_test.cu", os.path.join(d, "hdbscan_tree_export_test"),
                           standalone=True), d


def host_export(export_exe, cases):
    exe, d = export_exe
    inp, out = os.path.join(d, "in.bin"), os.path.join(d, "out.bin")
    with open(inp, "wb") as f:
        for src, dst, w, m, mcs, method, single, eps in cases:
            f.write(np.array([m, mcs, method == "leaf", single], np.int64).tobytes() + np.float64(eps).tobytes())
            f.write(np.asarray(src, np.int32).tobytes() + np.asarray(dst, np.int32).tobytes() +
                    np.asarray(w, np.float32).tobytes())
    res = subprocess.run([exe, inp, out], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0 and "PASS" in res.stdout, res.stdout + res.stderr
    raw, at, got = np.fromfile(out, np.uint8), 0, []

    def take(n, dt):
        nonlocal at
        v = raw[at:at + n * np.dtype(dt).itemsize].view(dt)
        at += n * np.dtype(dt).itemsize
        return v

    for c in cases:
        m = c[3]
        g = dict(n=int(take(1, np.int32)[0]), labels=take(m, np.int32), prob=take(m, np.float32))
        nc = int(take(1, np.int32)[0])
        g.update(single_root=bool(take(1, np.int32)[0]), thr=float(take(1, np.float64)[0]),
                 row_parent=take(m, np.int32), row_lambda=take(m, np.float64), parent=take(nc, np.int32),
                 owner=take(nc, np.int32), label=take(nc, np.int32), birth=take(nc, np.float64),
                 death=take(nc, np.float64))
        got.append(g)
    assert at == len(raw)
    return got


@pytest.mark.parametrize("kind,m,d", [("uniform", 300, 2), ("blobs", 500, 3), ("duplicates", 240, 2),
                                      ("uniform", 7, 2), ("uniform", 2, 2), ("uniform", 1, 3), ("blobs", 2000, 2)])
def test_host_tree_export_equals_oracle(export_exe, kind, m, d):
    """every exported array exactly, the labels unchanged by asking for the export"""
    x = data(kind, m, d, 200 + m)
    cases = []
    for ms in sorted({1, min(m, 4), min(m, 11)}):
        for metric in ("euclidean", "sqeuclidean"):
            src, dst, w, _ = H.mr_tree(x, ms, metric)
            for mcs in (2, 5, 30, max(2, m + 1)):
                for method, single, eps in SELECTIONS + [("eom", True, 1e30), ("leaf", False, 1e-30)]:
                    cases.append((src, dst, w, m, mcs, method, single, eps))
    for g, c in zip(host_export(export_exe, cases), cases):
        e = R.export(*c)
        assert g["labels"].tobytes() == e["labels"].tobytes(), c[3:]
        assert g["prob"].tobytes() == e["prob"].astype(np.float32).tobytes(), c[3:]
        for k in ("row_parent", "parent", "owner", "label"):
            assert (g[k] == e[k]).all(), (k, c[3:])
        for k in ("row_lambda", "birth", "death"):
            assert g[k].tobytes() == np.asarray(e[k], np.float64).tobytes(), (k, c[3:])
        assert g["single_root"] == e["single_root"] and g["thr"] == e["thr"], c[3:]


# ------------------------------------------------------------------------------------------------------------------
# the C ABI


def test_abi_declarations():
    hdr = open(os.path.join(ROOT, "include", "raft_b200.h")).read()
    for s in NEW:
        assert re.search(r"\b%s\(" % s, hdr), s
        assert s in _lib.SYMBOLS
        assert hasattr(L(), s)


def test_model_bytes_query():
    q = L().b2d_hdbscan_rbc_model_bytes
    for args in ((0, 2, 0), (-1, 2, 0), (2 ** 30, 2, 0), (10, 1, 0), (10, 4, 0), (10, 2, -1), (10, 2, 11)):
        assert q(*args) == SIZE_MAX, args
    for m, d in ((1, 2), (1000, 3), (10 ** 6, 2)):
        nl = int(np.ceil(np.sqrt(m)))
        index = L().b2d_ball_cover_index_bytes(m, d, 0)
        assert index + 48 * m + 4 * nl <= q(m, d, 0) <= index + 48 * m + 4 * nl + 12 * 256
        assert q(m, d, nl) == q(m, d, 0)


def test_model_contract_bytes():
    c = load("hdbscan_predict_model_contract.json")
    for m, d, nl, want in replay_bytes(c, "b2d_hdbscan_rbc_model_bytes"):
        assert (want == SIZE_MAX) == (not (1 <= m < 2 ** 30 and d in (2, 3) and 0 <= nl <= m)), (m, d, nl)


def test_model_contract_errors():
    assert replay_errors(load("hdbscan_predict_model_contract.json")) == 2 * 2 * 2 * 5


def fit_model(model=P * 256, **kw):
    a = dict(metric=L2SQRT, x=P, ldx=2, m=100, d=2, ms=5, mcs=10, eps=0.0, method=0, single=0, nl=0, seed=1, lab=P,
             prob=P, src=P, dst=P, w=P, nc=P, ws=P * 256, wsb=1 << 40)
    a.update(kw)
    return L().b2d_hdbscan_rbc_fit_model(None, a["metric"], a["x"], a["ldx"], a["m"], a["d"], a["ms"], a["mcs"],
                                         a["eps"], a["method"], a["single"], a["nl"], a["seed"], a["lab"], a["prob"],
                                         a["src"], a["dst"], a["w"], a["nc"], a["ws"], a["wsb"], model)


def test_fit_model_argument_errors_are_the_fits():
    """every argument error of the fit, with the fit's status and message, then the model's own two"""
    from test_hdbscan_rbc import test_invalid_arguments
    cases = list(test_invalid_arguments.pytestmark[0].args[1])
    assert len(cases) == 28
    for kw, rc, msg in cases:
        assert fit(**kw) == rc, kw
        want = L().b2d_last_error().decode()
        assert fit_model(**kw) == rc, kw
        assert L().b2d_last_error().decode() == want and want.startswith(msg), kw
    assert fit_model(model=None) == E and L().b2d_last_error().decode() == "null model"
    assert fit_model(model=P * 256 + 64) == E and L().b2d_last_error().decode() == "model must be 256-byte aligned"


def predict(model=P * 256, m=100, d=2, metric=L2SQRT, nl=0, ms=5, q=P, ldq=2, mq=10, lab=P, prob=P, nn=P, w=P):
    return L().b2d_hdbscan_rbc_approximate_predict(None, model, m, d, metric, nl, ms, q, ldq, mq, lab, prob, nn, w)


MS = "min_samples must be in [1, min(64, m)], got "


@pytest.mark.parametrize("kw,rc,msg", [
    (dict(metric=0), U, "hdbscan approximate_predict supports the L2Unexpanded and L2SqrtUnexpanded metrics, got metric 0"),
    (dict(metric=1), U, "hdbscan approximate_predict supports the L2Unexpanded and L2SqrtUnexpanded metrics, got metric 1"),
    (dict(d=4, ldq=4), U, "hdbscan approximate_predict supports d = 2 and d = 3, got d = 4"),
    (dict(d=1, ldq=1), U, "hdbscan approximate_predict supports d = 2 and d = 3, got d = 1"),
    (dict(m=0), E, "m must be in [1, 2^30)"),
    (dict(m=2 ** 30), E, "m must be in [1, 2^30)"),
    (dict(nl=-1), E, "n_landmarks must be in [0, m] (0: ceil(sqrt(m)))"),
    (dict(nl=101), E, "n_landmarks must be in [0, m] (0: ceil(sqrt(m)))"),
    (dict(ms=0), E, MS + "0"),
    (dict(ms=65), E, MS + "65"),
    (dict(m=3, ms=4), E, MS + "4"),
    (dict(model=None), E, "null model"),
    (dict(model=P * 256 + 8), E, "model must be 256-byte aligned"),
    (dict(mq=-1), E, "mq must be in [0, 2^31)"),
    (dict(mq=2 ** 31), E, "mq must be in [0, 2^31)"),
    (dict(q=None), E, "null queries"),
    (dict(ldq=1), E, "ldq smaller than d"),
    (dict(d=3, ldq=2), E, "ldq smaller than d"),
    (dict(lab=None), E, "null labels / probabilities"),
    (dict(prob=None), E, "null labels / probabilities"),
])
def test_predict_argument_errors(kw, rc, msg):
    assert predict(**kw) == rc, kw
    assert L().b2d_last_error().decode() == msg


def test_predict_no_queries_does_nothing():
    """mq = 0 returns at once, with or without a device: null outputs and queries are fine"""
    assert predict(mq=0, q=None, lab=None, prob=None, nn=None, w=None) == _lib.B2D_OK


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the error without a device")
def test_cuda_error_without_device():
    assert fit_model() == _lib.B2D_ERR_CUDA
    assert fit_model(m=1, ms=1, src=None, dst=None, w=None) == _lib.B2D_ERR_CUDA
    assert predict() == _lib.B2D_ERR_CUDA
    assert predict(d=3, ldq=7, metric=L2, nn=None, w=None) == _lib.B2D_ERR_CUDA


# ------------------------------------------------------------------------------------------------------------------
# Python


class FakeModel:
    pass


def fake_model(d=2):
    from raft_b200.cluster import HdbscanModel
    return HdbscanModel(None, FakeCuda((16,)), 100, d, L2SQRT, 0, 5)


@pytest.mark.parametrize("kw,exc,msg", [
    (dict(model=FakeModel()), TypeError, "model must be an HdbscanModel (from hdbscan_model), got FakeModel"),
    (dict(shape=(10, 3)), ValueError, "points have 3 columns, the model 2"),
    (dict(strides=(16, 8)), ValueError, "points must have contiguous rows"),
    (dict(shape=(10,)), ValueError, ""),
])
def test_python_predict_argument_errors(kw, exc, msg):
    from raft_b200.cluster import approximate_predict
    kw = dict(kw)
    model = kw.pop("model", None) or fake_model()
    q = FakeCuda(kw.pop("shape", (10, 2)), strides=kw.pop("strides", None))
    with pytest.raises(exc, match=re.escape(msg)):
        approximate_predict(model, q, handle=object())


def test_python_model_argument_errors_are_hdbscans():
    """hdbscan_model checks its arguments as hdbscan does, with the same messages"""
    from raft_b200.cluster import hdbscan, hdbscan_model
    from test_hdbscan_rbc import test_python_argument_errors
    cases = list(test_python_argument_errors.pytestmark[0].args[1])
    assert len(cases) == 11
    for kw, exc, msg in cases:
        kw = dict(kw)
        shape, strides = kw.pop("shape", (10, 2)), kw.pop("strides", None)
        for f in (hdbscan, hdbscan_model):
            with pytest.raises(exc, match=re.escape(msg)):
                f(FakeCuda(shape, strides=strides), handle=object(), **kw)


def test_python_signatures():
    from raft_b200 import cluster
    from raft_b200.cluster import HdbscanPrediction, approximate_predict, hdbscan, hdbscan_model
    assert list(inspect.signature(hdbscan_model).parameters.items())[1:] == \
        list(inspect.signature(hdbscan).parameters.items())[1:]
    assert list(inspect.signature(approximate_predict).parameters) == ["model", "points", "handle"]
    assert inspect.signature(approximate_predict).parameters["handle"].default is None
    assert HdbscanPrediction._fields == ("labels", "probabilities", "neighbors", "weights")
    for name in ("HdbscanModel", "HdbscanPrediction", "approximate_predict", "hdbscan_model"):
        assert hasattr(cluster, name)
