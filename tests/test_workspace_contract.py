"""CPU tier: the workspace contract of the C ABI against the fixtures under tests/golden (all recorded by
tests/golden/make_workspace_contract.py): the byte count of every *_workspace_bytes query over a grid that reaches every
branch of the layouts, and the status and message of every entry point given a null, short or misaligned workspace.
workspace_contract.json covers distances, nearest neighbours, select_k and the stats; the k-means, gram_matrix,
single-linkage and DBSCAN entry points have a fixture each."""
import json
import os

import pytest

from raft_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZE_MAX = 2 ** 64 - 1


def load(name):
    with open(os.path.join(ROOT, "tests", "golden", name)) as f:
        return json.load(f)


def replay_bytes(contract, fn):
    """Checks every recorded size of fn and returns the rows."""
    L = _lib.lib()
    rows = contract["bytes"][fn]
    for *args, want in rows:
        assert getattr(L, fn)(*args) == want, (fn, args)
    return rows


def replay_errors(contract):
    """The workspaces are fake addresses: replayed only without a GPU, so that a call which no longer fails in validation
    cannot hand one to a kernel.  Returns the number of cases."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    L = _lib.lib()
    for e in contract["errors"]:
        rc = getattr(L, e["fn"])(*e["args"])
        assert (rc, L.b2d_last_error().decode()) == (e["rc"], e["msg"]), (e["name"], e["case"])
    return len(contract["errors"])


def test_workspace_bytes():
    contract = load("workspace_contract.json")
    for fn in contract["bytes"]:
        replay_bytes(contract, fn)


def test_workspace_errors():
    replay_errors(load("workspace_contract.json"))


def test_kmeans_workspace_bytes():
    rows = replay_bytes(load("kmeans_workspace_contract.json"), "b2d_kmeans_workspace_bytes")
    assert len(rows) == 6 * 8 * 4 + 2 + 3
    for *args, want in rows:
        if min(args) < 0:
            assert want == SIZE_MAX, args


def test_kmeans_workspace_errors():
    assert replay_errors(load("kmeans_workspace_contract.json")) == 15


def test_gram_workspace_bytes():
    L = _lib.lib()
    rows = replay_bytes(load("gram_workspace_contract.json"), "b2d_gram_matrix_workspace_bytes")
    assert len(rows) == 6 * 4 * 16
    # the same sizes as the pairwise query of the metric each kernel transforms
    for kr, dt, m, n, k, want in rows:
        if 0 <= kr <= 3:
            assert want == L.b2d_pairwise_workspace_bytes(0 if kr == 2 else 6, dt, m, n, k), (kr, dt, m, n, k)
        else:
            assert want == SIZE_MAX


def test_gram_workspace_errors():
    assert replay_errors(load("gram_workspace_contract.json")) == 13


def test_single_linkage_workspace_bytes():
    rows = replay_bytes(load("single_linkage_workspace_contract.json"), "b2d_single_linkage_workspace_bytes")
    assert len(rows) == 8 * 8 * 5 + 3
    for *args, want in rows:
        if min(args[:2]) < 0:
            assert want == SIZE_MAX, args


def test_mst_workspace_bytes():
    rows = replay_bytes(load("single_linkage_workspace_contract.json"), "b2d_mst_workspace_bytes")
    assert len(rows) == 4 * 3 + 2


def test_single_linkage_workspace_errors():
    assert replay_errors(load("single_linkage_workspace_contract.json")) == 9


def test_dbscan_workspace_bytes():
    rows = replay_bytes(load("dbscan_workspace_contract.json"), "b2d_dbscan_workspace_bytes")
    for *args, want in rows:
        if min(args) < 0:
            assert want == SIZE_MAX, args


def test_dbscan_workspace_errors():
    assert replay_errors(load("dbscan_workspace_contract.json")) == 9
