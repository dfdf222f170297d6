"""CPU tier: the workspace contract of the k-means entry points against tests/golden/kmeans_workspace_contract.json
(recorded by tests/golden/make_kmeans_workspace_contract.py): the byte count of b2d_kmeans_workspace_bytes over a shape
grid, and the status and message of every k-means entry point given a null, short or misaligned workspace."""
import json
import os

import pytest

from raft_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def contract():
    with open(os.path.join(ROOT, "tests", "golden", "kmeans_workspace_contract.json")) as f:
        return json.load(f)


def test_kmeans_workspace_bytes(contract):
    L = _lib.lib()
    rows = contract["bytes"]["b2d_kmeans_workspace_bytes"]
    assert len(rows) == 6 * 8 * 4 + 2 + 3
    for *args, want in rows:
        assert L.b2d_kmeans_workspace_bytes(*args) == want, args
        if min(args) < 0:
            assert want == 2 ** 64 - 1


def test_kmeans_workspace_errors(contract):
    """The workspaces are fake addresses: replayed only without a GPU, so that a call which no longer fails in validation
    cannot hand one to a kernel."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    L = _lib.lib()
    assert len(contract["errors"]) == 15
    for e in contract["errors"]:
        rc = getattr(L, e["fn"])(*e["args"])
        assert (rc, L.b2d_last_error().decode()) == (e["rc"], e["msg"]), (e["name"], e["case"])
