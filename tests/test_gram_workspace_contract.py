"""CPU tier: the workspace contract of b2d_gram_matrix against tests/golden/gram_workspace_contract.json (recorded by
tests/golden/make_gram_workspace_contract.py): the byte count of b2d_gram_matrix_workspace_bytes for every kernel id and
dtype over the shape grid of the other queries, and the status and message of b2d_gram_matrix given a null, short or
misaligned workspace."""
import json
import os

import pytest

from raft_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def contract():
    with open(os.path.join(ROOT, "tests", "golden", "gram_workspace_contract.json")) as f:
        return json.load(f)


def test_gram_workspace_bytes(contract):
    L = _lib.lib()
    rows = contract["bytes"]["b2d_gram_matrix_workspace_bytes"]
    assert len(rows) == 6 * 4 * 16
    for *args, want in rows:
        assert L.b2d_gram_matrix_workspace_bytes(*args) == want, args
    # the same sizes as the pairwise query of the metric each kernel transforms
    for kr, dt, m, n, k, want in rows:
        if 0 <= kr <= 3:
            assert want == L.b2d_pairwise_workspace_bytes(0 if kr == 2 else 6, dt, m, n, k), (kr, dt, m, n, k)
        else:
            assert want == 2 ** 64 - 1


def test_gram_workspace_errors(contract):
    """The workspaces are fake addresses: replayed only without a GPU, so that a call which no longer fails in validation
    cannot hand one to a kernel."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    L = _lib.lib()
    assert len(contract["errors"]) == 13
    for e in contract["errors"]:
        rc = getattr(L, e["fn"])(*e["args"])
        assert (rc, L.b2d_last_error().decode()) == (e["rc"], e["msg"]), (e["name"], e["case"])
