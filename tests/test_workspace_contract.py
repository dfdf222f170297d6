"""CPU tier: the workspace contract of the C ABI against tests/golden/workspace_contract.json (recorded by
tests/golden/make_workspace_contract.py): the byte count of every *_workspace_bytes query over a grid that reaches every
branch of the layouts, and the status and message of every entry point given a null, short or misaligned workspace."""
import json
import os

import pytest

from raft_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def contract():
    with open(os.path.join(ROOT, "tests", "golden", "workspace_contract.json")) as f:
        return json.load(f)


def test_workspace_bytes(contract):
    L = _lib.lib()
    for fn, rows in contract["bytes"].items():
        for *args, want in rows:
            assert getattr(L, fn)(*args) == want, (fn, args)


def test_workspace_errors(contract):
    """The workspaces are fake addresses: replayed only without a GPU, so that a call which no longer fails in validation
    cannot hand one to a kernel."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    L = _lib.lib()
    for e in contract["errors"]:
        rc = getattr(L, e["fn"])(*e["args"])
        assert (rc, L.b2d_last_error().decode()) == (e["rc"], e["msg"]), (e["name"], e["case"])
