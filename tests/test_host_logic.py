"""CPU tier: host-side mirror of the pylibraft conventions and the multi-GPU exchange logic
(world_size-2 gloo run of the packed min-loc all-reduce)."""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

import oracle
from raft_b200.common.cai_wrapper import cai_wrapper
from raft_b200.distance.distance_type import DISTANCE_TYPES, DistanceType, resolve_metric
from raft_b200.distance.fused_l2_nn import shard_bounds
from raft_b200.distance.pairwise_distance import _layout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class FakeCai:
    def __init__(self, arr, ptr=0x1000):
        self.__cuda_array_interface__ = {"shape": arr.shape, "typestr": arr.dtype.str, "version": 3,
                                         "data": (ptr, False),
                                         "strides": None if arr.flags.c_contiguous else arr.strides}


def test_distance_type_values_match_reference_enum():
    assert int(DistanceType.L2Expanded) == 0 and int(DistanceType.L2SqrtExpanded) == 1
    assert int(DistanceType.CosineExpanded) == 2 and int(DistanceType.L1) == 3
    assert int(DistanceType.LpUnexpanded) == 9 and int(DistanceType.CorrelationExpanded) == 10
    assert int(DistanceType.Precomputed) == 100
    assert {int(v) for v in DistanceType} == {int(v) for v in oracle.DistanceType}


def test_metric_strings():
    assert resolve_metric("euclidean") == DistanceType.L2SqrtExpanded
    assert resolve_metric("sqeuclidean") == DistanceType.L2Expanded
    assert resolve_metric("cityblock") == DistanceType.L1
    assert resolve_metric("chebyshev") == DistanceType.Linf
    assert resolve_metric("minkowski") == DistanceType.LpUnexpanded
    assert resolve_metric("L2Unexpanded") == DistanceType.L2Unexpanded
    assert resolve_metric(8) == DistanceType.Canberra
    assert resolve_metric("hamming") == DistanceType.HammingUnexpanded
    assert resolve_metric("kl_divergence") == DistanceType.KLDivergence
    with pytest.raises(ValueError):
        resolve_metric("haversine")
    assert set(DISTANCE_TYPES) >= {"l2", "l1", "cosine", "correlation", "canberra", "inner_product", "lp"}


def test_cai_wrapper_and_layout():
    a = np.zeros((5, 7), np.float32)
    w = cai_wrapper(FakeCai(a))
    assert w.shape == (5, 7) and w.c_contiguous and not w.f_contiguous and w.data == 0x1000
    assert _layout(w) == (True, 7)
    f = np.asfortranarray(a)
    wf = cai_wrapper(FakeCai(f))
    assert wf.f_contiguous and _layout(wf) == (False, 5)
    padded = np.zeros((5, 16), np.float32)[:, :7]
    assert _layout(cai_wrapper(FakeCai(padded))) == (True, 16)
    with pytest.raises(TypeError):
        cai_wrapper(FakeCai(a)).validate_shape_dtype(expected_dtype=np.float64)
    with pytest.raises(ValueError):
        cai_wrapper(FakeCai(a)).validate_shape_dtype(expected_dims=1)
    with pytest.raises(TypeError):
        cai_wrapper(a)


def test_single_row_fortran_output_pitch():
    """x [1, k] against a Fortran-order y [n, k]: the result [1, n] is written in Fortran order, whose pitch is the
    column stride of `out` -- a single contiguous row also reads as C order with a pitch of n, which would put element
    (0, j) at j * n."""
    from raft_b200.distance.pairwise_distance import _operands
    x = np.zeros((1, 16), np.float32)
    y = np.asfortranarray(np.zeros((130, 16), np.float32))
    *_, row_major, ldx, ldy, ldd = _operands(FakeCai(x), FakeCai(y), FakeCai(np.zeros((1, 130), np.float32)))
    assert (row_major, ldx, ldy, ldd) == (False, 1, 130, 1)
    padded = np.zeros((130, 4), np.float32)[:, :1].T              # [1, 130] with a column stride of 4 elements
    *_, row_major, ldx, ldy, ldd = _operands(FakeCai(x), FakeCai(y), FakeCai(padded))
    assert (row_major, ldd) == (False, 4)
    *_, row_major, ldx, ldy, ldd = _operands(FakeCai(np.zeros((3, 16), np.float32)), FakeCai(np.zeros((130, 16), np.float32)),
                                             FakeCai(np.zeros((3, 136), np.float32)[:, :130]))
    assert (row_major, ldx, ldy, ldd) == (True, 16, 16, 136)


def test_shard_bounds_cover_database_exactly():
    for n, w in ((8_000_000, 8), (1001, 4), (7, 8), (5, 1)):
        cuts = [shard_bounds(n, w, r) for r in range(w)]
        assert cuts[0][0] == 0 and cuts[-1][1] == n
        assert all(cuts[i][1] == cuts[i + 1][0] for i in range(w - 1))


WORKER = textwrap.dedent('''
    import os, sys
    sys.path.insert(0, os.environ["B2D_ROOT"])
    import numpy as np, torch, torch.distributed as dist
    import oracle
    from raft_b200.distance.fused_l2_nn import shard_bounds
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:" + os.environ["B2D_PORT"],
                            rank=int(os.environ["RANK"]), world_size=int(os.environ["WORLD_SIZE"]))
    rank, world = dist.get_rank(), dist.get_world_size()
    x, _, c = oracle.make_blobs(257, 24, seed=11)
    y, _, _ = oracle.make_blobs(1003, 24, seed=12, centers=c)
    y[500] = y[3]                      # a tie across shards: the smaller global index must win
    x[0] = y[3]
    lo, hi = shard_bounds(y.shape[0], world, rank)
    # what the GPU kernel leaves in `keys` for this shard (host model: oracle.pack_minloc)
    d = oracle.pairwise_distance(x, y[lo:hi], oracle.DistanceType.L2Expanded)
    loc = np.argmin(d, axis=1)
    v = d[np.arange(len(x)), loc].astype(np.float32)            # ||x - y||^2, as the kernel packs it
    keys = torch.from_numpy(oracle.pack_minloc(v, loc + lo))
    dist.all_reduce(keys, op=dist.ReduceOp.MIN)                 # the ONE exchange step
    val, idx = oracle.unpack_minloc(keys.numpy())
    ref_idx, ref_val = oracle.fused_l2_nn(x, y)
    assert (idx == ref_idx).all(), (rank, np.nonzero(idx != ref_idx))
    assert idx[0] == 3
    assert np.allclose(np.maximum(val.astype(np.float64), 0), ref_val, rtol=1e-4, atol=1e-3)
    # the two-exchange form of fused_l2_nn_sharded: head of every shard, all-reduce (global bounds),
    # the rest of the shard continuing from the reduced keys (init_keys = 0 == elementwise MIN), all-reduce
    head = 100
    def shard_keys(a, b):
        dd = oracle.pairwise_distance(x, y[a:b], oracle.DistanceType.L2Expanded)
        ll = np.argmin(dd, axis=1)
        return torch.from_numpy(oracle.pack_minloc(dd[np.arange(len(x)), ll].astype(np.float32), ll + a))
    k2 = shard_keys(lo, lo + head)
    dist.all_reduce(k2, op=dist.ReduceOp.MIN)
    k2 = torch.minimum(k2, shard_keys(lo + head, hi))
    dist.all_reduce(k2, op=dist.ReduceOp.MIN)
    assert torch.equal(k2, keys)
    dist.barrier(); dist.destroy_process_group()
    print("rank", rank, "ok")
''')


def test_minloc_allreduce_world2_gloo(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    port = str(29000 + os.getpid() % 2000)
    procs = []
    for r in range(2):
        env = dict(os.environ, RANK=str(r), WORLD_SIZE="2", B2D_ROOT=ROOT, B2D_PORT=port)
        procs.append(subprocess.Popen([sys.executable, str(script)], env=env, stdout=subprocess.PIPE,
                                      stderr=subprocess.STDOUT, text=True))
    for p in procs:
        out, _ = p.communicate(timeout=240)
        assert p.returncode == 0, out
        assert "ok" in out


def test_pylibraft_alias_namespace():
    """`from pylibraft.distance import pairwise_distance` keeps working (drop-in alias package)."""
    import pylibraft.common
    import pylibraft.config
    import pylibraft.distance as d
    import raft_b200.distance as r
    assert d.pairwise_distance is r.pairwise_distance and d.fused_l2_nn_argmin is r.fused_l2_nn_argmin
    assert "euclidean" in d.DISTANCE_TYPES and callable(pylibraft.config.set_output_as)
    assert pylibraft.common.DeviceResources is not None


def test_exchange_plan_is_rank_invariant_and_covers_every_shard():
    """ADVICE r1 (medium): ranks whose shards differ by one row must issue the SAME number of all_reduces.  The
    plan depends on (n_total // world, world) only; a rank's last sub-chunk takes what its shard has left."""
    from raft_b200.distance import shard_bounds
    from raft_b200.distance.fused_l2_nn import SHARD_HEAD_ROWS, plan_exchanges
    for n_total, world in [(8_000_000, 8), (8_000_001, 8), (1_048_577, 8), (4 * SHARD_HEAD_ROWS * 8 + 3, 8),
                           (4 * SHARD_HEAD_ROWS * 2 - 1, 2), (1000, 4), (5, 8), (8_000_000, 2), (8_000_000, 1)]:
        plan = plan_exchanges(n_total // world, world)
        assert all(p >= 0 for p in plan) and sum(plan) == n_total // world
        assert len(plan) <= 4
        for r in range(world):
            lo, hi = shard_bounds(n_total, world, r)
            n_local, done = hi - lo, 0
            for c, rows in enumerate(plan):          # the loop of fused_l2_nn_sharded
                rows = n_local - done if c == len(plan) - 1 else max(0, min(rows, n_local - done))
                assert rows >= 0
                done += rows
            assert done == n_local
    assert plan_exchanges(1_000_000, 8)[0] == SHARD_HEAD_ROWS and len(plan_exchanges(1_000_000, 8)) >= 2


def pairwise_plan(metric, dtype, m, n, k, x=0x1000, y=0x2000, dist=0x3000, ldx=None, ldy=None, ldd=None, row_major=True):
    """b2d_debug_pairwise_plan as a dict; launches are (k-blocks, acc_mode, 'res' | 'str')."""
    import ctypes
    from raft_b200 import _lib
    ldx = ldx or (k if row_major else m)
    ldy = ldy or (k if row_major else n)
    ldd = ldd or (n if row_major else m)
    out = (ctypes.c_int * 70)()
    rc = _lib.lib().b2d_debug_pairwise_plan(int(metric), dtype, x, ldx, y, ldy, dist, ldd, m, n, k, int(row_major), out, 70)
    if rc:
        return rc
    path = ["none", "tensor", "simt", "simt-tma", "f64"][out[0]]
    store = "tma" if out[1] else "vec2" if out[2] else "scalar"
    launches = [(out[7 + 4 * i], out[8 + 4 * i], "res" if out[9 + 4 * i] else "str") for i in range(min(out[5], 16))]
    assert [out[6 + 4 * i] for i in range(len(launches))] == [sum(l[0] for l in launches[:i]) for i in range(len(launches))]
    return {"path": path, "store": store if path == "tensor" else None, "vec": (out[3], out[4]), "launches": launches}


def test_pairwise_plan_boundaries():
    """The dispatch decisions of b2d_pairwise_distance, without a device: resident | streaming at k = 128 | 129, one
    pass | K chunks at 320 | 321, the remainder chunk's kernel at 384 | 385 and 512 | 513, TMA | register stores by
    n % 4, ldd % 4 and the base address, 16-byte operand loads of the unexpanded kernels."""
    from raft_b200 import _lib
    DT = oracle.DistanceType
    F32, F16, F64 = _lib.B2D_F32, _lib.B2D_F16, _lib.B2D_F64
    for dt in (F32, F16):
        plan = lambda k, **kw: pairwise_plan(DT.L2Expanded, dt, 300, 256, k, **kw)
        assert plan(128) == {"path": "tensor", "store": "tma", "vec": (0, 0), "launches": [(4, 0, "res")]}
        assert plan(129)["launches"] == [(5, 0, "str")]
        assert plan(320)["launches"] == [(10, 0, "str")] and plan(320)["store"] == "tma"
        assert plan(321)["launches"] == [(8, 1, "str"), (3, 3, "res")] and plan(321)["store"] == "vec2"
        assert plan(384)["launches"] == [(8, 1, "str"), (4, 3, "res")]
        assert plan(385)["launches"] == [(8, 1, "str"), (5, 3, "str")]
        assert plan(512)["launches"] == [(8, 1, "str"), (8, 3, "str")]
        assert plan(513)["launches"] == [(8, 1, "str"), (8, 2, "str"), (1, 3, "res")]
        # the output's alignment decides how the tiles are stored
        assert plan(64, dist=0x3004)["store"] == "scalar" and plan(64, dist=0x3008)["store"] == "vec2"
        assert plan(64, ldd=257)["store"] == "scalar" and plan(64, ldd=258)["store"] == "vec2"
        assert plan(64, ldd=260)["store"] == "tma"
        assert plan(400, ldd=257)["store"] == "scalar" and plan(400, dist=0x3004)["store"] == "scalar"
        assert pairwise_plan(DT.L2Expanded, dt, 300, 254, 64, ldd=256)["store"] == "vec2"
        assert pairwise_plan(DT.L2Expanded, dt, 300, 252, 64)["store"] == "tma"
        # Fortran order: dist is written as [n][m], so m takes the part of n
        assert pairwise_plan(DT.L2Expanded, dt, 254, 300, 64, row_major=False)["store"] == "vec2"
        assert pairwise_plan(DT.L2Expanded, dt, 256, 301, 64, row_major=False)["store"] == "tma"
        # the ratio metrics run one pass at every k
        for metric in (DT.JaccardExpanded, DT.DiceExpanded):
            assert pairwise_plan(metric, dt, 300, 256, 1024)["launches"] == [(32, 0, "str")]
        assert len(pairwise_plan(DT.InnerProduct, dt, 300, 256, 1024)["launches"]) == 4
    # unexpanded kernels: fp32 only, each operand vectorised on its own
    ux = lambda k, **kw: pairwise_plan(DT.L1, F32, 200, 100, k, **kw)
    assert ux(32) == {"path": "simt-tma", "store": None, "vec": (1, 1), "launches": [(0, 0, "str")]}
    assert ux(32, x=0x1004)["vec"] == (0, 1) and ux(32, y=0x2004)["vec"] == (1, 0) and ux(32, y=0x2004)["path"] == "simt"
    assert ux(32, ldx=33)["vec"] == (0, 1) and ux(32, ldy=34)["vec"] == (1, 0) and ux(32, ldx=36, ldy=40)["vec"] == (1, 1)
    assert ux(31)["vec"] == (0, 0) and ux(4)["vec"] == (1, 1) and ux(5)["vec"] == (0, 0)
    assert ux(32, row_major=False)["vec"] == (0, 0)
    assert pairwise_plan(DT.L1, F64, 200, 100, 32)["path"] == "f64"
    assert pairwise_plan(DT.L2Expanded, F64, 200, 100, 32)["path"] == "f64"
    assert pairwise_plan(DT.L1, F32, 0, 100, 32)["path"] == "none"
    # refusals are those of b2d_pairwise_distance
    for metric in oracle.UNEXPANDED:
        assert pairwise_plan(metric, F16, 200, 100, 32) == _lib.B2D_ERR_UNSUPPORTED
        assert _lib.lib().b2d_pairwise_workspace_bytes(int(metric), F16, 200, 100, 32) == 2 ** 64 - 1
    assert pairwise_plan(13, F32, 200, 100, 32) == _lib.B2D_ERR_UNSUPPORTED
    assert pairwise_plan(DT.L1, F32, 200, 100, 32, ldx=31) == _lib.B2D_ERR_INVALID_ARG
