"""GPU tier: masked_l2_nn (the fused L2 1-NN under a row x group adjacency mask) through the Python wrapper against the
fp64 reference, and its relation to fused_l2_nn.  The per-row bound is the one of test_masked_nn_paths_gpu.py."""
import numpy as np
import pytest
import torch

import oracle
from masked_nn_ref import FLT_MAX, NO_CANDIDATE, masked_l2_nn as ref_masked_l2_nn
from raft_b200 import LogicError, _lib
from raft_b200.distance import fused_l2_nn, masked_l2_nn
from test_masked_nn_paths_gpu import assert_sqrt_law, check

pytestmark = pytest.mark.gpu


def blobs(m, n, k, seed=0):
    x, _, c = oracle.make_blobs(m, k, seed=177 + seed)
    y, _, _ = oracle.make_blobs(n, k, seed=199 + seed, centers=c)
    return x, y


def groups_of(layout, n, rng):
    """group_idxs (ends of the groups) for a layout of the rows of y."""
    if layout == "tiny":            # 1-7 rows: every tile is PARTIAL
        sizes = []
        while sum(sizes) < n:
            sizes.append(int(rng.integers(1, 8)))
    elif layout == "aligned":       # 256 rows: groups follow the y blocks
        sizes = [256] * ((n + 255) // 256)
    elif layout == "misaligned":    # >= 256 rows straddling the 128-row halves, with empty groups in between
        sizes = []
        while sum(sizes) < n:
            sizes += [int(rng.integers(256, 700)), 0]
    else:                           # last group ends before n: the rows behind it are in no group
        sizes = [300, 0, 200, 450]
    ends = np.minimum(np.cumsum(sizes), n)
    if layout == "short":
        ends = np.minimum(ends, n - 37)
    return ends.astype(np.int32)


def adjacency(kind, m, G, rng, x_groups=None):
    if kind == "all":
        return np.ones((m, G), bool)
    if kind == "none":
        return np.zeros((m, G), bool)
    if kind == "cc":                # connect_components: every group except the row's own colour
        a = np.ones((m, G), bool)
        a[np.arange(m), x_groups] = False
        return a
    return rng.random((m, G)) < float(kind)


def run_and_check(x, y, adj, gidx, sqrt=False, **kw):
    """The Python wrapper against the fp64 masked arg-min, every row, no count allowance (`check`); with sqrt, the
    values are sqrtf of the squared call's, bit for bit."""
    xd, yd, ad, gd = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (x, y, adj, gidx))
    gi, gv = masked_l2_nn(xd, yd, ad, gd, **kw)
    gi, gv = gi.cpu().numpy(), gv.cpu().numpy()
    check(x, y, adj, gidx, gi, gv)
    if sqrt:
        si, sv = masked_l2_nn(xd, yd, ad, gd, sqrt=True, **kw)
        assert_sqrt_law(gi, gv, si.cpu().numpy(), sv.cpu().numpy())
    return gi, gv


@pytest.mark.parametrize("k", [2, 32, 96, 128, 200, 320])
@pytest.mark.parametrize("layout", ["tiny", "aligned", "misaligned", "short"])
@pytest.mark.parametrize("kind", ["all", "none", "0.1", "0.5", "cc"])
@pytest.mark.parametrize("n", [1000, 800])
def test_masked_l2_nn_vs_reference(k, layout, kind, n):
    rng = np.random.default_rng(k * 7 + len(layout) * 3 + len(kind) + n)
    # ragged: 3 x tiles (the last one partial); 4 y blocks, the last with both halves (n = 1000) or one (n = 800)
    m = 333
    x, y = blobs(m, n, k, seed=k)
    gidx = groups_of(layout, n, rng)
    G = len(gidx)
    x_groups = rng.integers(0, G, size=m)
    run_and_check(x, y, adjacency(kind, m, G, rng, x_groups), gidx)


@pytest.mark.parametrize("k", [64, 200])
def test_all_true_is_bit_identical_to_exact_fused_l2_nn(k):
    x, y = blobs(2000, 20000, k, seed=3)
    gidx = np.arange(1000, 20001, 1000, dtype=np.int32)      # 20 groups, every one adjacent: every tile is ALL
    adj = torch.ones((2000, len(gidx)), dtype=torch.bool, device="cuda")
    L = _lib.lib()
    _lib.check(L.b2d_set_option(b"nn_screen", 0.0))
    try:
        xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
        fi, fv = fused_l2_nn(xd, yd, sqrt=False)
        mi, mv = masked_l2_nn(xd, yd, adj, torch.from_numpy(gidx).cuda())
    finally:
        _lib.check(L.b2d_set_option(b"nn_screen", 1.0))
    assert torch.equal(fi, mi)
    assert torch.equal(fv.view(torch.int32), mv.view(torch.int32))


def _abi_call(x, y, adj, gidx, out, init_out):
    """b2d_masked_l2_nn straight through the C ABI (init_out = 0 reduces into out)."""
    L = _lib.lib()
    m, k = x.shape
    n, G = y.shape[0], adj.shape[1]
    ws = torch.empty(L.b2d_masked_l2_nn_workspace_bytes(m, n, k, G), dtype=torch.uint8, device="cuda")
    _lib.check(L.b2d_masked_l2_nn(None, out.data_ptr(), x.data_ptr(), k, y.data_ptr(), k, None, None, adj.data_ptr(),
                                  adj.stride(0), gidx.data_ptr(), G, m, n, k, 0, init_out, ws.data_ptr(), ws.numel()))
    torch.cuda.synchronize()


def test_all_false_gives_no_candidate_and_keeps_callers_values():
    x, y = blobs(300, 700, 32)
    xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    gidx = torch.tensor([100, 400, 700], dtype=torch.int32, device="cuda")
    adj = torch.zeros((300, 3), dtype=torch.uint8, device="cuda")
    gi, gv = masked_l2_nn(xd, yd, adj, gidx)
    assert (gi.cpu().numpy() == NO_CANDIDATE).all() and (gv.cpu().numpy() == np.float32(FLT_MAX)).all()
    out = torch.empty((300, 2), dtype=torch.int32, device="cuda")
    out[:, 0] = torch.arange(300, dtype=torch.int32)
    out[:, 1] = torch.full((300,), 1e30).view(torch.int32)
    keep = out.clone()
    _abi_call(xd, yd, adj, gidx, out, init_out=0)
    assert torch.equal(out, keep)
    # a live mask with init_out = 0: argmin_op of the caller's value and the masked result
    adj[:150, 1] = 1
    _abi_call(xd, yd, adj, gidx, out, init_out=0)
    ri, rv = ref_masked_l2_nn(x, y, adj.cpu().numpy(), gidx.cpu().numpy())
    got_i, got_v = out[:, 0].cpu().numpy(), out[:, 1].view(torch.float32).cpu().numpy()
    win = rv < 1e30
    assert (got_i[~win] == keep[:, 0].cpu().numpy()[~win]).all()
    assert (got_i[win] == ri[win]).all() and win[:150].all() and not win[150:].any()


def test_duplicates_and_nan_rows_do_not_leak_across_the_mask():
    x, y = blobs(256, 1024, 48, seed=5)
    gidx = np.array([256, 512, 768, 1024], dtype=np.int32)
    adj = np.zeros((256, 4), bool)
    adj[:, 2] = True                                  # only rows 512..767 of y are candidates
    y[3] = y[600]                                     # the same point in a non-adjacent (row 3) and an adjacent group
    x[:20] = y[600]
    y[100:110] = np.nan                               # NaN rows, non-adjacent
    y[900] = np.nan
    gi, gv = masked_l2_nn(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), torch.from_numpy(adj).cuda(),
                          torch.from_numpy(gidx).cuda())
    gi, gv = gi.cpu().numpy(), gv.cpu().numpy()
    assert (gi[:20] == 600).all()
    # (distance 0 in the expanded form |x|^2 + |y|^2 - 2<x,y>: zero up to the cancellation of the norms)
    assert (gv[:20] <= 1e-6 * (x[:20].astype(np.float64) ** 2).sum(1)).all()
    assert np.isfinite(gv).all() and ((gi >= 512) & (gi < 768)).all()
    check(x, y, adj, gidx, gi, gv)


def test_options_and_layouts():
    rng = np.random.default_rng(9)
    m, n, k = 500, 1500, 40
    x, y = blobs(m, n, k, seed=9)
    gidx = np.cumsum(rng.integers(1, 60, size=60)).astype(np.int32)
    gidx = np.minimum(gidx, n)
    G = len(gidx)
    adj = rng.random((m, G)) < 0.3
    xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    gd = torch.from_numpy(gidx.astype(np.int64)).cuda()            # int64 group_idxs: converted on the device
    base_i, base_v = masked_l2_nn(xd, yd, torch.from_numpy(adj).cuda(), gd)
    check(x, y, adj, gidx, base_i.cpu().numpy(), base_v.cpu().numpy())
    # precomputed norms as a Python caller computes them (fp32 sums): their rounding error widens the bound
    xn, yn = (xd * xd).sum(1), (yd * yd).sum(1)
    i2, v2 = masked_l2_nn(xd, yd, torch.from_numpy(adj).cuda(), gd, xn=xn, yn=yn)
    check(x, y, adj, gidx, i2.cpu().numpy(), v2.cpu().numpy(), xn=xn.cpu().numpy(), yn=yn.cpu().numpy())
    # uint8 and a padded pitch
    wide = torch.zeros((m, G + 13), dtype=torch.uint8, device="cuda")
    wide[:, :G] = torch.from_numpy(adj.astype(np.uint8)).cuda()
    i3, v3 = masked_l2_nn(xd, yd, wide[:, :G], gd)
    assert torch.equal(i3, base_i) and torch.equal(v3, base_v)
    # sqrt
    run_and_check(x, y, adj, gidx, sqrt=True)


@pytest.mark.parametrize("gidx", [[100, 50, 300], [100, 200, 3000], [-1, 10, 20]])
def test_invalid_group_idxs_raise(gidx):
    x, y = blobs(64, 300, 16)
    adj = torch.ones((64, 3), dtype=torch.bool, device="cuda")
    with pytest.raises(LogicError):
        masked_l2_nn(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), adj,
                     torch.tensor(gidx, dtype=torch.int32, device="cuda"))


def test_int64_group_idxs_outside_int32_raise():
    x, y = blobs(64, 300, 16)
    adj = torch.ones((64, 3), dtype=torch.bool, device="cuda")
    gidx = torch.tensor([100, 2 ** 32 + 200, 300], dtype=torch.int64, device="cuda")   # would wrap to 200
    with pytest.raises(LogicError):
        masked_l2_nn(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), adj, gidx)


@pytest.mark.parametrize("k", [64, 200])
def test_sparse_pattern_reduced_size(k):
    """Pattern (b) of scripts/masked_nn_time.py at 16384 x 16384: groups of 1024 rows, each 64-row slab of x adjacent
    to 8 random groups -- half the tiles are NONE and skipped (k = 200: the streaming variant skips per half)."""
    rng = np.random.default_rng(21)
    m = n = 16384
    x, y = blobs(m, n, k, seed=21)
    G = n // 1024
    gidx = np.arange(1024, n + 1, 1024, dtype=np.int32)
    adj = np.zeros((m, G), bool)
    for s in range(m // 64):
        adj[64 * s:64 * s + 64, rng.choice(G, 8, replace=False)] = True
    run_and_check(x, y, adj, gidx)


@pytest.mark.parametrize("k", [64, 200])
def test_none_runs_for_one_slab_followed_by_live_tiles(k):
    """Long runs of tiles that are NONE for one consumer warpgroup and live for the other, followed by a tile live for
    both inside the same work item: the even 64-row slab of x tile t (warpgroup 0) is adjacent to group 0 only unless
    t % 4 == 3, the odd slab (warpgroup 1) to every group.  With groups of 1024 rows, in every y block outside group 0
    warpgroup 0 skips three tiles (resident k = 64: 6 stages, more than the ring's 5) or, streaming (k = 200), halves of
    7 stages each, then multiplies again."""
    m = n = 16384
    x, y = blobs(m, n, k, seed=31)
    G = n // 1024
    gidx = np.arange(1024, n + 1, 1024, dtype=np.int32)
    adj = np.ones((m, G), bool)
    for t in range(m // 128):
        if t % 4 != 3:
            adj[128 * t:128 * t + 64, 1:] = False
    run_and_check(x, y, adj, gidx)


def test_cpp_shim_on_gpu(tmp_path):
    """raft::distance::masked_l2_nn with MinAndDistanceReduceOp (KVP out), MinReduceOp (float out, sqrt) and
    initOutBuffer = false, against a host brute force (tests/cpp/masked_nn_test.cu)."""
    import subprocess
    import cpp_build
    exe = cpp_build.build("masked_nn_test.cu", str(tmp_path / "masked_nn_test"))
    res = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert res.returncode == 0 and "PASS" in res.stdout, res.stdout + res.stderr
