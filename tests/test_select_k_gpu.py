"""select_k on the GPU, compared exactly with oracle/select_k.py: values bit-equal, indices equal, no tolerance."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

import oracle
from oracle.select_k import select_k as ref_select_k
from raft_b200 import LogicError, _lib
from raft_b200.distance import DistanceType, pairwise_distance
from raft_b200.matrix import select_k
from raft_b200.neighbors import brute_force

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"

# cpp/tests/matrix/select_k.cu:9-60 of the reference (rows, len, k), the 1 x 10^9 rows replaced by 1 x 2^27
REFERENCE_SHAPES = (
    [(1, 130, 15), (1, 128, 15)] + [(20, 700, k) for k in (1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 16)]
    + [(100, 1700, k) for k in (17, 31, 32, 33, 63, 64, 65, 255, 256, 511, 512, 1023, 1024, 1700)]
    + [(100, 100000, k) for k in (1, 2, 3, 7, 16, 31, 32, 60, 100, 200, 1000, 2000, 100000, 2048, 1237)]
    + [(100000, 100, 100), (1, 2 ** 27, 1), (1, 2 ** 27, 256)])
# both sides of every layout switch (whole-row sort up to len 2048; split rows below 264 rows; list sort in shared memory
# up to k = 4096, cub above) and of the row kernel's buffer (a row of up to ~12000 elements read once)
SWITCH_SHAPES = [(7, 2048, 100), (7, 2049, 100), (263, 40000, 50), (264, 40000, 50), (300, 9000, 4096), (300, 9000, 4097),
                 (5, 70000, 4096), (5, 70000, 4097), (300, 4096, 2048), (300, 12000, 10), (300, 13000, 10), (1, 2049, 2049)]


def check(x, k, select_min, in_idx=None, **kw):
    v, i = select_k(x, k=k, select_min=select_min, in_idx=in_idx, **kw)
    torch.cuda.synchronize()
    rv, ri = ref_select_k(x.cpu().numpy(), v.shape[1], select_min, None if in_idx is None else in_idx.cpu().numpy())
    gv, gi = v.cpu().numpy(), i.cpu().numpy()
    assert gv.shape == rv.shape and gi.dtype == np.int64
    bad = (gi != ri) | (gv.view(np.uint32) != rv.view(np.uint32))
    assert not bad.any(), "%d mismatches, first at %s" % (bad.sum(), np.argwhere(bad)[0])
    return gv, gi


def make(kind, rows, n, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    if kind == "normal":
        return torch.randn((rows, n), device=DEV, generator=g)
    if kind == "equal":
        return torch.full((rows, n), 1.5, device=DEV)
    if kind == "four":
        return torch.tensor([-1.0, 0.25, 3.0, 7.5], device=DEV)[torch.randint(0, 4, (rows, n), device=DEV, generator=g)]
    if kind == "top21":   # every value agrees in its top 22 bits: the first two 11-bit digits tie
        low = torch.randint(0, 2 ** 10, (rows, n), device=DEV, generator=g, dtype=torch.int32)
        return (torch.full((rows, n), 0x3FC00000, dtype=torch.int32, device=DEV) | low).view(torch.float32)
    if kind == "ascending":
        return torch.arange(n, device=DEV, dtype=torch.float32).repeat(rows, 1) - n / 2
    if kind == "descending":
        return n / 2 - torch.arange(n, device=DEV, dtype=torch.float32).repeat(rows, 1)
    if kind == "special":
        pool = np.array([0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00000, 0x7F800123, 0xFFA00001,
                         0x00000001, 0x80000001, 0x007FFFFF, 0x807FFFFF, 0x3F800000, 0xBF800000], dtype=np.uint32)
        p = torch.from_numpy(pool.view(np.int32)).to(DEV)
        sel = torch.randint(0, len(pool) + 4, (rows, n), device=DEV, generator=g)
        return torch.where(sel < len(pool), p[sel.clamp(max=len(pool) - 1)].view(torch.float32),
                           torch.randn((rows, n), device=DEV, generator=g))
    if kind == "negative":
        return -torch.rand((rows, n), device=DEV, generator=g) - 1e-3
    raise ValueError(kind)


@pytest.mark.parametrize("rows,n,k", REFERENCE_SHAPES + SWITCH_SHAPES)
def test_shapes(rows, n, k):
    x = make("normal", rows, n, seed=rows * 7 + k)
    for select_min in (True, False):
        check(x, k, select_min)


DISTS = ["normal", "equal", "four", "top21", "ascending", "descending", "special", "negative"]
LAYOUT_SHAPES = [(50, 1000, 17), (300, 20000, 100), (300, 6000, 1000), (4, 300000, 64), (300, 9000, 5000),
                 (3, 100000, 4500)]


@pytest.mark.parametrize("kind", DISTS)
@pytest.mark.parametrize("rows,n,k", LAYOUT_SHAPES)
def test_distributions(kind, rows, n, k):
    x = make(kind, rows, n, seed=k)
    for select_min in (True, False):
        _, gi = check(x, k, select_min)
        if kind == "equal":
            assert (gi == np.arange(k)[None, :]).all()


@pytest.mark.parametrize("rows,n,k", [(20, 700, 9), (300, 20000, 100), (4, 300000, 64), (3, 100000, 4500)])
def test_payload_and_preallocated_outputs(rows, n, k):
    x = make("four", rows, n, seed=3)
    pay = torch.randint(-2 ** 62, 2 ** 62, (rows, n), device=DEV, dtype=torch.int64)
    dist = torch.empty((rows, k), device=DEV)
    idx = torch.empty((rows, k), device=DEV, dtype=torch.int64)
    for select_min in (True, False):
        check(x, None, select_min, in_idx=pay, distances=dist, indices=idx)
        v, i = select_k(x, select_min=select_min, in_idx=pay, distances=dist, indices=idx)
        assert v is dist and i is idx


def test_argument_errors():
    x = torch.randn((4, 100), device=DEV)
    with pytest.raises(LogicError):
        select_k(x, k=0)
    with pytest.raises(LogicError):
        select_k(x, k=101)
    with pytest.raises(LogicError):
        select_k(x[:, ::2], k=3)
    with pytest.raises(LogicError):
        select_k(x.t(), k=3)


def test_known_answers_of_the_reference():
    cases = json.load(open(os.path.join(ROOT, "tests", "golden", "select_k_edgecases.json")))["cases"]
    for c in cases:
        x = torch.tensor([[float(t) for t in c["input"]]], device=DEV)
        v, i = select_k(x, k=c["k"], select_min=c["select_min"])
        want = np.array([float(t) for t in c["values"]], dtype=np.float32)
        got = v.cpu().numpy()[0]
        assert ((got == want) | (np.isnan(got) & np.isnan(want))).all(), c["name"]
        assert i.cpu().numpy()[0].tolist() == c["indices"], c["name"]
        check(x, c["k"], c["select_min"])


@pytest.mark.parametrize("rows,n,k", [(1000, 500, 20), (300, 20000, 100), (4, 300000, 64), (3, 100000, 4500)])
def test_graph_capture_no_sync_no_alloc(rows, n, k):
    """b2d_select_k through ctypes, captured in a CUDA graph with preallocated buffers and replayed once."""
    L = _lib.lib()
    x = make("four", rows, n, seed=11)
    ws = torch.empty(max(256, L.b2d_select_k_workspace_bytes(rows, n, k)), dtype=torch.uint8, device=DEV)
    ov = torch.full((rows, k), -7.0, device=DEV)
    oi = torch.full((rows, k), -7, dtype=torch.int64, device=DEV)

    def call(stream):
        _lib.check(L.b2d_select_k(ctypes.c_void_p(stream), x.data_ptr(), n, None, rows, n, k, 0, ov.data_ptr(),
                                  oi.data_ptr(), ws.data_ptr(), ws.numel()))

    call(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    ev, ei = ov.clone(), oi.clone()
    ov.fill_(-7.0)
    oi.fill_(-7)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        call(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(ov.view(torch.int32), ev.view(torch.int32)) and torch.equal(oi, ei)
    check(x, k, False)


def test_cityblock_knn_with_100_neighbours_from_two_slabs():
    """pairwise_distance (L1) over two column slabs of y, select_k of each, then select_k of [slab-0 top-k | slab-1
    top-k] with the slab results' indices as in_idx.  Small-integer data: every distance is exact, so ties abound and
    the result must equal the oracle's kNN exactly, tie rule included."""
    rng = np.random.default_rng(2)
    xh = rng.integers(0, 4, (300, 16)).astype(np.float32)
    yh = rng.integers(0, 4, (5000, 16)).astype(np.float32)
    x, y = torch.from_numpy(xh).to(DEV), torch.from_numpy(yh).to(DEV)
    kk, cut = 100, 2600
    vals, idxs = [], []
    for j0, j1 in ((0, cut), (cut, 5000)):
        d = torch.as_tensor(pairwise_distance(x, y[j0:j1], metric=DistanceType.L1), device=DEV)
        v, i = select_k(d, k=kk)
        vals.append(v)
        idxs.append(i + j0)
    v, i = select_k(torch.cat(vals, 1).contiguous(), k=kk, in_idx=torch.cat(idxs, 1).contiguous())
    ri, rv = oracle.knn(xh, yh, kk, DistanceType.L1)
    assert (i.cpu().numpy() == ri).all()
    assert (v.cpu().numpy() == rv.astype(np.float32)).all()


def test_l2_select_matches_fused_knn():
    torch.manual_seed(4)
    x, y = torch.randn((500, 32), device=DEV), torch.randn((20000, 32), device=DEV)
    kk = 64
    d = torch.as_tensor(pairwise_distance(x, y, metric=DistanceType.L2Expanded), device=DEV)
    v, i = select_k(d, k=kk)
    bd, bi = brute_force.knn(y, x, k=kk)
    i, bi = i.cpu().numpy(), bi.cpu().numpy()
    dh = d.cpu().numpy()
    diff = i != bi
    assert diff.mean() < 0.01
    # where the two orders differ, the two rows' distances are fp32 near-ties
    ra, rb = np.take_along_axis(dh, i, 1), np.take_along_axis(dh, bi, 1)
    assert (np.abs(ra - rb)[diff] <= 1e-4 * np.maximum(1.0, np.abs(ra[diff]))).all()
    assert np.allclose(v.cpu().numpy(), bd.cpu().numpy(), rtol=1e-4, atol=1e-4)
