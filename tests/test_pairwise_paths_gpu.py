"""GPU tier: the dense pairwise distance on every dispatch path of the host code, against the fp64 oracle.

Every case builds its operands from (m, n, k, dtype, order, paddings, base offsets in elements, alias), fills the whole
output allocation with NaN and its padding with a sentinel, asks b2d_debug_pairwise_plan which kernels the call will run,
asserts that this is the path the case is named after, runs the call and compares with the oracle.  A changed threshold
in the host code therefore fails the case that would silently have left its path.

Paths of the tensor kernel (EPI_STORE) the host code can produce, each named by at least one case below, for fp32 and
for fp16 inputs (test_every_tensor_path_is_named_by_a_case checks the list against the plans of the cases):

    kernel     acc_mode              stores
    resident   0 (single pass)       tma | vec2 | scalar        k <= 128
    resident   3 (last K chunk)      vec2 | scalar              remainder chunk of 1..4 k-blocks: k = 321..384, 513, 640
    streaming  0 (single pass)       tma | vec2 | scalar        128 < k <= 320; Jaccard / Dice at every k > 128
    streaming  1 (first K chunk)     vec2 | scalar              k > 320
    streaming  2 (middle K chunk)    vec2 | scalar              k > 512
    streaming  3 (last K chunk)      vec2 | scalar              k = 385..512, 1024

("vec2": register stores, 8-byte vectors on the tiles wholly inside dist; "scalar": odd pitch or a base that is only
4-byte aligned.  The resident kernel never runs acc_mode 1 or 2: every chunk but the last has 8 k-blocks.  K chunks
never use TMA stores.)

fp64 SIMT kernel (64 x 64 tiles, 16-column k-blocks): m, n in {1, 63, 64, 65}, k in {1, 15, 16, 17, 300}, both orders,
padded pitches, aliased inputs, a NaN row, every metric, and the Gram matrices' fp64 branch.
fp32 unexpanded kernels (128 x 128 tiles, 32-column k-blocks): all ten metrics at k in {1, 3, 4, 5, 31, 32, 33, 64}
with (vec_x, vec_y) = (1, 1) (the TMA-fed kernel), (1, 0), (0, 1), (0, 0), and Fortran order.

Sections: 1 streaming kernel, 2 K-chunked accumulation, 3 fp16 inputs, 4 fp64, 5 unexpanded SIMT."""
import ctypes

import numpy as np
import pytest
import torch

import oracle
from oracle import DistanceType as DT
from raft_b200 import _lib
from raft_b200.common import DeviceResources
from raft_b200.distance import pairwise_distance
from raft_b200.distance.pairwise_distance import _operands

pytestmark = pytest.mark.gpu
EPS = 1e-4
PAD = -7.0            # what the padding of an output holds before and after a call
JUNK = 777.0          # what the padding of an input holds: finite, so a kernel that reads it computes wrong values
NP = {"f32": np.float32, "f16": np.float16, "f64": np.float64}
L2 = (DT.L2Expanded, DT.L2SqrtExpanded, DT.L2Unexpanded, DT.L2SqrtUnexpanded)
SEEN = {}             # (dtype, kernel, acc_mode, stores) -> a case that ran it


# ---------------------------------------------------------------------------------------------------------------------
# operands, plan, comparison

def data(metric, m, n, k, seed=0):
    """fp64-free host data of the kind the metric is defined on."""
    rng = np.random.default_rng(1000 + seed)
    if metric in (DT.KLDivergence, DT.JensenShannon, DT.HellingerExpanded):
        x, y = rng.random((m, k)) + 0.05, rng.random((n, k)) + 0.05
        x /= x.sum(1, keepdims=True); y /= y.sum(1, keepdims=True)
    elif metric in (DT.HammingUnexpanded, DT.RusselRaoExpanded, DT.JaccardExpanded, DT.DiceExpanded):
        x, y = rng.random((m, k)) > 0.5, rng.random((n, k)) > 0.5
    elif metric == DT.BrayCurtis:
        x, y = rng.random((m, k)) * 9 + 0.1, rng.random((n, k)) * 9 + 0.1
    else:
        x, _, c = oracle.make_blobs(m, k, seed=1234 + seed)
        y, _, _ = oracle.make_blobs(n, k, seed=4321 + seed, centers=c)
    return x.astype(np.float32), y.astype(np.float32)


def place(a, order="C", pad=0, off=0, junk=JUNK):
    """The matrix `a` on the device in the given order, with `pad` extra elements per leading dimension and its first
    element `off` elements behind an allocation boundary; everything around the values holds `junk`."""
    t = torch.from_numpy(np.ascontiguousarray(a))
    r, c = t.shape
    if order == "F":
        r, c, t = c, r, t.t()
    buf = torch.full((off + r * (c + pad),), junk, dtype=t.dtype, device="cuda")
    v = buf[off:].view(r, c + pad)[:, :c]
    v.copy_(t)
    return v.t() if order == "F" else v


class Out:
    """An [m, n] output in `order` with padding and base offset: NaN where the result goes, PAD everywhere else."""

    def __init__(self, m, n, dtype=torch.float32, order="C", pad=0, off=0):
        r, c = (n, m) if order == "F" else (m, n)
        self.buf = torch.full((off + r * (c + pad),), PAD, dtype=dtype, device="cuda")
        v = self.buf[off:].view(r, c + pad)[:, :c]
        v.fill_(float("nan"))
        self.view = v.t() if order == "F" else v

    def result(self):
        """the result; the padding must still hold PAD"""
        got = self.view.cpu().numpy().copy()
        self.view.fill_(PAD)
        assert bool((self.buf == PAD).all()), "the call wrote outside the result"
        return got


def plan_of(metric, X, Y, out):
    """b2d_debug_pairwise_plan for exactly the arguments pairwise_distance(X, Y, out=out) passes to the C ABI."""
    x_cai, y_cai, d_cai, _, row_major, ldx, ldy, ldd = _operands(X, Y, out)
    dt = {np.dtype(np.float32): _lib.B2D_F32, np.dtype(np.float16): _lib.B2D_F16, np.dtype(np.float64): _lib.B2D_F64}[x_cai.dtype]
    words = (ctypes.c_int * 70)()
    _lib.check(_lib.lib().b2d_debug_pairwise_plan(int(metric), dt, x_cai.data, ldx, y_cai.data, ldy, d_cai.data, ldd,
                                                  x_cai.shape[0], y_cai.shape[0], x_cai.shape[1], int(row_major), words, 70))
    path = ["none", "tensor", "simt", "simt-tma", "f64"][words[0]]
    stores = "tma" if words[1] else "vec2" if words[2] else "scalar"
    launches = [(words[7 + 4 * i], words[8 + 4 * i], "res" if words[9 + 4 * i] else "str") for i in range(words[5])]
    return {"path": path, "stores": stores, "vec": (words[3], words[4]), "launches": launches}


def want_plan(pl, text):
    """`text`: the path a case is named after -- 'tma 5:0:str', 'scalar 8:1:str 3:3:res' (stores, then k-blocks :
    acc_mode : kernel of every launch), 'simt 1 0' (vec_x vec_y), 'simt-tma', 'f64'."""
    if pl["path"] == "tensor":
        got = " ".join([pl["stores"]] + ["%d:%d:%s" % l for l in pl["launches"]])
    elif pl["path"] == "simt":
        got = "simt %d %d" % pl["vec"]
    else:
        got = pl["path"]
    assert got == text, f"the case is for path '{text}' but the host code plans '{got}'"


def run(metric, x, y, path, dtype="f32", order="C", xpad=0, ypad=0, opad=0, xoff=0, yoff=0, ooff=0, alias=False, p=2.0,
        handle=None):
    """One call on placed copies of x and y (alias: y is x itself) into a NaN-filled output; the plan is checked against
    `path` before anything is launched.  Returns the result as a numpy array."""
    xh = x.astype(NP[dtype])
    X = place(xh, order, xpad, xoff)
    Y = X if alias else place(y.astype(NP[dtype]), order, ypad, yoff)
    out = Out(x.shape[0], x.shape[0] if alias else y.shape[0], torch.float64 if dtype == "f64" else torch.float32, order,
              opad, ooff)
    pl = plan_of(metric, X, Y, out.view)
    want_plan(pl, path)
    if pl["path"] == "tensor":
        for _, acc, kern in pl["launches"]:
            SEEN.setdefault((dtype, kern, acc, pl["stores"]), path)
    pairwise_distance(X, Y, out=out.view, metric=metric, p=p, handle=handle)
    torch.cuda.synchronize()
    return out.result()


def norms(x, y):
    return oracle.row_norm_sq(x)[:, None] + oracle.row_norm_sq(y)[None, :]


def check32(metric, got, x, y, tag, p=2.0):
    """fp32 / fp16 inputs (x, y: the values the kernel was given): the standing 1e-4 rule, with the |x||y|-scaled bound
    for InnerProduct (test_pairwise_gpu.py::test_inner_product_vs_oracle) and the floor of 8 ulp of (xn + yn) for the
    expanded L2 forms on near-coincident pairs (test_fuzz_gpu.py::test_random_shapes_all_paths)."""
    ref = oracle.pairwise_distance(x, y, metric, p)
    assert got.shape == ref.shape
    if metric == DT.InnerProduct:
        scale = np.sqrt(oracle.row_norm_sq(x))[:, None] * np.sqrt(oracle.row_norm_sq(y))[None, :]
        bad = ~(np.abs(got - ref) <= 1e-5 * scale + 1e-6)
    else:
        bad = ~oracle.compare_approx(got, ref, EPS)
        if metric in (DT.L2Expanded, DT.L2SqrtExpanded):
            sq = metric == DT.L2SqrtExpanded
            g2 = got.astype(np.float64) ** 2 if sq else got.astype(np.float64)
            bad &= ~(np.abs(g2 - (ref ** 2 if sq else ref)) <= 8 * 2.0 ** -24 * norms(x, y))
    assert not bad.any(), (tag, int(bad.sum()), tuple(np.argwhere(bad)[0]), got[tuple(np.argwhere(bad)[0])],
                           ref[tuple(np.argwhere(bad)[0])])
    return ref


# ---------------------------------------------------------------------------------------------------------------------
# 1. streaming kernel (128 < k <= 320): ragged edges, few items, both register epilogues

STREAM = [
    # id, m, n, k, out pad, out offset, path
    ("stream-nkb5-tma-m1", 1, 512, 129, 0, 0, "tma 5:0:str"),
    ("stream-nkb5-tma-m64-half-y-block", 64, 356, 129, 0, 0, "tma 5:0:str"),
    ("stream-nkb5-tma-m65", 65, 256, 129, 0, 0, "tma 5:0:str"),
    ("stream-nkb5-tma-m127-padded", 127, 260, 130, 4, 0, "tma 5:0:str"),
    ("stream-nkb5-tma-one-item", 100, 200, 160, 0, 0, "tma 5:0:str"),
    ("stream-nkb7-tma-4-items", 129, 300, 200, 0, 0, "tma 7:0:str"),
    ("stream-nkb10-tma-m385", 385, 644, 320, 0, 0, "tma 10:0:str"),
    ("stream-nkb10-tma-m1-n4", 1, 4, 320, 0, 0, "tma 10:0:str"),
    ("stream-nkb5-regstore-vec2-n%4", 193, 387, 129, 1, 0, "vec2 5:0:str"),
    ("stream-nkb5-regstore-vec2-base8", 130, 256, 160, 2, 2, "vec2 5:0:str"),
    ("stream-nkb5-regstore-scalar-odd-pitch", 193, 387, 129, 0, 0, "scalar 5:0:str"),
    ("stream-nkb9-regstore-scalar-base4", 257, 512, 288, 0, 1, "scalar 9:0:str"),
    ("stream-nkb10-regstore-scalar-m1", 1, 301, 320, 0, 3, "scalar 10:0:str"),
    ("stream-nkb10-regstore-vec2-m127", 127, 130, 320, 0, 0, "vec2 10:0:str"),
]


@pytest.mark.parametrize("case", STREAM, ids=[c[0] for c in STREAM])
@pytest.mark.parametrize("metric", [DT.L2Expanded, DT.CosineExpanded], ids=["l2", "cosine"])
def test_streaming_kernel_edges(metric, case):
    tag, m, n, k, opad, ooff, path = case
    x, y = data(metric, m, n, k, seed=k + m)
    check32(metric, run(metric, x, y, path, opad=opad, ooff=ooff), x, y, tag)


def sampled_check(m, n, k, opad, ooff, path):
    """A result too large for a full oracle matrix: 2e5 sampled pairs, the corners, and every element finite (the
    output starts as NaN, so a tile that was never written shows)."""
    g = torch.Generator(device="cuda").manual_seed(m + k)
    centers = torch.rand(5, k, device="cuda", generator=g) * 20 - 10
    x = centers[torch.randint(0, 5, (m,), device="cuda", generator=g)] + torch.randn(m, k, device="cuda", generator=g)
    y = centers[torch.randint(0, 5, (n,), device="cuda", generator=g)] + torch.randn(n, k, device="cuda", generator=g)
    out = Out(m, n, pad=opad, off=ooff)
    pl = plan_of(DT.L2Expanded, x, y, out.view)
    want_plan(pl, path)
    pairwise_distance(x, y, out=out.view, metric=DT.L2Expanded)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(out.view).all())
    ii = torch.randint(0, m, (200000,), device="cuda", generator=g)
    jj = torch.randint(0, n, (200000,), device="cuda", generator=g)
    ii[:4] = torch.tensor([0, m - 1, 0, m - 1], device="cuda"); jj[:4] = torch.tensor([0, n - 1, n - 1, 0], device="cuda")
    got = out.view[ii, jj].cpu().numpy()
    ref = ((x[ii].cpu().numpy().astype(np.float64) - y[jj].cpu().numpy().astype(np.float64)) ** 2).sum(axis=1)
    ok, msg = oracle.match_approx(got, ref, EPS)
    assert ok, msg
    out.view.fill_(PAD)
    assert bool((out.buf == PAD).all())


@pytest.mark.parametrize("m,n,k,opad,ooff,path", [
    (70001, 1124, 160, 0, 0, "tma 5:0:str"),       # 547 x tiles x 5 y blocks (the last of one half): 3 tiles per item
    (70001, 700, 320, 1, 0, "scalar 10:0:str"),    # 547 x 3: 2 tiles per item, scalar register stores
    (50001, 1027, 160, 1, 0, "vec2 5:0:str"),      # 391 x 5: 2 tiles per item, vector register stores, n % 4 = 3
], ids=["stream-nkb5-tma-3-tiles-per-item", "stream-nkb10-scalar-2-tiles-per-item", "stream-nkb5-vec2-2-tiles-per-item"])
def test_streaming_kernel_several_x_tiles_per_item(m, n, k, opad, ooff, path):
    sampled_check(m, n, k, opad, ooff, path)


# ---------------------------------------------------------------------------------------------------------------------
# 2. K-chunked accumulation (k > 320)

CHUNK = [
    # id, metric, m, n, k, kwargs of run, path
    ("chunk-8+3-resident-acc3-vec2", DT.L2Expanded, 300, 260, 321, {}, "vec2 8:1:str 3:3:res"),
    ("chunk-8+3-resident-acc3-alias", DT.L2SqrtExpanded, 300, 300, 330, {"alias": True}, "vec2 8:1:str 3:3:res"),
    ("chunk-8+4-resident-acc3-scalar-odd-pitch", DT.L2Expanded, 257, 259, 384, {}, "scalar 8:1:str 4:3:res"),
    ("chunk-8+5-stream-acc3-padded-ldd", DT.L2Expanded, 200, 150, 385, {"opad": 10}, "vec2 8:1:str 5:3:str"),
    ("chunk-8+5-stream-acc3-scalar-base4", DT.L2SqrtExpanded, 130, 256, 400, {"ooff": 1}, "scalar 8:1:str 5:3:str"),
    ("chunk-8+8-stream-inner-product", DT.InnerProduct, 129, 513, 512, {"opad": 1}, "vec2 8:1:str 8:3:str"),
    ("chunk-8+8+1-resident-acc3-vec2", DT.L2Expanded, 193, 300, 513, {}, "vec2 8:1:str 8:2:str 1:3:res"),
    ("chunk-8+8+1-resident-acc3-scalar-alias", DT.L2Expanded, 259, 259, 513, {"alias": True},
     "scalar 8:1:str 8:2:str 1:3:res"),
    ("chunk-8+8+4-cosine-fortran", DT.CosineExpanded, 260, 190, 640, {"order": "F"}, "vec2 8:1:str 8:2:str 4:3:res"),
    ("chunk-8+3-correlation-fortran-scalar", DT.CorrelationExpanded, 131, 77, 350, {"order": "F", "xpad": 3, "ypad": 1},
     "scalar 8:1:str 3:3:res"),
    ("chunk-8x4-stream-acc2-scalar", DT.L2Expanded, 129, 131, 1024, {}, "scalar 8:1:str 8:2:str 8:2:str 8:3:str"),
    ("chunk-8x4-stream-acc2-vec2-padded-inputs", DT.L2SqrtExpanded, 64, 258, 1000, {"xpad": 5, "ypad": 8, "opad": 6},
     "vec2 8:1:str 8:2:str 8:2:str 8:3:str"),
    ("chunk-8+8-hellinger", DT.HellingerExpanded, 150, 140, 512, {}, "vec2 8:1:str 8:3:str"),
    ("chunk-8+3-russelrao", DT.RusselRaoExpanded, 150, 141, 333, {}, "scalar 8:1:str 3:3:res"),
]


@pytest.mark.parametrize("case", CHUNK, ids=[c[0] for c in CHUNK])
@pytest.mark.parametrize("dtype", ["f32", "f16"])
def test_k_chunked_accumulation(dtype, case):
    """The first chunk overwrites (the output starts as NaN), the read-back stays inside the result (the padding keeps
    its sentinel), the post-processing runs once, on the last chunk."""
    tag, metric, m, n, k, kw, path = case
    x, y = data(metric, m, n, k, seed=k)
    x, y = x.astype(NP[dtype]), y.astype(NP[dtype])
    got = run(metric, x, y, path, dtype=dtype, **kw)
    check32(metric, got, x, x if kw.get("alias") else y, tag)
    if kw.get("alias"):
        assert (np.diag(got) == 0).all(), "d(i, i) of aliased inputs must be exactly 0"


def test_k_chunked_partial_sums_cross_zero():
    """InnerProduct (no clamp) and L2 on data whose per-chunk contributions have opposite signs: columns [0, 256) of y
    are those of x, columns [256, 512) their negatives, so the inner product's partial sum after the first chunk is
    |x_a|^2 and the total is near 0, and the L2 cross term of the first chunk alone cancels the norms of those columns.
    (For the L2 family every partial sum is |x_a - y_a|^2 + |x_rest|^2 + |y_rest|^2 >= 0, so an early clamp could not
    change a finite result; what must not run early is the rest of the post-processing, which the sqrt cases above
    cover.)"""
    rng = np.random.default_rng(3)
    x = rng.standard_normal((200, 512)).astype(np.float32)
    y = np.concatenate([x[:160, :256], -x[:160, 256:]], axis=1)
    y += 0.01 * rng.standard_normal(y.shape).astype(np.float32)
    for metric in (DT.InnerProduct, DT.L2Expanded, DT.L2SqrtExpanded):
        check32(metric, run(metric, x, y, "vec2 8:1:str 8:3:str"), x, y, metric)


@pytest.mark.parametrize("dtype", ["f32", "f16"])
def test_k_chunked_nan_rows_and_outlier_rows(dtype):
    """A NaN poisons its row / column through every chunk and nothing else; rows far below the matrix maximum take
    their own exponent (the per-row factors apply to every chunk's products)."""
    x, y = data(DT.L2Expanded, 200, 270, 400, seed=9)
    x[::3] *= 2.0 ** -13
    y[5] *= 2.0 ** -14
    x, y = x.astype(NP[dtype]), y.astype(NP[dtype])
    x[7, 300] = np.nan
    y[201, 13] = np.nan
    for metric in (DT.L2Expanded, DT.CosineExpanded):
        got = run(metric, x, y, "vec2 8:1:str 5:3:str", dtype=dtype, opad=2)
        assert np.isnan(got[7]).all() and np.isnan(got[:, 201]).all()
        kr, kc = np.arange(200) != 7, np.arange(270) != 201
        sub = got[kr][:, kc]
        assert np.isfinite(sub).all()
        check32(metric, sub, x[kr], y[kc], (metric, dtype))


@pytest.mark.parametrize("metric", [DT.JaccardExpanded, DT.DiceExpanded, DT.RusselRaoExpanded, DT.HellingerExpanded,
                                    DT.InnerProduct, DT.CosineExpanded])
def test_k_1024_every_expanded_metric(metric):
    """k = 1024.  Jaccard and Dice run one 32-k-block MMA chain (the ratio needs the whole inner product), the others
    four K chunks; all hold the 1e-4 rule, on indicator data (exact) and on non-negative real data."""
    ratio = metric in (DT.JaccardExpanded, DT.DiceExpanded)
    path = "tma 32:0:str" if ratio else "vec2 8:1:str 8:2:str 8:2:str 8:3:str"
    x, y = data(metric, 300, 260, 1024, seed=1)
    got = run(metric, x, y, path)
    ref = check32(metric, got, x, y, metric)
    if metric == DT.RusselRaoExpanded:
        assert np.array_equal(got, ref.astype(np.float32)), "indicator data: exact integer sums, k a power of two"
    if ratio:
        assert np.abs(got - ref).max() <= 2.0 ** -22, "indicator data: exact integer sums, one rounded ratio"
        rng = np.random.default_rng(8)
        x = (rng.random((300, 1024)) * 2).astype(np.float32)
        y = (x[rng.integers(0, 300, 260)] * (1 + 0.05 * rng.standard_normal((260, 1024)))).astype(np.float32)  # near pairs
        got = run(metric, x, y, path)
        ref = check32(metric, got, x, y, metric)
    print("measured", metric.name, "k=1024 max |got - ref| =", float(np.abs(got - ref).max()),
          "max relative =", float((np.abs(got - ref) / np.maximum(np.abs(ref), 1e-30)).max()))


# ---------------------------------------------------------------------------------------------------------------------
# cross-path equality, only where every arithmetic step is shared

@pytest.mark.parametrize("k,first,launches", [(96, "tma", "3:0:res"), (200, "tma", "7:0:str"),
                                              (400, "vec2", "8:1:str 5:3:str"), (513, "vec2", "8:1:str 8:2:str 1:3:res")],
                         ids=["resident", "streaming", "chunk-8+5", "chunk-8+8+1"])
def test_store_paths_are_bit_identical(k, first, launches):
    """The same problem through TMA stores, vector register stores and scalar register stores, and from padded /
    offset copies of the inputs: the epilogue computes the same registers, only the way out differs.  Twice the same
    call: the same bits."""
    for metric in (DT.L2SqrtExpanded, DT.CosineExpanded):
        x, y = data(metric, 300, 388, k, seed=k)
        base = run(metric, x, y, f"{first} {launches}")
        check32(metric, base, x, y, (metric, k))
        assert np.array_equal(base, run(metric, x, y, f"{first} {launches}"))
        assert np.array_equal(base, run(metric, x, y, f"vec2 {launches}", opad=2))
        assert np.array_equal(base, run(metric, x, y, f"scalar {launches}", opad=1))
        assert np.array_equal(base, run(metric, x, y, f"scalar {launches}", ooff=1))
        assert np.array_equal(base, run(metric, x, y, f"{first} {launches}", xpad=3, ypad=9, xoff=1, yoff=2))


# ---------------------------------------------------------------------------------------------------------------------
# 3. fp16 inputs: the oracle on the fp16 values is the exact reference

F16_LAYOUTS = [
    # id, k, kwargs, path for a 200 x 136 result
    ("f16-k7-odd-ld", 7, {}, "tma 1:0:res"),
    ("f16-k33-base-2-bytes", 33, {"xoff": 1, "yoff": 3}, "tma 2:0:res"),
    ("f16-k64-padded-ld", 64, {"xpad": 3, "ypad": 8, "opad": 1}, "scalar 2:0:res"),
    ("f16-k100-fortran", 100, {"order": "F", "xpad": 1, "ypad": 2}, "tma 4:0:res"),
    ("f16-k129-streaming-padded", 129, {"xpad": 1, "yoff": 1, "opad": 2}, "vec2 5:0:str"),
    ("f16-k320-streaming-fortran", 320, {"order": "F", "ooff": 1}, "scalar 10:0:str"),
    ("f16-k330-chunked-odd-ld", 330, {"xpad": 1, "ypad": 1}, "vec2 8:1:str 3:3:res"),
]


@pytest.mark.parametrize("case", F16_LAYOUTS, ids=[c[0] for c in F16_LAYOUTS])
@pytest.mark.parametrize("metric", oracle.EXPANDED, ids=[mt.name for mt in oracle.EXPANDED])
def test_fp16_every_expanded_metric_and_layout(metric, case):
    tag, k, kw, path = case
    if metric in (DT.JaccardExpanded, DT.DiceExpanded) and k > 320:
        path = path.split()[0].replace("vec2", "tma") + " 11:0:str"      # never chunked
    x, y = data(metric, 200, 136, k, seed=k)
    x, y = x.astype(np.float16), y.astype(np.float16)
    check32(metric, run(metric, x, y, path, dtype="f16", **kw), x, y, (tag, metric))


def has_lo(handle):
    """the word of the tensor path's workspace that says some operand element needed its fp16 lo half"""
    return int(handle.workspace(256)[12:16].view(torch.int32).item())


@pytest.mark.parametrize("k,path", [(96, "tma 3:0:res"), (200, "tma 7:0:str"), (400, "vec2 8:1:str 5:3:str")])
def test_fp16_integer_data_is_exact_on_the_one_product_path(k, path):
    rng = np.random.default_rng(k)
    x = rng.integers(-8, 9, (300, k)).astype(np.float16)
    y = rng.integers(-8, 9, (260, k)).astype(np.float16)
    h = DeviceResources()
    for metric in (DT.L2Expanded, DT.InnerProduct):
        got = run(metric, x, y, path, dtype="f16", handle=h)
        h.sync()
        assert np.array_equal(got.astype(np.float64), oracle.pairwise_distance(x, y, metric))
        assert has_lo(h) == 0
    # ordinary fp16 data too: a power-of-two scale keeps every fp16 value exact, so the lo halves stay empty
    xb, yb = data(DT.L2Expanded, 300, 260, k)
    run(DT.L2Expanded, xb.astype(np.float16), yb.astype(np.float16), path, dtype="f16", handle=h)
    h.sync()
    assert has_lo(h) == 0
    run(DT.L2Expanded, xb, yb, path, handle=h)
    h.sync()
    assert has_lo(h) == 1     # (the word is live: fp32 data does need them)


def test_fp16_values_at_the_edges_of_the_format():
    """65504, subnormals, rows of zeros, and NaN / Inf rows, which stay local."""
    rng = np.random.default_rng(6)
    x = rng.standard_normal((150, 72)).astype(np.float16)
    y = rng.standard_normal((140, 72)).astype(np.float16)
    x[3] = 0; y[4] = 0
    x[5] = 65504; y[6] = -65504; x[7, ::2] = 65504
    x[8] = np.float16(6e-8) * rng.integers(1, 9, 72); y[9] = np.float16(6e-8) * rng.integers(1, 9, 72)   # subnormals
    x[10, 5] = np.nan; y[11, 70] = np.inf; x[12, 0] = -np.inf
    for metric in (DT.L2Expanded, DT.L2SqrtExpanded, DT.InnerProduct, DT.CosineExpanded):
        got = run(metric, x, y, "tma 3:0:res", dtype="f16")
        assert not np.isfinite(got[10]).any() and not np.isfinite(got[12]).any() and not np.isfinite(got[:, 11]).any()
        kr, kc = ~np.isin(np.arange(150), (10, 12)), np.arange(140) != 11
        if metric == DT.CosineExpanded:      # a zero row has no direction: NaN, as in the definition
            assert np.isnan(got[3][kc]).all() and np.isnan(got[kr][:, 4]).all()
            kr &= np.arange(150) != 3; kc &= np.arange(140) != 4
        sub = got[kr][:, kc]
        assert np.isfinite(sub).all()
        check32(metric, sub, x[kr], y[kc], metric)
    assert run(DT.L2Expanded, x, y, "tma 3:0:res", dtype="f16")[3, 4] == 0


def test_fp16_unexpanded_metrics_are_refused():
    a = torch.zeros(8, 16, dtype=torch.float16, device="cuda")
    out = torch.zeros(8, 8, device="cuda")
    L = _lib.lib()
    for metric in oracle.UNEXPANDED:
        assert L.b2d_pairwise_workspace_bytes(int(metric), _lib.B2D_F16, 8, 8, 16) == 2 ** 64 - 1
        rc = L.b2d_pairwise_distance(None, int(metric), _lib.B2D_F16, a.data_ptr(), 16, a.data_ptr(), 16, out.data_ptr(), 8,
                                     8, 8, 16, 1, 2.0, None, 0)
        assert rc == _lib.B2D_ERR_UNSUPPORTED
        with pytest.raises(ValueError):
            pairwise_distance(a, a, metric=metric)
    torch.cuda.synchronize()
    assert bool((out == 0).all())


# ---------------------------------------------------------------------------------------------------------------------
# 4. fp64 SIMT kernel

F64_ALL = tuple(oracle.EXPANDED) + tuple(oracle.UNEXPANDED)
ULP = 2.0 ** -52


def check64(metric, got, x, y, tag, p=3.0):
    """|got - ref| <= 64 ulp of the magnitude the metric is computed at: the value itself for the sums of
    non-negative terms (L1, L2 in the difference form, Linf, Canberra, Lp, Hamming, BrayCurtis), xn + yn for the L2
    family (the oracle itself uses the expanded form), |x||y| for the inner product, 1 for the ratios; on the squares
    for the metrics that end in a square root of a difference.  Measured worst cases: DESIGN.md, numerics."""
    ref = oracle.pairwise_distance(x, y, metric, p)
    g, r = got, ref
    if metric in (DT.HellingerExpanded, DT.JensenShannon):
        g, r = got ** 2, ref ** 2
    if metric in L2:
        floor = norms(x, y)
        if metric in (DT.L2SqrtExpanded, DT.L2SqrtUnexpanded):
            g, r = got ** 2, ref ** 2
    elif metric == DT.InnerProduct:
        floor = np.sqrt(oracle.row_norm_sq(x))[:, None] * np.sqrt(oracle.row_norm_sq(y))[None, :]
    elif metric == DT.CorrelationExpanded:   # k <x, y> - sum x sum y cancels: the error is an ulp of k |x||y| over the centred norms
        k = x.shape[1]
        cx = np.sqrt(k * oracle.row_norm_sq(x) / np.maximum(k * oracle.row_norm_sq(x) - x.sum(1) ** 2, 1e-300))
        cy = np.sqrt(k * oracle.row_norm_sq(y) / np.maximum(k * oracle.row_norm_sq(y) - y.sum(1) ** 2, 1e-300))
        floor = cx[:, None] * cy[None, :]
    elif metric in (DT.L1, DT.Linf, DT.Canberra, DT.LpUnexpanded, DT.HammingUnexpanded, DT.BrayCurtis):
        floor = 0.0
    else:
        floor = 1.0
    err = np.abs(g - r)
    tol = 64 * ULP * (np.abs(r) + floor)
    both_nan = np.isnan(g) & np.isnan(r)
    bad = ~((err <= tol) | both_nan)
    assert not bad.any(), (tag, metric, int(bad.sum()), tuple(np.argwhere(bad)[0]), float(np.nanmax(err / np.maximum(tol, 1e-300))))
    with np.errstate(invalid="ignore", divide="ignore"):
        return float(np.nanmax(np.where(tol > 0, err / (tol / 64), 0.0)))


def data64(metric, m, n, k, seed):
    x, y = data(metric, m, n, k, seed)
    x, y = x.astype(np.float64), y.astype(np.float64)
    if metric not in (DT.HammingUnexpanded, DT.RusselRaoExpanded, DT.JaccardExpanded, DT.DiceExpanded):
        x *= 1 + 1e-9; y *= 1 - 1e-9          # values that fp32 cannot represent
    return x, y


F64_SHAPES = [(1, 1, 1), (63, 65, 15), (64, 64, 16), (65, 63, 17), (1, 130, 16), (130, 1, 33), (65, 129, 300)]


@pytest.mark.parametrize("metric", F64_ALL, ids=[mt.name for mt in F64_ALL])
def test_fp64_tile_and_k_block_edges(metric):
    worst = 0.0
    for i, (m, n, k) in enumerate(F64_SHAPES):
        if metric == DT.CorrelationExpanded and k < 3:
            continue
        x, y = data64(metric, m, n, k, seed=i)
        for order, kw in (("C", {}), ("C", {"xpad": 3, "ypad": 1, "opad": 5, "ooff": 1}), ("F", {}),
                          ("F", {"xpad": 2, "ypad": 7, "opad": 3})):
            got = run(metric, x, y, "f64", dtype="f64", order=order, p=3.0, **kw)
            worst = max(worst, check64(metric, got, x, y, (m, n, k, order, kw)))
    print("measured fp64", metric.name, "worst error in ulp of the metric's magnitude:", round(worst, 2))


def test_fp64_aliased_inputs_and_nan_row():
    x, _ = data64(DT.L2Expanded, 130, 1, 37, seed=2)
    for metric in L2 + (DT.L1, DT.Linf, DT.Canberra):
        got = run(metric, x, x, "f64", dtype="f64", alias=True, opad=1)
        assert (np.diag(got) == 0).all(), metric          # the difference form: exact zeros
        check64(metric, got, x, x, metric)
    x[7, 36] = np.nan
    y, _ = data64(DT.L2Expanded, 70, 1, 37, seed=3)
    for metric in (DT.L2Expanded, DT.CosineExpanded, DT.L1, DT.InnerProduct):
        got = run(metric, x, y, "f64", dtype="f64")
        assert np.isnan(got[7]).all() and np.isfinite(np.delete(got, 7, axis=0)).all()
        check64(metric, np.delete(got, 7, axis=0), np.delete(x, 7, axis=0), y, metric)


def test_fp64_gram_matrices_share_the_kernel():
    from raft_b200.distance import gram_matrix
    x, y = data64(DT.L2Expanded, 65, 63, 17, seed=5)
    x *= 0.1; y *= 0.1
    X, Y = place(x, pad=1), place(y, pad=2)
    ip = x @ y.T
    d2 = np.maximum(norms(x, y) - 2 * ip, 0)
    for kernel, kw, ref in (("linear", {}, ip), ("polynomial", {"gamma": 0.5, "coef0": 1.0, "degree": 3}, (0.5 * ip + 1.0) ** 3),
                            ("rbf", {"gamma": 0.25}, np.exp(-0.25 * d2)), ("tanh", {"gamma": 0.01, "coef0": 0.5}, np.tanh(0.01 * ip + 0.5))):
        out = Out(65, 63, torch.float64, pad=3)
        gram_matrix(X, Y, out=out.view, kernel=kernel, **kw)
        torch.cuda.synchronize()
        got = out.result()
        assert np.abs(got - ref).max() <= 1e-13 * max(1.0, np.abs(ref).max()), (kernel, float(np.abs(got - ref).max()))


# ---------------------------------------------------------------------------------------------------------------------
# 5. fp32 unexpanded kernels: the SIMT kernel's load paths and the TMA-fed kernel

UX_LAYOUTS = [
    # id, kwargs, path when k % 4 == 0 (otherwise no operand vectorises: "simt 0 0")
    ("aligned", {}, "simt-tma"),
    ("x-base-off-4-bytes", {"xoff": 1}, "simt 0 1"),
    ("y-base-off-8-bytes", {"yoff": 2}, "simt 1 0"),
    ("x-odd-ld", {"xpad": 1}, "simt 0 1"),
    ("y-ld%4=2", {"ypad": 2, "opad": 3}, "simt 1 0"),
    ("both-padded-ld%4=0", {"xpad": 4, "ypad": 8}, "simt-tma"),
    ("both-off", {"xoff": 1, "yoff": 3, "ooff": 1}, "simt 0 0"),
    ("fortran", {"order": "F"}, "simt 0 0"),
    ("fortran-padded", {"order": "F", "xpad": 3, "ypad": 4, "opad": 1}, "simt 0 0"),
]


@pytest.mark.parametrize("layout", UX_LAYOUTS, ids=[c[0] for c in UX_LAYOUTS])
@pytest.mark.parametrize("metric", oracle.UNEXPANDED, ids=[mt.name for mt in oracle.UNEXPANDED])
def test_unexpanded_load_paths(metric, layout):
    tag, kw, path = layout
    for k in (1, 3, 4, 5, 31, 32, 33, 64):
        if k == 1 and kw.get("order") == "F":
            continue                       # a single column has no memory order of its own
        x, y = data(metric, 130, 129, k, seed=k)
        got = run(metric, x, y, path if k % 4 == 0 else "simt 0 0", p=3.0, **kw)
        check32(metric, got, x, y, (tag, metric, k), p=3.0)


def test_unexpanded_fortran_order_swaps_which_operand_is_first():
    """In Fortran order the kernel's first operand is y; neither vectorises, and KLDivergence keeps its direction."""
    x, y = data(DT.KLDivergence, 140, 70, 32, seed=4)
    got = run(DT.KLDivergence, x, y, "simt 0 0", order="F", xpad=2)
    check32(DT.KLDivergence, got, x, y, "kl-fortran")
    assert not oracle.match_approx(got, oracle.pairwise_distance(y, x, DT.KLDivergence).T, EPS)[0]


@pytest.mark.parametrize("dtype,metric,path", [("f32", DT.L2Expanded, "scalar 1:0:res"), ("f32", DT.L1, "simt 0 0"),
                                               ("f64", DT.L2Expanded, "f64")])
def test_single_row_in_fortran_order(dtype, metric, path):
    """m = 1 against a Fortran-order y: the [1, n] result's pitch is its column stride (1 when contiguous), not n."""
    x, y = data(metric, 1, 130, 20, seed=1)
    ref = oracle.pairwise_distance(x, y, metric)
    for opad in (0, 2):
        got = run(metric, x, y, path, dtype=dtype, order="F", opad=opad)
        assert oracle.match_approx(got, ref, EPS)[0]
    got = pairwise_distance(place(x.astype(NP[dtype]), "F"), place(y.astype(NP[dtype]), "F"), metric=metric).copy_to_host()
    assert got.shape == (1, 130) and oracle.match_approx(got, ref, EPS)[0]


# ---------------------------------------------------------------------------------------------------------------------

TENSOR_PATHS = [(kern, acc, st) for kern, acc, sts in (("res", 0, ("tma", "vec2", "scalar")), ("res", 3, ("vec2", "scalar")),
                                                        ("str", 0, ("tma", "vec2", "scalar")), ("str", 1, ("vec2", "scalar")),
                                                        ("str", 2, ("vec2", "scalar")), ("str", 3, ("vec2", "scalar")))
                for st in sts]


@pytest.mark.parametrize("dtype", ["f32", "f16"])
def test_every_tensor_path_is_named_by_a_case(dtype):
    """The table of the module docstring: small fp32 / fp16 calls fill what the cases above did not run in this
    process (a deselected run), then every producible (kernel, acc_mode, stores) combination must have been planned."""
    x, y = data(DT.L2Expanded, 130, 132, 1024, seed=77)
    fill = [(96, 0, 0, "tma 3:0:res"), (96, 2, 0, "vec2 3:0:res"), (96, 1, 0, "scalar 3:0:res"),
            (200, 0, 0, "tma 7:0:str"), (200, 2, 0, "vec2 7:0:str"), (200, 0, 1, "scalar 7:0:str"),
            (330, 0, 0, "vec2 8:1:str 3:3:res"), (330, 1, 0, "scalar 8:1:str 3:3:res"),
            (1024, 0, 0, "vec2 8:1:str 8:2:str 8:2:str 8:3:str"), (1024, 1, 0, "scalar 8:1:str 8:2:str 8:2:str 8:3:str")]
    for k, opad, ooff, path in fill:
        xs, ys = x[:, :k].astype(NP[dtype]), y[:, :k].astype(NP[dtype])
        check32(DT.L2Expanded, run(DT.L2Expanded, xs, ys, path, dtype=dtype, opad=opad, ooff=ooff), xs, ys, path)
    missing = [c for c in TENSOR_PATHS if (dtype,) + c not in SEEN]
    assert not missing, missing
    assert {c[1:] for c in SEEN if c[0] == dtype} == set(TENSOR_PATHS)     # and the host code produces no other
