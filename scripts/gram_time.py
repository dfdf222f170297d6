"""Times gram_matrix against what it replaces, on one GPU in one process: the fused call, pairwise_distance alone at the same
shape (InnerProduct, or L2Expanded for rbf), and the composition pairwise_distance + an in-place torch transform of the
m x n result.  CUDA events around each call, after warm-up; the median of --runs.  Prints the card and its power limit
first, then one table row per case (and a JSON line per case with --json).

  python scripts/gram_time.py [--runs 5] [--warmup 2] [--json]
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from measure import card, time_ms  # noqa: E402
from raft_b200.distance import gram_matrix, pairwise_distance  # noqa: E402
from raft_b200.common import DeviceResources  # noqa: E402

PARAMS = {"linear": (0, 1.0, 0.0), "polynomial": (3, 1.0 / 128, 1.0), "rbf": (0, 1.0 / 256, 0.0), "tanh": (0, 1.0 / 128, -0.5)}


def transform(out, kernel, degree, gamma, coef0):
    """the composition's second pass, in place on the m x n result"""
    if kernel == "rbf":
        out.mul_(-gamma).exp_()
    elif kernel == "tanh":
        out.mul_(gamma).add_(coef0).tanh_()
    elif kernel == "polynomial":
        out.mul_(gamma).add_(coef0).pow_(degree)


def case(label, m, n, k, col_major, kernels, h, args, compose):
    g = torch.Generator(device="cuda").manual_seed(1)
    if col_major:
        x = torch.randn((k, m), device="cuda", generator=g).t()
        y = torch.randn((k, n), device="cuda", generator=g).t()
        out = torch.empty((n, m), device="cuda").t()
    else:
        x = torch.randn((m, k), device="cuda", generator=g)
        y = torch.randn((n, k), device="cuda", generator=g)
        out = torch.empty((m, n), device="cuda")
    rows = []
    base_ms = {}
    st = h.torch_stream   # the events go on the handle's stream, where the calls run
    with torch.cuda.stream(st):
        for kernel in kernels:
            degree, gamma, coef0 = PARAMS[kernel]
            metric = "sqeuclidean" if kernel == "rbf" else "inner_product"
            if metric not in base_ms:
                base_ms[metric] = statistics.median(time_ms(
                    lambda: pairwise_distance(x, y, out=out, metric=metric, handle=h), args.runs, args.warmup,
                    stream=st))
            fused = statistics.median(time_ms(
                lambda: gram_matrix(x, y, kernel, degree=degree, gamma=gamma, coef0=coef0, out=out, handle=h), args.runs,
                args.warmup, stream=st))
            comp = None
            if compose:
                def composition():
                    pairwise_distance(x, y, out=out, metric=metric, handle=h)
                    transform(out, kernel, degree, gamma, coef0)
                comp = statistics.median(time_ms(composition, args.runs, args.warmup, stream=st))
            r = {"shape": label, "kernel": kernel, "fused_ms": round(fused, 3), "pairwise_ms": round(base_ms[metric], 3),
                 "ratio_to_pairwise": round(fused / base_ms[metric], 3),
                 "composition_ms": None if comp is None else round(comp, 3)}
            rows.append(r)
            print("| %s | %s | %.2f | %.2f | %.3f | %s |" % (label, kernel, fused, base_ms[metric], fused / base_ms[metric],
                                                          "-" if comp is None else "%.2f" % comp), flush=True)
            if args.json:
                print(json.dumps(r), flush=True)
    del x, y, out
    torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--json", action="store_true")
    args = ap.parse_args()
    c = card()
    print("card: %s, power limit / max SM clock: %s W, %s MHz" % (c["name"], c["power_limit"], c["clocks_max_sm"]))
    print("| m x n x k | kernel | fused ms | pairwise ms | fused / pairwise | composition ms |")
    print("|---|---|---|---|---|---|")
    h = DeviceResources()
    kernels = list(PARAMS)
    case("100000 x 100000 x 128", 100000, 100000, 128, False, kernels, h, args, True)
    case("1000000 x 2048 x 64, column-major", 1000000, 2048, 64, True, kernels, h, args, True)
    case("60000 x 60000 x 784 (K-chunked)", 60000, 60000, 784, False, kernels, h, args, True)


if __name__ == "__main__":
    main()
