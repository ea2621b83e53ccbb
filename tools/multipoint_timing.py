#!/usr/bin/env python3
"""CUDA-event timing of the subproduct-tree entry points against the kernels they replace, Goldilocks, ms per call.

  multieval    ops.poly_multieval on the tree vs ops.poly_eval (one CTA per point) at d = m = 2^6 … 2^20; the direct
               kernel stops after the first size where one call exceeds --direct-cap-ms
  interpolate  the tree vs the literal interp_* kernels (g = 0) at k = 2^6 … 2^13, the tree alone up to 2^22
  from_roots   the tree vs k sequential linear products in one CTA (g = 0) at k = 2^7 … 2^13, the tree up to 2^22

The tree is forced with RONK_TREE_MIN=1 on its own context.  Each crossover printed is the smallest size measured from
which the tree is faster at every larger measured size.  The card's name and power limit are printed with the numbers."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from ronkathon_b200 import Context, ops  # noqa: E402

GL = 0xFFFFFFFF00000001


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(iters):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        out.append(s.elapsed_time(e))
        if out[-1] > 500:  # long calls: one sample is enough
            break
    return round(statistics.median(out), 4)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def crossover(rows, a, b):
    """Smallest size from which rows[size][a] < rows[size][b] at every larger size where both were measured."""
    sizes = sorted(s for s in rows if a in rows[s] and b in rows[s])
    best = None
    for s in reversed(sizes):
        if rows[s][a] < rows[s][b]:
            best = s
        else:
            break
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--direct-cap-ms", type=float, default=2000.0)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    stream = torch.cuda.current_stream().cuda_stream
    ctx = Context(0, stream)
    os.environ["RONK_TREE_MIN"] = "1"
    tree = Context(0, stream)
    del os.environ["RONK_TREE_MIN"]
    res = {"card": card()}

    ev, direct_on = {}, True
    for lg in range(6, 21):
        n = 1 << lg
        f, xs = ops.splitmix_fill(ctx, n, 1, GL), ops.splitmix_fill(ctx, n, 2, GL)
        ev[n] = {"tree": timed(lambda: ops.poly_multieval(tree, f, xs), args.iters)}
        if direct_on:
            ev[n]["direct"] = timed(lambda: ops.poly_eval(ctx, f, xs), args.iters)
            direct_on = ev[n]["direct"] <= args.direct_cap_ms
        del f, xs
    res["multieval_ms"] = ev
    res["multieval_crossover"] = crossover(ev, "tree", "direct")

    it = {}
    for lg in range(6, 23):
        k = 1 << lg
        xs, ys = ops.splitmix_fill(ctx, k, 3, GL), ops.splitmix_fill(ctx, k, 4, GL)
        it[k] = {"tree": timed(lambda: ops.poly_interpolate(tree, xs, ys), args.iters)}
        if k <= 8192:
            it[k]["literal"] = timed(lambda: ops.poly_interpolate(ctx, xs, ys, g=0), args.iters)
        del xs, ys
    res["interpolate_ms"] = it
    res["interpolate_crossover"] = crossover(it, "tree", "literal")

    fr = {}
    for lg in range(7, 23):
        k = 1 << lg
        xs = ops.splitmix_fill(ctx, k, 5, GL)
        fr[k] = {"tree": timed(lambda: ops.poly_from_roots(tree, xs), args.iters)}
        if k <= 8192:
            fr[k]["linear"] = timed(lambda: ops.poly_from_roots(ctx, xs, g=0), args.iters)
        del xs
    res["from_roots_ms"] = fr
    res["from_roots_crossover"] = crossover(fr, "tree", "linear")
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
