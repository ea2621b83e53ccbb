#!/usr/bin/env python3
"""CUDA-event timing of the batched multipoint entry points against a loop of single-row calls, Goldilocks, ms per call.

  batched vs loop   ops.poly_multieval_batch / poly_interpolate_batch at batch 1, 16, 256 with m = d = 2^12, 2^16, 2^20
                    (shapes past the 2^32-word cap are skipped), against the same rows through ops.poly_multieval /
                    poly_interpolate one at a time; the two are timed alternately, --reps times each, in one process, and
                    their outputs must agree word for word
  crossover         at each of --cross-batches, the tree (RONK_TREE_MIN=1) against the literal kernels (g = 0) and the
                    default context's choice: multieval at m = d = 2^10 … 2^16, interpolation at k = 2^8 … 2^13

The default context runs the path rule as shipped.  Each crossover printed is the smallest size measured from which the
tree is faster at every larger measured size.  The card's name and power limit are printed with the numbers."""
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
    return statistics.median(out)


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


def distinct_points(ctx, n, seed):
    xs = ops.splitmix_fill(ctx, n + 64, seed, GL)
    u = torch.unique(xs)   # int64 order; the points only need to be distinct
    assert u.numel() >= n
    return u[:n].contiguous()


def batched_vs_loop(ctx, batch, lg, reps, iters):
    n = 1 << lg
    xs = distinct_points(ctx, n, 1)
    f = ops.splitmix_fill(ctx, batch * n, 2, GL).view(batch, n)
    row = {}
    ev_b = ops.poly_multieval_batch(ctx, f, xs)
    ev_l = torch.stack([ops.poly_multieval(ctx, f[b], xs) for b in range(batch)])
    it_b = ops.poly_interpolate_batch(ctx, xs, ev_b)
    it_l = torch.stack([ops.poly_interpolate(ctx, xs, ev_b[b]) for b in range(batch)])
    ctx.sync()
    assert torch.equal(ev_b, ev_l) and torch.equal(it_b, it_l) and torch.equal(it_b, f), f"outputs differ at {batch} × 2^{lg}"
    del ev_l, it_b, it_l
    samples = {k: [] for k in ("multieval_batched", "multieval_loop", "interpolate_batched", "interpolate_loop")}
    for _ in range(reps):
        samples["multieval_batched"].append(timed(lambda: ops.poly_multieval_batch(ctx, f, xs), iters))
        samples["multieval_loop"].append(timed(lambda: [ops.poly_multieval(ctx, f[b], xs) for b in range(batch)], iters))
        samples["interpolate_batched"].append(timed(lambda: ops.poly_interpolate_batch(ctx, xs, ev_b), iters))
        samples["interpolate_loop"].append(timed(lambda: [ops.poly_interpolate(ctx, xs, ev_b[b]) for b in range(batch)],
                                                 iters))
    for k, v in samples.items():
        row[k] = round(statistics.median(v), 4)
        row[k + "_spread"] = round(max(v) - min(v), 4)
    row["multieval_speedup"] = round(row["multieval_loop"] / row["multieval_batched"], 2)
    row["interpolate_speedup"] = round(row["interpolate_loop"] / row["interpolate_batched"], 2)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batches", default="1,16,256")
    ap.add_argument("--logs", default="12,16,20")
    ap.add_argument("--cross-batches", default="1,2,16,256", help="batches of the tree-against-literal sweep")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    stream = torch.cuda.current_stream().cuda_stream
    ctx = Context(0, stream)
    os.environ["RONK_TREE_MIN"] = "1"
    tree = Context(0, stream)
    del os.environ["RONK_TREE_MIN"]
    res = {"card": card(), "batched_vs_loop_ms": {}}

    for batch in (int(b) for b in args.batches.split(",")):
        for lg in (int(v) for v in args.logs.split(",")):
            if batch << (lg + 1) > 1 << 32:   # the root's 2^⌈log2(2d - 1)⌉ words per row
                continue
            res["batched_vs_loop_ms"][f"{batch}x2^{lg}"] = batched_vs_loop(ctx, batch, lg, args.reps, args.iters)
            torch.cuda.empty_cache()

    for batch in (int(b) for b in args.cross_batches.split(",")):
        ev, it = {}, {}
        for lg in range(10, 17):
            n = 1 << lg
            xs, f = distinct_points(ctx, n, 3), ops.splitmix_fill(ctx, batch * n, 4, GL).view(batch, n)
            ev[n] = {"tree": timed(lambda: ops.poly_multieval_batch(tree, f, xs), args.iters),
                     "literal": timed(lambda: ops.poly_multieval_batch(ctx, f, xs, g=0), args.iters),
                     "default": timed(lambda: ops.poly_multieval_batch(ctx, f, xs), args.iters)}
        for lg in range(8, 14):
            k = 1 << lg
            xs, ys = distinct_points(ctx, k, 5), ops.splitmix_fill(ctx, batch * k, 6, GL).view(batch, k)
            it[k] = {"tree": timed(lambda: ops.poly_interpolate_batch(tree, xs, ys), args.iters),
                     "literal": timed(lambda: ops.poly_interpolate_batch(ctx, xs, ys, g=0), args.iters),
                     "default": timed(lambda: ops.poly_interpolate_batch(ctx, xs, ys), args.iters)}
        res[f"crossover_batch{batch}_multieval_ms"] = {n: {k: round(v, 4) for k, v in r.items()} for n, r in ev.items()}
        res[f"crossover_batch{batch}_multieval"] = crossover(ev, "tree", "literal")
        res[f"crossover_batch{batch}_interpolate_ms"] = {n: {k: round(v, 4) for k, v in r.items()} for n, r in it.items()}
        res[f"crossover_batch{batch}_interpolate"] = crossover(it, "tree", "literal")
        torch.cuda.empty_cache()
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
