#!/usr/bin/env python3
"""Timing of ronk_poly_divrem_batch_u64 (poly.cu / poly_div.cu), ms per call: the median of --iters calls after one warm
call, the host clock around each call (the call is synchronous).

Over Goldilocks (g = 7, the Goldilocks policy) and BabyBear (g = 31, the Montgomery policy) at da ∈ {2^6, 2^8, 2^10, 2^12, 2^16, 2^20}, db ∈ {2, 17, da/2 + 1}, a shared divisor and one
divisor per row, batch ∈ {1, 2, 16, 256, 4096} capped at 2^28 words per call (--primes, --da and --batches narrow the
sweep), four timings per shape:
  literal  the batched call on a context made with RONK_DIVREM_BATCH_PATH=1,
  newton   the same with RONK_DIVREM_BATCH_PATH=2,
  default  the measured rule,
  loop     one ronk_poly_divrem_u64 call per row.
The literal kernel takes about L = da - db + 1 sequential steps of about da/256 words per thread each: where L·da passes
--literal-max it is not timed ("-"), nor is a loop of more than --loop-max rows (its time per row is that of 256 rows).
Each line names the path the rule took and whether it is the faster of literal and newton, or within 2 % of it.  With
--json the rows go to that file as JSON lines.  The card's name and power limit are printed with the numbers."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from ronkathon_b200 import Context, _lib, ops  # noqa: E402

GL = 0xFFFFFFFF00000001
PRIMES = {"goldilocks": (GL, 7), "babybear": (2013265921, 31)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(iters):
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t) * 1e3)
    return statistics.median(out)


def forced(path):
    os.environ["RONK_DIVREM_BATCH_PATH"] = str(path)
    try:
        return Context(0, torch.cuda.current_stream().cuda_stream)
    finally:
        del os.environ["RONK_DIVREM_BATCH_PATH"]


def rand(n, seed, p):
    g = np.random.default_rng(seed)
    return (g.integers(0, 1 << 63, n, dtype=np.uint64) * 2 + g.integers(0, 2, n, dtype=np.uint64)) % np.uint64(p)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--literal-max", type=float, default=2.0 ** 28)
    ap.add_argument("--loop-max", type=int, default=256)
    ap.add_argument("--max-words", type=int, default=1 << 28)
    ap.add_argument("--json", default="")
    ap.add_argument("--primes", default="goldilocks,babybear")
    ap.add_argument("--da", default="6,8,10,12,16,20", help="log2 da values")
    ap.add_argument("--batches", default="1,2,16,256,4096")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    print(f"# {card()}")
    ctx = Context(0, torch.cuda.current_stream().cuda_stream)
    lit, newt = forced(1), forced(2)
    sink = open(args.json, "w") if args.json else None
    for name in args.primes.split(","):
        sweep(name, *PRIMES[name], ctx, lit, newt, sink, args)
    print(f"# {card()}")


def sweep(name, p, g, ctx, lit, newt, sink, args):
    print(f"# {name}: p = {p}, g = {g}")
    print(f"{'da':>8} {'db':>8} {'b':>5} {'batch':>5} {'literal':>9} {'newton':>9} {'default':>9} {'loop':>9}  rule")
    for lda in (int(v) for v in args.da.split(",")):
        da = 1 << lda
        for db in sorted({2, 17, da // 2 + 1}):
            L = da - db + 1
            for batch in (int(v) for v in args.batches.split(",")):
                if batch * da > args.max_words:
                    continue
                A = ops.to_device(rand(batch * da, lda * 7 + db, p).reshape(batch, da))
                Bn = rand(batch * db, db + 3, p).reshape(batch, db)
                Bn[:, -1] = Bn[:, -1] % np.uint64(p - 1) + np.uint64(1)
                for shared in (True, False):
                    B = ops.to_device(Bn[0] if shared else Bn)
                    row = {"prime": name, "da": da, "db": db, "shared": shared, "batch": batch}
                    if L * da <= args.literal_max:
                        row["literal"] = timed(lambda: ops.poly_divrem_batch(lit, A, B, p=p, g=g), args.iters)
                    row["newton"] = timed(lambda: ops.poly_divrem_batch(newt, A, B, p=p, g=g), args.iters)
                    row["default"] = timed(lambda: ops.poly_divrem_batch(ctx, A, B, p=p, g=g), args.iters)
                    n = min(batch, args.loop_max)
                    q, r = torch.empty_like(A[0]), torch.empty_like(A[0])

                    def loop():
                        for y in range(n):
                            by = B if shared else B[y]
                            ctx.call("ronk_poly_divrem_u64", p, g, _lib._ptr(A[y]), da, _lib._ptr(by), db, _lib._ptr(q),
                                     _lib._ptr(r))
                    row["loop"] = timed(loop, 1) * batch / n
                    ctx.prof_fetch()
                    ctx.prof_enable(True)
                    ops.poly_divrem_batch(ctx, A, B, p=p, g=g)
                    ctx.sync()
                    ctx.prof_enable(False)
                    names = [nm for nm, _ in ctx.prof_fetch()]
                    rule = ("literal" if "poly_divrem_rows" in names or "poly_divrem" in names else
                            "linear" if "div_linear_apply" in names else "newton")
                    row["rule"] = rule
                    best = min(row.get("literal", float("inf")), row["newton"])
                    ok = rule == "linear" or batch == 1 or row.get(rule, float("inf")) <= 1.02 * best
                    row["rule_ok"] = ok
                    f = lambda k: f"{row[k]:9.3f}" if k in row else f"{'-':>9}"  # noqa: E731
                    print(f"{da:8d} {db:8d} {'s' if shared else 'r':>5} {batch:5d} {f('literal')} {f('newton')} {f('default')} "
                          f"{f('loop')}  {rule}{'' if ok else '  <-- not the faster path'}", flush=True)
                    if sink:
                        sink.write(json.dumps(row) + "\n")
                del A


if __name__ == "__main__":
    main()
