#!/usr/bin/env python3
"""CUDA-event timing of ronk_rs_decode_at_u64 on Goldilocks: ms per batched call (median of --iters calls after one warm
call), rows per second, and the kernel split of one profiled call (ronk_prof: ms per kernel name, summed).

Cases (each row the evaluations of a seeded message with `errors` positions changed, so every row decodes):
  - shamir: 2^16 secrets, n = 64 shares at x = 1..64, threshold k = 32, 16 wrong shares per row;
  - tree: 256 rows, n = 4096 seeded distinct points, n - k = 2048, a full radius of errors;
  - cap: 8 rows, n = 2^16 seeded distinct points, n - k = RONK_RS_MAX_PARITY, a full radius of errors;
  - omega_tree, omega_cap: the last two shapes at x_i = ω_n^i through ronk_rs_decode_u64, to state what arbitrary
    points cost.
The card's name and power limit are read in the same run and printed with the numbers."""
import argparse
import json
import os
import statistics
import subprocess
import sys
from collections import defaultdict

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from ronkathon_b200 import Context, ops  # noqa: E402

GL = 0xFFFFFFFF00000001
GL_M1 = -0xFFFFFFFF   # p - 1 as the int64 torch stores
CAP = 8191            # RONK_RS_MAX_PARITY
# name, n, k, batch, errors, points ("shamir": 1..n, "random": seeded distinct, "omega": ronk_rs_decode_u64)
CASES = [("shamir", 64, 32, 1 << 16, 16, "shamir"), ("tree", 4096, 2048, 256, 1024, "random"),
         ("cap", 1 << 16, (1 << 16) - CAP, 8, CAP // 2, "random"), ("omega_tree", 4096, 2048, 256, 1024, "omega"),
         ("omega_cap", 1 << 16, (1 << 16) - CAP, 8, CAP // 2, "omega")]


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
    return statistics.median(out)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def received(c, n, k, batch, errors, points, seed):
    """(xs or None, messages, rows): batch seeded messages evaluated at the points, `errors` distinct positions per row
    changed (v → v + 1 mod p)."""
    msg = ops.splitmix_fill(c, batch * k, seed, GL)
    if points == "omega":
        xs, cw = None, ops.rs_encode(c, msg, n, batch).view(batch, n)
    else:
        xs = torch.arange(1, n + 1, dtype=torch.int64, device="cuda") if points == "shamir" else ops.splitmix_fill(c, n, seed + 1, GL)
        assert torch.unique(xs).numel() == n
        cw = ops.poly_multieval_batch(c, msg.view(batch, k), xs)
    g = torch.Generator(device="cuda").manual_seed(seed)
    pos = torch.argsort(torch.rand(batch, n, device="cuda", generator=g), dim=1)[:, :errors]
    v = cw.gather(1, pos)
    cw.scatter_(1, pos, torch.where(v == GL_M1, torch.zeros_like(v), v + 1))
    return xs, msg, cw.reshape(-1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--cases", default=",".join(c[0] for c in CASES))
    args = ap.parse_args()
    torch.cuda.set_device(0)
    c = Context(0, torch.cuda.current_stream().cuda_stream)
    res = {}
    for name, n, k, batch, errors, points in CASES:
        if name not in args.cases.split(","):
            continue
        xs, msg, rx = received(c, n, k, batch, errors, points, 1)
        if xs is None:
            run = lambda: ops.rs_decode(c, rx, k, None, batch)  # noqa: E731
        else:
            run = lambda: ops.rs_decode_at(c, xs, rx, k, None, batch)  # noqa: E731
        out, st = run()
        torch.cuda.synchronize()
        assert torch.equal(out, msg) and bool((st == errors).all()), name
        ms = timed(run, args.iters)
        c.prof_enable(True)
        run()
        split = defaultdict(float)
        for nm, t in c.prof_fetch():
            split[nm] += t
        c.prof_enable(False)
        res[name] = {"n": n, "k": k, "batch": batch, "errors_per_row": errors, "points": points, "ms": round(ms, 4),
                     "rows_per_s": round(batch / ms * 1e3), "kernels_ms": {nm: round(t, 4) for nm, t in split.items()}}
        print(name, res[name], file=sys.stderr, flush=True)
        del xs, msg, rx, out, st
    print(json.dumps({"card": card(), "cases": res}, indent=1))
    c.close()


if __name__ == "__main__":
    main()
