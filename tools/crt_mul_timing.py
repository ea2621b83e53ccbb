#!/usr/bin/env python3
"""CUDA-event timing of ronk_poly_mul_u64's multi-modular path (poly_crt.cu), ms per call (median of --iters calls after
one warm call).

1. Schoolbook against the multi-modular path at da = db = 2^6 … 2^16, on one prime per prime count: 101 (k = 1), 2^31 - 1
   and p32 = 4295294977 (k = 2; p32's own transforms fit up to 2^16 points, so below da = 2^16 both contexts take them),
   and 2^64 - 279 (k = 3).  The schoolbook kernel is forced with RONK_CRT_MUL_MIN=2^62, the multi-modular path with
   RONK_CRT_MUL_MIN=1, each on its own context.  Each crossover printed is the smallest da·db from which the
   multi-modular path wins at every larger size measured.
2. Unbalanced shapes: da = 2^0 … 2^12 against db = 2^16, 2^20 and 2^24 on the same primes (2^31 - 1 for k = 2).  The
   schoolbook kernel does min(da, db) multiplies per coefficient, the multi-modular path about k·log2(L) whatever the
   shape, so the shorter operand decides.  Each short-side crossover printed is the smallest da from which the
   multi-modular path wins at every larger da measured, for every db.
3. The multi-modular path at 2^23 × 2^23 for each k next to the Goldilocks product of the same size (its own transforms),
   with the kernel split of one profiled call.

The card's name and power limit are printed with the numbers."""
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
PRIMES = {"f101": (101, 2, 1), "m31": ((1 << 31) - 1, 7, 2), "p32": (4295294977, 5, 2), "2^64-279": ((1 << 64) - 279, 5, 3)}


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


def context(stream, crt_min):
    os.environ["RONK_CRT_MUL_MIN"] = str(crt_min)
    try:
        return Context(0, stream)
    finally:
        del os.environ["RONK_CRT_MUL_MIN"]


def split(c, fn):
    """ms per kernel name of one profiled call."""
    torch.cuda.synchronize()
    c.prof_fetch()
    c.prof_enable(True)
    try:
        fn()
        rows = c.prof_fetch()
    finally:
        c.prof_enable(False)
    out = {}
    for name, ms in rows:
        out[name] = round(out.get(name, 0.0) + ms, 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--max-log", type=int, default=16)
    ap.add_argument("--big-log", type=int, default=23)
    ap.add_argument("--skew-iters", type=int, default=5)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    stream = torch.cuda.current_stream().cuda_stream
    school, crt = context(stream, 1 << 62), context(stream, 1)
    result = {"card": card(), "ms": {}, "crossover_da_db": {}}
    for name, (p, g, k) in PRIMES.items():
        rows = {}
        for lg in range(6, args.max_log + 1):
            a, b = ops.splitmix_fill(crt, 1 << lg, 1, p), ops.splitmix_fill(crt, 1 << lg, 2, p)
            r = {"schoolbook": timed(lambda: ops.poly_mul(school, a, b, p, g), args.iters),
                 "crt": timed(lambda: ops.poly_mul(crt, a, b, p, g), args.iters)}
            rows[lg] = r
            print(name, lg, r, file=sys.stderr, flush=True)
        best = None
        for lg in sorted(rows, reverse=True):
            if rows[lg]["crt"] < rows[lg]["schoolbook"]:
                best = 1 << (2 * lg)
            else:
                break
        result["ms"][name] = {f"2^{lg}": rows[lg] for lg in sorted(rows)}
        result["crossover_da_db"][name] = best
    result["ms_unbalanced"], result["crossover_short_side"] = {}, {}
    for name in ("f101", "m31", "2^64-279"):
        p, g, k = PRIMES[name]
        per_db, worst = {}, 1
        for ldb in (16, 20, 24):
            b = ops.splitmix_fill(crt, 1 << ldb, 5, p)
            rows = {}
            for lda in range(0, 13):
                a = ops.splitmix_fill(crt, 1 << lda, 6, p)
                rows[lda] = {"schoolbook": timed(lambda: ops.poly_mul(school, a, b, p, g), args.skew_iters),
                             "crt": timed(lambda: ops.poly_mul(crt, a, b, p, g), args.skew_iters)}
                print(name, f"2^{lda} x 2^{ldb}", rows[lda], file=sys.stderr, flush=True)
            best = None
            for lda in sorted(rows, reverse=True):
                if rows[lda]["crt"] < rows[lda]["schoolbook"]:
                    best = 1 << lda
                else:
                    break
            per_db[f"2^{ldb}"] = {"ms": {f"2^{l}": rows[l] for l in sorted(rows)}, "crossover_da": best}
            worst = max(worst, best or (1 << 13))
            del b
        result["ms_unbalanced"][name] = per_db
        result["crossover_short_side"][name] = worst
    n = 1 << args.big_log
    big = {}
    for name, (p, g, k) in list(PRIMES.items()) + [("goldilocks", (GL, 7, 0))]:
        if name == "p32":
            continue
        a, b = ops.splitmix_fill(crt, n, 3, p), ops.splitmix_fill(crt, n, 4, p)
        fn = lambda: ops.poly_mul(crt, a, b, p, g)  # noqa: E731
        big[name] = {"k": k, "ms": timed(fn, args.iters), "kernels_ms": split(crt, fn)}
        print(name, big[name], file=sys.stderr, flush=True)
        del a, b
    result[f"2^{args.big_log}x2^{args.big_log}"] = big
    print(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
