#!/usr/bin/env python3
"""CUDA-event timing of ronk_ntt_any_u64 on Goldilocks, ms per call (median of --iters calls after one warm call).

For n ∈ {3, 5, 15, 17, 255, 257} × 2^k up to 2^25 it times Bluestein (forced with RONK_ANYNTT_MIN=1 on its own
context), the literal O(n²) kernels (forced with RONK_ANYNTT_MIN=2^30, while one call stays under --literal-cap-ms) and
the power-of-two transform of N = 2^⌈log2(2n - 1)⌉ points that Bluestein runs two of.  The crossover printed is the
smallest n from which Bluestein wins at every larger n measured.  The card's name and power limit are printed with the
numbers."""
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


def context(stream, min_n):
    os.environ["RONK_ANYNTT_MIN"] = str(min_n)
    try:
        return Context(0, stream)
    finally:
        del os.environ["RONK_ANYNTT_MIN"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--literal-cap-ms", type=float, default=1000.0)
    ap.add_argument("--max-log", type=int, default=25)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    stream = torch.cuda.current_stream().cuda_stream
    plain, blue, lit = Context(0, stream), context(stream, 1), context(stream, 1 << 30)
    rows = {}
    for odd in (3, 5, 15, 17, 255, 257):
        literal_on = True
        k = 0
        while odd << k < 1 << args.max_log:
            n = odd << k
            k += 1
            log_N = (2 * n - 2).bit_length()
            x = ops.splitmix_fill(plain, n, 1, GL)
            y = ops.splitmix_fill(plain, 1 << log_N, 2, GL)
            r = {"N": 1 << log_N,
                 "bluestein": timed(lambda: ops.ntt_any_(blue, x, n), args.iters),
                 "pow2_N": timed(lambda: ops.ntt_(plain, y, log_N), args.iters)}
            if literal_on and n <= 1 << 17:
                r["literal"] = timed(lambda: ops.ntt_any_(lit, x, n), args.iters)
                literal_on = r["literal"] <= args.literal_cap_ms
            r["bluestein_over_pow2_N"] = round(r["bluestein"] / r["pow2_N"], 2)
            rows[n] = r
            del x, y
            print(n, r, file=sys.stderr, flush=True)
    sizes = sorted(n for n in rows if "literal" in rows[n])
    best = None
    for n in reversed(sizes):
        if rows[n]["bluestein"] < rows[n]["literal"]:
            best = n
        else:
            break
    print(json.dumps({"card": card(), "ms": {str(n): rows[n] for n in sorted(rows)}, "crossover": best}, indent=1))


if __name__ == "__main__":
    main()
