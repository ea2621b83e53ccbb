#!/usr/bin/env python3
"""CUDA-event timing of ronk_poly_divrem_u64 (ops.poly_divrem) on Goldilocks, ms per call.

For each (da, db) it reports the call time with profiling off (median of --iters calls after a warm-up), then, from one
profiled call, the share of kernel time spent in the transform kernels and the number of launches.  One 2^24-point
transform is timed in the same run, so the division can be stated in transforms, and the literal single-CTA kernel
(g = 0) is timed at a size where it finishes.  The card's name and power limit are printed with the numbers."""
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
SIZES = [(1 << 16, (1 << 15) + 1), (1 << 20, (1 << 19) + 1), (1 << 24, (1 << 23) + 1), (1 << 24, (1 << 12) + 1)]


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
    return round(statistics.median(out), 4), round(min(out), 4), round(max(out), 4)


def is_transform(name):
    return "ntt" in name  # ntt3_*, intt3_*, ntt_single, ntt_pass*, ntt16_cluster, …


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    ctx = Context(0, torch.cuda.current_stream().cuda_stream)
    res = {"card": card()}
    x = ops.splitmix_fill(ctx, 1 << 24, 1, GL)
    res["ntt_2^24_ms"] = timed(lambda: ops.ntt_(ctx, x, 24), args.iters)[0]
    del x
    for da, db in SIZES:
        a, b = ops.splitmix_fill(ctx, da, 2, GL), ops.splitmix_fill(ctx, db, 3, GL)
        b[-1] = 5
        med, lo, hi = timed(lambda: ops.poly_divrem(ctx, a, b), args.iters)
        ctx.prof_fetch()
        ctx.prof_enable(True)
        ops.poly_divrem(ctx, a, b)
        recs = ctx.prof_fetch()
        ctx.prof_enable(False)
        total = sum(ms for _, ms in recs)
        ntt = sum(ms for n, ms in recs if is_transform(n))
        res[f"divrem_{da}_{db}"] = {"ms": med, "min": lo, "max": hi, "in_2^24_transforms": round(med / res["ntt_2^24_ms"], 1),
                                    "transform_share_of_kernel_time": round(ntt / total, 3), "launches": len(recs)}
        del a, b
    da, db = 1 << 12, (1 << 11) + 1
    a, b = ops.splitmix_fill(ctx, da, 4, GL), ops.splitmix_fill(ctx, db, 5, GL)
    b[-1] = 5
    res[f"literal_g0_{da}_{db}"] = {"ms": timed(lambda: ops.poly_divrem(ctx, a, b, g=0), 3)[0]}
    res[f"newton_{da}_{db}"] = {"ms": timed(lambda: ops.poly_divrem(ctx, a, b), args.iters)[0]}
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
