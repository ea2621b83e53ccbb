#!/usr/bin/env python3
"""CUDA-event timing of the coset transforms and the LDE (ntt_coset.cu), ms per call: the median of --iters calls
after one warm call, the variants of one shape interleaved call by call so that they see the same clocks.

1. Forward and inverse coset transforms against the plain ronk_ntt_u64 of the same shape, and against the unfused
   three-call route (ronk_field_powers_u64, ronk_field_mul_u64, ronk_ntt_u64), for Goldilocks (g = 7) and BabyBear at
   2^14, 2^16, 2^20, 2^22 and 2^24, at batch 1 and at the batch that fills 2^24 words.
2. The LDE from 2^20 to 2^22 and from 2^21 to 2^24 coefficients, with each launch's share of one profiled call (the pad
   kernel against the transform).

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

GL, BB = 0xFFFFFFFF00000001, 2013265921
FIELDS = {"goldilocks": (GL, 7), "babybear": (BB, 31)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def interleaved(fns, iters):
    """{name: median ms} of the callables in fns, called in turn, each once per round."""
    for fn in fns.values():
        fn()
    torch.cuda.synchronize()
    samples = {k: [] for k in fns}
    for _ in range(iters):
        for k, fn in fns.items():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn()
            e.record()
            torch.cuda.synchronize()
            samples[k].append(s.elapsed_time(e))
    return {k: round(statistics.median(v), 4) for k, v in samples.items()}


def transforms(ctx, iters):
    for name, (p, g) in FIELDS.items():
        for log_n in (14, 16, 20, 22, 24):
            for batch in sorted({1, 1 << (24 - log_n)}):
                n = batch << log_n
                a = ops.splitmix_fill(ctx, n, 1, p)
                pw = torch.empty(1 << log_n, dtype=torch.int64, device="cuda")
                factor, full = torch.empty_like(a), torch.empty_like(a)
                s = 3 if name == "babybear" else 5

                def three_call():
                    # the factor of every row, as a user without the fused call builds it: powers, then one multiply
                    ctx.call("ronk_field_powers_u64", p, s, 1, pw.data_ptr(), 1 << log_n)
                    factor.view(batch, -1).copy_(pw.expand(batch, -1))
                    ctx.call("ronk_field_mul_u64", p, a.data_ptr(), factor.data_ptr(), full.data_ptr(), n)
                    ops.ntt_(ctx, full, log_n, batch=batch, p=p, g=g)

                t = interleaved({
                    "plain_fwd": lambda: ops.ntt_(ctx, a, log_n, batch=batch, p=p, g=g),
                    "coset_fwd": lambda: ops.ntt_coset_(ctx, a, log_n, s, batch=batch, p=p, g=g),
                    "plain_inv": lambda: ops.ntt_(ctx, a, log_n, batch=batch, inverse=True, p=p, g=g),
                    "coset_inv": lambda: ops.ntt_coset_(ctx, a, log_n, s, batch=batch, inverse=True, p=p, g=g),
                    "three_call_fwd": three_call,
                }, iters)
                t.update(field=name, log_n=log_n, batch=batch,
                         coset_over_plain_fwd=round(t["coset_fwd"] / t["plain_fwd"], 3),
                         coset_over_plain_inv=round(t["coset_inv"] / t["plain_inv"], 3),
                         coset_over_three_call=round(t["coset_fwd"] / t["three_call_fwd"], 3))
                print(json.dumps(t), flush=True)


def lde(ctx, iters):
    for log_d, log_n in ((20, 22), (21, 24)):
        c = ops.splitmix_fill(ctx, 1 << log_d, 2, GL)
        t = interleaved({"lde": lambda: ops.lde(ctx, c, log_n, 7)}, iters)
        ctx.sync()
        ctx.prof_fetch()
        ctx.prof_enable(True)
        ops.lde(ctx, c, log_n, 7)
        recs = ctx.prof_fetch()
        ctx.prof_enable(False)
        total = sum(ms for _, ms in recs)
        t.update(field="goldilocks", d=1 << log_d, N=1 << log_n,
                 launches={n: round(ms, 4) for n, ms in recs},
                 pad_share=round(sum(ms for n, ms in recs if n == "lde_pad") / total, 3))
        print(json.dumps(t), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    ctx = Context(0, torch.cuda.current_stream().cuda_stream)
    print(json.dumps({"card": card()}), flush=True)
    transforms(ctx, args.iters)
    lde(ctx, args.iters)


if __name__ == "__main__":
    main()
