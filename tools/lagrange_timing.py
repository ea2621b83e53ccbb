#!/usr/bin/env python3
"""CUDA-event timing of the Lagrange-basis evaluation and opening on a coset (poly_bary.cu), ms per call: the median of
--iters calls after one warm call, the variants of one shape interleaved call by call so that they see the same clocks.

For Goldilocks (g = 7) on the coset 7·H_n, n = 2^16 … 2^24, batch 1, 16 and 256 (up to 2^30 words of evaluations) and
m = 1, 2 and 8 points:
  eval   ops.lagrange_eval, against the route without it: a copy, the inverse coset transform, then ronk_poly_eval_u64 per
         row (batch ≤ 16);
  open   ops.lagrange_open at a point off the coset and at a node, against the route: a copy, the inverse coset
         transform, then per row ronk_poly_eval_u64 (the value), ronk_poly_div_linear_u64 by X - z and the forward coset
         transform of the quotient (batch ≤ 16).
For m = 1 the achieved rate 8·batch·n bytes per call is printed against the H100 SXM's 3.35 TB/s.  The single-point
ronk_poly_lagrange_eval_u64_host (O(n²) in one CTA) is timed once at 2^14 and 2^16.

The card's name and power limit are printed with the numbers."""
import argparse
import ctypes as C
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
from ronkathon_b200 import Context, ops  # noqa: E402

GL, S = 0xFFFFFFFF00000001, 7
HBM = 3.35e12


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


def shapes(log_n, batch, m, ctx, iters):
    n = 1 << log_n
    rows = ops.splitmix_fill(ctx, batch * n, log_n, GL).view(batch, n)
    xs = ops.splitmix_fill(ctx, m, 99, GL)
    w = pow(7, (GL - 1) // n, GL)
    z_off, z_on = 12345, S * pow(w, 5, GL) % GL
    fns = {
        "eval": lambda: ops.lagrange_eval(ctx, rows, xs, n, shift=S),
    }
    if m == 1:
        fns["open_off"] = lambda: ops.lagrange_open(ctx, rows, z_off, n, shift=S)
        fns["open_on"] = lambda: ops.lagrange_open(ctx, rows, z_on, n, shift=S)
    if batch <= 16:
        coeffs = torch.empty_like(rows)
        q = torch.empty(n, dtype=torch.int64, device="cuda")
        rem = torch.empty(1, dtype=torch.int64, device="cuda")
        zt = torch.tensor([z_off], dtype=torch.int64, device="cuda")

        def route_eval():
            coeffs.copy_(rows)
            ops.ntt_coset_(ctx, coeffs.view(-1), log_n, S, batch=batch, inverse=True)
            for b in range(batch):
                ops.poly_eval(ctx, coeffs[b], xs)

        def route_open():
            coeffs.copy_(rows)
            ops.ntt_coset_(ctx, coeffs.view(-1), log_n, S, batch=batch, inverse=True)
            for b in range(batch):
                ops.poly_eval(ctx, coeffs[b], zt)
                ctx.call("ronk_poly_div_linear_u64", GL, coeffs[b].data_ptr(), n, GL - z_off, 1, q.data_ptr(), rem.data_ptr())
                ops.ntt_coset_(ctx, q, log_n, S)

        fns["route_eval"] = route_eval
        if m == 1:
            fns["route_open"] = route_open
    t = interleaved(fns, iters)
    t.update(field="goldilocks", log_n=log_n, batch=batch, m=m)
    if "route_eval" in t:
        t["eval_speedup"] = round(t["route_eval"] / t["eval"], 2)
    if "route_open" in t:
        t["open_speedup"] = round(t["route_open"] / t["open_off"], 2)
    if m == 1:
        for k in ("eval", "open_off"):
            t[f"{k}_TBps"] = round(8 * batch * n / (t[k] * 1e-3) / 1e12, 3)
            t[f"{k}_of_hbm"] = round(8 * batch * n / (t[k] * 1e-3) / HBM, 3)
    print(json.dumps(t), flush=True)
    ctx.sync()
    ctx.prof_fetch()
    ctx.prof_enable(True)
    ops.lagrange_eval(ctx, rows, xs, n, shift=S)
    if m == 1:
        ops.lagrange_open(ctx, rows, z_on, n, shift=S)
    recs = ctx.prof_fetch()
    ctx.prof_enable(False)
    print(json.dumps({"log_n": log_n, "batch": batch, "m": m, "launches": [[k, round(v, 4)] for k, v in recs]}), flush=True)
    del rows, fns
    torch.cuda.empty_cache()


def host_twin(ctx):
    for log_n in (14, 16):
        n = 1 << log_n
        y = np.arange(1, n + 1, dtype=np.uint64)
        res = C.c_uint64()
        ctx.call("ronk_poly_lagrange_eval_u64_host", GL, 7, y.ctypes.data_as(C.c_void_p), n, 12345, C.byref(res))
        t0 = time.perf_counter()
        ctx.call("ronk_poly_lagrange_eval_u64_host", GL, 7, y.ctypes.data_as(C.c_void_p), n, 12345, C.byref(res))
        host_ms = (time.perf_counter() - t0) * 1e3
        yt = ops.to_device(y).view(1, n)
        xt = ops.to_device(np.array([12345], dtype=np.uint64))
        t = interleaved({"eval": lambda: ops.lagrange_eval(ctx, yt, xt, n)}, 10)
        print(json.dumps({"host_twin_ms_wall": round(host_ms, 3), "eval": t["eval"], "log_n": log_n, "batch": 1, "m": 1}),
              flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--max-words", type=int, default=1 << 30)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    ctx = Context(0, torch.cuda.current_stream().cuda_stream)
    print(json.dumps({"card": card()}), flush=True)
    host_twin(ctx)
    for log_n in (16, 18, 20, 22, 24):
        for batch in (1, 16, 256):
            if batch << log_n > args.max_words:
                continue
            for m in (1, 2, 8):
                shapes(log_n, batch, m, ctx, args.iters)


if __name__ == "__main__":
    main()
