#!/usr/bin/env python3
"""CUDA-event timing of ronk_poly_mul_batch_u64 (poly_batch.cu), ms per call: the median of --iters calls after one
warm call.

1. One batched call against a loop of ronk_poly_mul_u64 calls over the same rows, at shapes users run:
   2^16 × (9 × 9) over F101, 2^14 × (256 × 256) over Goldilocks and BabyBear, 2^10 × (2^12 × 2^12) and
   16 × (2^20 × 2^20) over Goldilocks.
2. The crossovers, at a fixed total of 2^22 output words (batch = 2^22 / L), each path forced on its own context with
   RONK_POLY_BATCH_PATH (1 = schoolbook, 2 = transforms, 3 = batched transforms even where the fused kernel fits):
   schoolbook against fused at da = db = 2^1 … 2^10 (Goldilocks, BabyBear), fused against the batched transforms at
   L = 2^8 … 2^11, and schoolbook against multi-modular at da = db = 2^3 … 2^11 for k = 1, 2, 3 (101, 2^31 - 1,
   2^64 - 279).  For each, da·db / (N·log2 N) of the smallest size from which the transform path wins at every larger
   size is printed: the constants of poly_batch.cu.
3. The kernel split of one profiled call per path, including the pad / clip share of the batched transforms.

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

GL, BB, F101 = 0xFFFFFFFF00000001, 2013265921, 101
CRT = {"k1_f101": (101, 2), "k2_m31": ((1 << 31) - 1, 7), "k3_2^64-279": ((1 << 64) - 279, 5)}


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


def context(stream, path):
    os.environ["RONK_POLY_BATCH_PATH"] = str(path)
    try:
        return Context(0, stream)
    finally:
        del os.environ["RONK_POLY_BATCH_PATH"]


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


def rows(c, batch, d, p, seed):
    return ops.splitmix_fill(c, batch * d, seed, p).view(batch, d)


def crossover(table, key_fast, key_slow):
    """the smallest size from which key_fast beats key_slow at every larger size, or None"""
    best = None
    for size in sorted(table, reverse=True):
        if table[size][key_fast] < table[size][key_slow]:
            best = size
        else:
            break
    return best


def per_point(d):
    L = 2 * d - 1
    lg = (L - 1).bit_length()
    return round(d * d / ((1 << lg) * lg), 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=7)
    ap.add_argument("--loop-iters", type=int, default=2)
    ap.add_argument("--total-log", type=int, default=22)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    stream = torch.cuda.current_stream().cuda_stream
    auto = Context(0, stream)
    forced = {k: context(stream, k) for k in (1, 2, 3)}
    result = {"card": card(), "batched_vs_loop": {}, "crossovers": {}, "kernel_split": {}}

    for name, (batch, d, p, g) in {"2^16x(9x9)_f101": (1 << 16, 9, F101, 2), "2^14x(256x256)_gl": (1 << 14, 256, GL, 7),
                                   "2^14x(256x256)_babybear": (1 << 14, 256, BB, 31),
                                   "2^10x(2^12x2^12)_gl": (1 << 10, 1 << 12, GL, 7),
                                   "16x(2^20x2^20)_gl": (16, 1 << 20, GL, 7)}.items():
        a, b = rows(auto, batch, d, p, 1), rows(auto, batch, d, p, 2)
        out = torch.empty(2 * d - 1, dtype=torch.int64, device="cuda")

        def loop():
            for r in range(batch):
                auto.call("ronk_poly_mul_u64", p, g, a[r].data_ptr(), d, b[r].data_ptr(), d, out.data_ptr())
        r = {"batched_ms": timed(lambda: ops.poly_mul_batch(auto, a, b, p, g), args.iters),
             "batched_shared_b_ms": timed(lambda: ops.poly_mul_batch(auto, a, b[0], p, g), args.iters),
             "loop_ms": timed(loop, args.loop_iters),
             "kernels_ms": split(auto, lambda: ops.poly_mul_batch(auto, a, b, p, g))}
        r["speedup"] = round(r["loop_ms"] / r["batched_ms"], 1)
        result["batched_vs_loop"][name] = r
        print(name, r, file=sys.stderr, flush=True)
        del a, b

    total = 1 << args.total_log

    def sweep(p, g, logs, ka, kb):
        table = {}
        for lg in logs:
            d = 1 << lg
            batch = max(1, total // (2 * d - 1))
            a, b = rows(auto, batch, d, p, 3), rows(auto, batch, d, p, 4)
            table[d] = {ka: timed(lambda: ops.poly_mul_batch(forced[ka], a, b, p, g), args.iters),
                        kb: timed(lambda: ops.poly_mul_batch(forced[kb], a, b, p, g), args.iters)}
            print(p, d, table[d], file=sys.stderr, flush=True)
        return table

    for name, (p, g) in {"gl": (GL, 7), "babybear": (BB, 31)}.items():
        t = sweep(p, g, range(1, 11), 1, 2)
        best = crossover(t, 2, 1)
        result["crossovers"][f"school_vs_fused_{name}"] = {
            "ms_by_d": {d: {"school": v[1], "fused": v[2]} for d, v in t.items()},
            "fused_wins_from_d": best, "per_point": per_point(best) if best else None}
        t = {}
        for L in (1 << 8, 1 << 9, 1 << 10, 1 << 11):
            da, db = L // 2, L // 2 + 1
            batch = max(1, total // L)
            a, b = rows(auto, batch, da, p, 5), rows(auto, batch, db, p, 6)
            t[L] = {"fused": timed(lambda: ops.poly_mul_batch(forced[2], a, b, p, g), args.iters),
                    "long": timed(lambda: ops.poly_mul_batch(forced[3], a, b, p, g), args.iters)}
            print(name, "L", L, t[L], file=sys.stderr, flush=True)
        result["crossovers"][f"fused_vs_long_{name}"] = t
    for name, (p, g) in CRT.items():
        t = sweep(p, g, range(3, 12), 1, 2)
        best = crossover(t, 2, 1)
        result["crossovers"][f"school_vs_crt_{name}"] = {
            "ms_by_d": {d: {"school": v[1], "crt": v[2]} for d, v in t.items()},
            "crt_wins_from_d": best, "per_point": per_point(best) if best else None}

    for name, (c, p, g, batch, d, shared) in {
            "school_2^16x(9x9)_f101": (forced[1], F101, 2, 1 << 16, 9, False),
            "fused_2^14x(256x256)_gl": (forced[2], GL, 7, 1 << 14, 256, False),
            "long_2^10x(2^12x2^12)_gl": (forced[2], GL, 7, 1 << 10, 1 << 12, False),
            "long_shared_b_2^10x(2^12x2^12)_gl": (forced[2], GL, 7, 1 << 10, 1 << 12, True),
            "long_16x(2^20x2^20)_gl": (forced[2], GL, 7, 16, 1 << 20, False),
            "crt_k1_2^10x(2^10x2^10)_f101": (forced[2], F101, 2, 1 << 10, 1 << 10, False),
            "crt_k3_2^10x(2^10x2^10)_2^64-279": (forced[2], (1 << 64) - 279, 5, 1 << 10, 1 << 10, False)}.items():
        a, b = rows(auto, batch, d, p, 7), rows(auto, batch, d, p, 8)
        bb = b[0] if shared else b
        fn = lambda: ops.poly_mul_batch(c, a, bb, p, g)  # noqa: E731
        fn()
        result["kernel_split"][name] = {"ms": timed(fn, args.iters), "kernels_ms": split(c, fn)}
        print(name, result["kernel_split"][name], file=sys.stderr, flush=True)
        del a, b, bb
    print(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
