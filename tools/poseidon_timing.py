#!/usr/bin/env python3
"""Timing of ronk_poseidon_permute_u64 and ronk_poseidon_sponge_u64 (poseidon.cu) on Goldilocks with α = 7, 8 full and
22 partial rounds, and constants from splitmix64.

- Permutations per second for 2^20 and 2^24 states at width 8, 12 and 16, in place.
- Sponge rows per second for 2^20 rows of 64 and 256 words at rate 8 (widths 12 and 16), 4 words squeezed per row.
- The algorithmic field-multiplication count of a permutation, R·t² for the MDS layers plus the S-box products
  (4 per x^7: x², x³, x⁶, x⁷; num_f·t + num_p S-boxes), over kernel time.
- The one-core C oracle (tests/poseidon_oracle.c, %-reduced __int128 products) on 2^12 states, for context only.
- Oracle parity on 64 sampled rows of every timed output.

Each number is the median of --iters calls timed with CUDA events on the context's stream after --warmup calls.  The
card's name, power limit and maximum SM clock are printed with the numbers; --json writes the rows as JSON lines."""
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle  # noqa: E402
import poseidon_oracle as po  # noqa: E402
from ronkathon_b200 import Context, ops  # noqa: E402
from ronkathon_b200.hashes import PoseidonConfig  # noqa: E402

GL = oracle.GOLDILOCKS
ALPHA, NUM_F, NUM_P = 7, 8, 22
SBOX_MULS = 4


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def configs(t):
    rc = oracle.splitmix(GL, 100 + t, (NUM_F + NUM_P) * t)
    mds = oracle.splitmix(GL, 200 + t, t * t).reshape(t, t)
    return (PoseidonConfig(t, ALPHA, NUM_P, NUM_F, rc.tolist(), mds.tolist()),
            po.Config(GL, t, ALPHA, NUM_P, NUM_F, rc.tolist(), mds.tolist()))


def muls_per_permutation(t):
    return (NUM_F + NUM_P) * t * t + (NUM_F * t + NUM_P) * SBOX_MULS


def timed(ctx, fn, warmup, iters):
    stream = torch.cuda.ExternalStream(ctx.stream) if ctx.stream else torch.cuda.current_stream()
    for _ in range(warmup):
        fn()
    ctx.sync()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        fn()
        b.record(stream)
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def sample(n, k=64, seed=0):
    return np.sort(np.random.default_rng(seed).choice(n, size=min(k, n), replace=False))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--widths", default="8,12,16")
    ap.add_argument("--log-batches", default="20,24")
    ap.add_argument("--iters", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--json", default="")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    print(f"# {card()}", flush=True)
    ctx = Context(0, torch.cuda.current_stream().cuda_stream)
    sink = open(args.json, "w") if args.json else None

    def emit(line):
        if sink:
            sink.write(json.dumps(line) + "\n")
            sink.flush()

    print(f"{'op':>8} {'t':>3} {'rows':>9} {'len':>4} {'ms':>9} {'rows/s':>10} {'Gmul/s':>8} {'parity':>7}", flush=True)
    for t in (int(v) for v in args.widths.split(",")):
        cfg, orc = configs(t)
        for lg in (int(v) for v in args.log_batches.split(",")):
            n = 1 << lg
            start = ops.to_device(oracle.splitmix(GL, 300 + lg, n * t)).view(n, t)
            states = start.clone()
            ms = timed(ctx, lambda: ops.poseidon_permute_(ctx, states, cfg), args.warmup, args.iters)
            # parity: one permutation of the start states, checked on sampled rows
            states.copy_(start)
            ops.poseidon_permute_(ctx, states, cfg)
            ctx.sync()
            idx = sample(n, seed=lg)
            got = ops.to_host(states[torch.from_numpy(idx).cuda()].contiguous()).reshape(-1, t)
            ok = np.array_equal(got, po.permute(orc, ops.to_host(start[torch.from_numpy(idx).cuda()].contiguous())))
            rate = n / (ms * 1e-3)
            gmul = rate * muls_per_permutation(t) / 1e9
            print(f"{'permute':>8} {t:3d} {n:9d} {t:4d} {ms:9.3f} {rate:10.3e} {gmul:8.1f} {str(ok):>7}", flush=True)
            emit({"op": "permute", "width": t, "rows": n, "ms": ms, "permutations_per_s": rate, "gmul_per_s": gmul,
                  "muls_per_permutation": muls_per_permutation(t), "parity": ok})
            del start, states
            torch.cuda.empty_cache()
    for t in (12, 16):
        cfg, orc = configs(t)
        for length in (64, 256):
            n, rate_w, n_out = 1 << 20, 8, 4
            rows = ops.to_device(oracle.splitmix(GL, 400 + length, n * length)).view(n, length)
            out = None

            def call():
                nonlocal out
                out = ops.poseidon_sponge(ctx, rows, n_out, rate_w, cfg)
            ms = timed(ctx, call, args.warmup, args.iters)
            perms = -(-length // rate_w)
            idx = sample(n, seed=length)
            got = ops.to_host(out[torch.from_numpy(idx).cuda()].contiguous()).reshape(-1, n_out)
            ok = np.array_equal(got, po.sponge_rows(orc, rate_w, ops.to_host(rows[torch.from_numpy(idx).cuda()].contiguous())
                                                   .reshape(-1, length), n_out))
            r = n / (ms * 1e-3)
            gmul = r * perms * muls_per_permutation(t) / 1e9
            print(f"{'sponge':>8} {t:3d} {n:9d} {length:4d} {ms:9.3f} {r:10.3e} {gmul:8.1f} {str(ok):>7}", flush=True)
            emit({"op": "sponge", "width": t, "rate": rate_w, "rows": n, "len": length, "n_out": n_out, "ms": ms,
                  "rows_per_s": r, "permutations_per_row": perms, "gmul_per_s": gmul, "parity": ok})
            del rows, out
            torch.cuda.empty_cache()
    for t in (8, 12, 16):
        _, orc = configs(t)
        st = oracle.splitmix(GL, 500 + t, 4096 * t).reshape(4096, t)
        t0 = time.perf_counter()
        po.permute(orc, st)
        r = 4096 / (time.perf_counter() - t0)
        print(f"# one-core C oracle, width {t}: {r:.3e} permutations/s", flush=True)
        emit({"op": "oracle_permute", "width": t, "permutations_per_s": r})
    print(f"# {card()}")


if __name__ == "__main__":
    main()
