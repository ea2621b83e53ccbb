#!/usr/bin/env python3
"""Timing of ronk_sha256 and the SHA-256 Merkle entries (sha256.cu) on device-resident inputs.

- SHA-256 throughput (hashes/s, and GB/s of message bytes) for 2^20 and 2^24 messages of 32, 64 and 1024 bytes.
- Tree builds (ronk_merkle_build_sha256) of 2^20 and 2^24 leaves of 32 bytes: time and compressions/s.
- Proof gather (ronk_merkle_proofs_sha256) and verification (ronk_merkle_verify_sha256) of 2^20 items on the 2^20-leaf
  tree.
- Python's hashlib on one core, on 2^16 messages of each length, for context only.
- Parity with hashlib on 64 sampled outputs of every timed call (digests, tree nodes against their children, proofs
  through verification).

Each number is the median of --iters calls timed with CUDA events on the context's stream after --warmup calls.  The
calls that read a device flag synchronise once each, inside the timed window, as a user's call does.  The card's name,
power limit and maximum SM clock are printed with the numbers; --json writes the rows as JSON lines."""
import argparse
import hashlib
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


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


def blocks(length):
    return (length + 8) // 64 + 1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=7)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    ctx = Context(0, torch.cuda.current_stream().cuda_stream)
    gen = torch.Generator(device="cuda").manual_seed(1)
    rng = np.random.default_rng(2)
    rows = []
    print("card:", card())

    def emit(row):
        rows.append(row)
        print(json.dumps(row))

    # ---- SHA-256 of fixed-length messages --------------------------------------------------------------------------
    for log_n in (20, 24):
        n = 1 << log_n
        for length in (32, 64, 1024):
            data = torch.randint(0, 256, (n * length,), dtype=torch.uint8, device="cuda", generator=gen)
            offs = torch.arange(0, (n + 1) * length, length, dtype=torch.int64, device="cuda")
            out = torch.empty((n, 32), dtype=torch.uint8, device="cuda")
            args_ = (ops._lib._ptr(data), data.numel(), ops._lib._ptr(offs), n, ops._lib._ptr(out))
            ms = timed(ctx, lambda: ctx.call("ronk_sha256", *args_), args.warmup, args.iters)
            pick = rng.integers(0, n, 64)
            h = out.cpu().numpy()
            ok = all(h[i].tobytes() == hashlib.sha256(data[i * length:(i + 1) * length].cpu().numpy().tobytes()).digest()
                     for i in pick)
            emit({"what": "sha256", "n": n, "len": length, "ms": ms, "hashes_per_s": n / ms * 1e3,
                  "input_GB_per_s": n * length / ms / 1e6, "bytes_moved_GB_per_s": n * (length + 8 + 32) / ms / 1e6,
                  "compressions_per_s": n * blocks(length) / ms * 1e3, "parity": ok})
            del data, offs, out
            torch.cuda.empty_cache()

    # ---- tree builds, proofs and verification ---------------------------------------------------------------------
    for log_n in (20, 24):
        n = 1 << log_n
        data = torch.randint(0, 256, (n * 32,), dtype=torch.uint8, device="cuda", generator=gen)
        offs = torch.arange(0, (n + 1) * 32, 32, dtype=torch.int64, device="cuda")
        sizes, lo = ops.merkle_levels(n)
        nodes = torch.empty((sum(sizes), 32), dtype=torch.uint8, device="cuda")
        args_ = (ops._lib._ptr(data), data.numel(), ops._lib._ptr(offs), n, ops._lib._ptr(nodes))
        before = ctx.launches
        ctx.call("ronk_merkle_build_sha256", *args_)
        launches = ctx.launches - before
        ms = timed(ctx, lambda: ctx.call("ronk_merkle_build_sha256", *args_), args.warmup, args.iters)
        h = nodes.cpu().numpy()
        ok = True
        for l in range(1, len(sizes)):
            for i in rng.integers(0, sizes[l], 4):
                c0, c1 = lo[l - 1] + 2 * i, lo[l - 1] + min(2 * i + 1, sizes[l - 1] - 1)
                ok &= h[lo[l] + i].tobytes() == hashlib.sha256(h[c0].tobytes() + h[c1].tobytes()).digest()
        for i in rng.integers(0, n, 16):
            ok &= h[i].tobytes() == hashlib.sha256(data[32 * i:32 * i + 32].cpu().numpy().tobytes()).digest()
        comps = n * 1 + (sum(sizes) - n) * 2
        emit({"what": "merkle_build", "n": n, "leaf_len": 32, "launches": launches, "ms": ms,
              "leaves_per_s": n / ms * 1e3, "compressions_per_s": comps / ms * 1e3, "parity": bool(ok)})
        if log_n == 20:
            m = n
            L = len(sizes) - 1
            idx = torch.from_numpy(rng.integers(0, n, m).astype(np.int64)).cuda()
            sib = torch.empty((m, L, 32), dtype=torch.uint8, device="cuda")
            sides = torch.empty((m, L), dtype=torch.uint8, device="cuda")
            pargs = (ops._lib._ptr(nodes), n, ops._lib._ptr(idx), m, ops._lib._ptr(sib), ops._lib._ptr(sides))
            ms_p = timed(ctx, lambda: ctx.call("ronk_merkle_proofs_sha256", *pargs), args.warmup, args.iters)
            # the items are the leaves at idx, gathered as one contiguous batch
            ii = idx.cpu().numpy()
            items = data.view(n, 32)[idx].contiguous().view(-1)
            ioffs = torch.arange(0, (m + 1) * 32, 32, dtype=torch.int64, device="cuda")
            ok_t = torch.empty(m, dtype=torch.uint8, device="cuda")
            root = nodes[-1].contiguous()
            vargs = (ops._lib._ptr(root), ops._lib._ptr(items), items.numel(), ops._lib._ptr(ioffs), m, ops._lib._ptr(sib),
                     ops._lib._ptr(sides), L, ops._lib._ptr(ok_t))
            ms_v = timed(ctx, lambda: ctx.call("ronk_merkle_verify_sha256", *vargs), args.warmup, args.iters)
            s, d = sib.cpu().numpy(), sides.cpu().numpy()
            pok = bool(ok_t.cpu().numpy().all())
            for j in rng.integers(0, m, 8):
                x = int(ii[j]) >> np.arange(L)
                pok &= bool((d[j] == (1 - (x & 1))).all())
                pok &= all(s[j, l].tobytes() == h[lo[l] + (int(x[l]) ^ 1)].tobytes() for l in range(L))
            emit({"what": "merkle_proofs", "m": m, "depth": L, "ms": ms_p, "proofs_per_s": m / ms_p * 1e3,
                  "GB_per_s_written": m * L * 33 / ms_p / 1e6, "parity": pok})
            emit({"what": "merkle_verify", "m": m, "depth": L, "ms": ms_v, "proofs_per_s": m / ms_v * 1e3,
                  "compressions_per_s": m * (1 + 2 * L) / ms_v * 1e3, "parity": pok})
        del data, offs, nodes
        torch.cuda.empty_cache()

    # ---- hashlib on one core -----------------------------------------------------------------------------------------
    for length in (32, 64, 1024):
        msgs = [rng.integers(0, 256, length, dtype=np.uint8).tobytes() for _ in range(1 << 16)]
        t0 = time.perf_counter()
        for x in msgs:
            hashlib.sha256(x).digest()
        dt = time.perf_counter() - t0
        emit({"what": "hashlib_one_core", "n": len(msgs), "len": length, "hashes_per_s": len(msgs) / dt,
              "input_GB_per_s": len(msgs) * length / dt / 1e9})

    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            f.write(json.dumps({"card": card()}) + "\n")
            for r in rows:
                f.write(json.dumps(r) + "\n")
    ctx.close()
    sys.exit(0 if all(r.get("parity", True) for r in rows) else 1)


if __name__ == "__main__":
    main()
