#!/usr/bin/env python3
"""CUDA-event timing of ronk_rs_decode_u64 on Goldilocks: ms per batched call (median of --iters calls after one warm
call), codewords per second, and the kernel split of one profiled call (ronk_prof: ms per kernel name, summed).

Cases (each row a codeword of a seeded message with `errors` positions changed, so every row decodes):
  - n = 256, k = 224, batch 2^16, 16 errors per row (power-of-two transforms);
  - n = 255, k = 223, batch 2^16, 16 errors (the literal path's batched O(n²) kernel);
  - n = 2^16, n - k = RONK_RS_MAX_PARITY, a full radius of errors, batch 8 (the locator's sequential steps);
  - n = 3·2^20, n - k = 4096, a full radius of errors, batch 4 (Bluestein).
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
CASES = [("n256_k224", 256, 224, 1 << 16, 16), ("n255_k223_literal", 255, 223, 1 << 16, 16),
         ("n65536_cap", 1 << 16, (1 << 16) - CAP, 8, CAP // 2), ("n3x2^20_m4096", 3 << 20, (3 << 20) - 4096, 4, 2048)]


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


def received(c, n, k, batch, errors, seed):
    """batch codewords of seeded messages with `errors` distinct positions per row changed (v → v + 1 mod p)."""
    msg = ops.splitmix_fill(c, batch * k, seed, GL)
    cw = ops.rs_encode(c, msg, n, batch).view(batch, n)
    g = torch.Generator(device="cuda").manual_seed(seed)
    pos = torch.argsort(torch.rand(batch, n, device="cuda", generator=g), dim=1)[:, :errors]
    v = cw.gather(1, pos)
    cw.scatter_(1, pos, torch.where(v == GL_M1, torch.zeros_like(v), v + 1))
    return msg, cw.reshape(-1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--cases", default=",".join(c[0] for c in CASES))
    args = ap.parse_args()
    torch.cuda.set_device(0)
    c = Context(0, torch.cuda.current_stream().cuda_stream)
    res = {}
    for name, n, k, batch, errors in CASES:
        if name not in args.cases.split(","):
            continue
        msg, rx = received(c, n, k, batch, errors, 1)
        out, st = ops.rs_decode(c, rx, k, None, batch)
        torch.cuda.synchronize()
        assert torch.equal(out, msg) and bool((st == errors).all()), name
        ms = timed(lambda: ops.rs_decode(c, rx, k, None, batch), args.iters)
        c.prof_enable(True)
        ops.rs_decode(c, rx, k, None, batch)
        split = defaultdict(float)
        for nm, t in c.prof_fetch():
            split[nm] += t
        c.prof_enable(False)
        res[name] = {"n": n, "k": k, "batch": batch, "errors_per_row": errors, "ms": round(ms, 4),
                     "codewords_per_s": round(batch / ms * 1e3), "kernels_ms": {nm: round(t, 4) for nm, t in split.items()}}
        print(name, res[name], file=sys.stderr, flush=True)
        del msg, rx, out, st
    print(json.dumps({"card": card(), "cases": res}, indent=1))
    c.close()


if __name__ == "__main__":
    main()
