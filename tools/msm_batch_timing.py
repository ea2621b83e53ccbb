#!/usr/bin/env python3
"""Timing of ronk_msm_pluto_ext_batch (msm.cu), ms per call, against a loop of ronk_msm_pluto_ext over the same device
rows.  Both are synchronous; each timing is the host clock around one call (or one loop).  After --warmup calls of each,
the two are timed alternately --iters times and the medians are printed.

Rows are uniform scalars < 17 over whole-group points (Infinity mixed in), at batch ∈ --batches × n ∈ --ns (7 is the
reference's SRS length).  For the batched call the line also gives the scalar bytes read per second (batch·n / time)
and that rate's share of the H100 SXM data sheet's 3.35 TB/s; batch 1 compares the batched entry with the single call.
The card's name, power limit and maximum SM clock are printed with the numbers; --json writes the rows as JSON lines."""
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
from ronkathon_b200 import Context, _lib  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def points(n, seed):
    """Whole-group points: every on-curve (x0, 0, y0, y1 ∈ {0, 1}) word, drawn at random, about 2 % Infinity."""
    import oracle
    base = [bytes([x0, 0, y0, y1]) for x0 in range(101) for y0 in range(101) for y1 in (0, 1)
            if oracle.on_curve(bytes([x0, 0, y0, y1]))]
    base = np.frombuffer(b"".join(base), dtype=np.uint8).reshape(-1, 4)
    rng = np.random.default_rng(seed)
    pts = base[rng.integers(0, len(base), n)].copy()
    pts[rng.integers(0, n, max(1, n // 50))] = 0xFF
    return torch.from_numpy(pts).cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,2,16,256,4096")
    ap.add_argument("--ns", default="7,4096,65536,1048576")
    ap.add_argument("--iters", type=int, default=21)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default="")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    print(f"# {card()}", flush=True)
    ctx = Context(0, torch.cuda.current_stream().cuda_stream)
    lib = _lib.lib()
    sink = open(args.json, "w") if args.json else None
    print(f"{'n':>8} {'batch':>6} {'batched ms':>11} {'loop ms':>10} {'speed-up':>9} {'GB/s':>8} {'of 3.35 TB/s':>13}")
    for n in (int(v) for v in args.ns.split(",")):
        P = points(n, n)
        for batch in (int(v) for v in args.batches.split(",")):
            g = torch.Generator(device="cuda").manual_seed(batch * 7 + n)
            S = torch.randint(0, 17, (batch, n), dtype=torch.uint8, device="cuda", generator=g)
            out = torch.empty((batch, 4), dtype=torch.uint8, device="cuda")
            one = np.empty(4, dtype=np.uint8)
            rows = [S[r].data_ptr() for r in range(batch)]

            def batched():
                ctx.check(lib.ronk_msm_pluto_ext_batch(ctx._h, P.data_ptr(), n, S.data_ptr(), n, batch, out.data_ptr()))

            def loop():
                for r in rows:
                    ctx.check(lib.ronk_msm_pluto_ext(ctx._h, P.data_ptr(), n, r, n, one.ctypes.data))

            for _ in range(args.warmup):
                batched()
                loop()
            want = out.cpu().numpy()
            loop_words = []
            for r in range(min(batch, 4)):   # the words agree on the timed inputs
                lib.ronk_msm_pluto_ext(ctx._h, P.data_ptr(), n, rows[r], n, one.ctypes.data)
                loop_words.append(one.tobytes())
            assert [want[r].tobytes() for r in range(min(batch, 4))] == loop_words
            tb, tl = [], []
            for _ in range(args.iters):
                for fn, acc in ((batched, tb), (loop, tl)):
                    torch.cuda.synchronize()
                    t = time.perf_counter()
                    fn()
                    acc.append((time.perf_counter() - t) * 1e3)
            b, lp = statistics.median(tb), statistics.median(tl)
            rate = batch * n / (b * 1e-3)
            row = {"n": n, "batch": batch, "batched_ms": b, "loop_ms": lp, "speedup": lp / b, "bytes_per_s": rate,
                   "share_of_hbm": rate / HBM_BYTES_PER_S}
            print(f"{n:8d} {batch:6d} {b:11.4f} {lp:10.4f} {lp / b:8.2f}x {rate / 1e9:8.1f} {100 * rate / HBM_BYTES_PER_S:12.1f}%",
                  flush=True)
            if sink:
                sink.write(json.dumps(row) + "\n")
            del S, out
    print(f"# {card()}")


if __name__ == "__main__":
    main()
