#!/usr/bin/env python3
"""Timing of ronk_kzg_check_pluto_ext_batch (pairing.cu): rows per second and bytes per second at n = 2^16 … 2^26.

Each call is synchronous; each timing is the host clock around one call, after --warmup calls, and the median of --iters
is printed.  A row moves 10 bytes in (commitment, proof, point, value) and 1 byte out, so bytes/s is 11·n over the time,
and its share of the H100 SXM data sheet's 3.35 TB/s is printed beside it.  The rows are the openings of one valid
proof against every commitment of E[17] under every value whose check is defined, drawn at random, so about one row in
17 verifies.

The one-time table build (the commit's group tables on the host, then pairing_table_kernel's 83 521 Miller loops) is
timed on a fresh context as its first call at n = 1, beside the second call; the table kernel's own time comes from the
library's launch profiler.  The card's name, power limit and maximum SM clock are printed with the numbers; --json
writes the rows as JSON lines."""
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
from ronkathon_b200 import Context, _lib  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
BYTES_PER_ROW = 11


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def grid_rows():
    """(C uint8 [m, 4], proof, z, V uint8 [m], ok bool [m]): every E[17] commitment × value whose check is defined."""
    import oracle
    import pairing_oracle as po
    g1, g2 = oracle.setup()
    gen = bytes([36, 0, 0, 31])

    def smul(p, s):
        acc = b"\xff" * 4
        for _ in range(s):
            acc = oracle.point_add(acc, p)
        return acc
    e17 = sorted({oracle.point_add(smul(g1[0], i), smul(gen, j)) for i in range(17) for j in range(17)})
    f, z = [7, 16, 1, 11, 1], 3
    q = oracle.open_(f, z, g1)
    C = [c for c in e17 for _ in range(17)]
    V = [v for _ in e17 for v in range(17)]
    ok, panic = po.kzg_check_many(C, [q] * len(C), [z] * len(C), V, g1, g2)
    keep = np.flatnonzero(~panic)
    Ca = np.frombuffer(b"".join(C), np.uint8).reshape(-1, 4)[keep]
    return Ca, q, z, np.asarray(V, np.uint8)[keep], ok[keep], g1, g2


def table_build(g1d, g2d, row):
    """(first call ms, second call ms, pairing_table kernel ms) on a fresh context, n = 1."""
    ctx = Context(0, torch.cuda.current_stream().cuda_stream)
    lib = _lib.lib()
    C, Q, Z, V = row
    ok = torch.empty(1, dtype=torch.uint8, device="cuda")
    ts = []
    ctx.prof_enable(True)
    for _ in range(2):
        torch.cuda.synchronize()
        t = time.perf_counter()
        ctx.check(lib.ronk_kzg_check_pluto_ext_batch(ctx._h, C.data_ptr(), Q.data_ptr(), Z.data_ptr(), V.data_ptr(), 1,
                                                      g1d.data_ptr(), 7, g2d.data_ptr(), 2, ok.data_ptr()))
        ts.append((time.perf_counter() - t) * 1e3)
    kernel = sum(ms for name, ms in ctx.prof_fetch() if name == "pairing_table")
    ctx.close()
    return ts[0], ts[1], kernel


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-ns", default="16,18,20,22,24,26")
    ap.add_argument("--iters", type=int, default=21)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default="")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    print(f"# {card()}", flush=True)
    Ca, q, z, Va, oka, g1, g2 = grid_rows()
    g1d = torch.from_numpy(np.frombuffer(b"".join(g1), np.uint8).copy()).cuda()
    g2d = torch.from_numpy(np.frombuffer(b"".join(g2), np.uint8).copy()).cuda()
    Cg, Vg = torch.from_numpy(Ca.copy()).cuda(), torch.from_numpy(Va.copy()).cuda()
    okg = torch.from_numpy(oka.astype(np.uint8)).cuda()
    qd = torch.tensor(list(q), dtype=torch.uint8, device="cuda")
    first, second, kern = table_build(g1d, g2d, (Cg[:1].contiguous(), qd, torch.tensor([z], dtype=torch.uint8, device="cuda"),
                                                 Vg[:1].contiguous()))
    sink = open(args.json, "w") if args.json else None
    line = {"table_first_call_ms": first, "second_call_ms": second, "pairing_table_kernel_ms": kern}
    print(f"# table build: first call {first:.3f} ms (host group tables + pairing_table kernel {kern:.3f} ms), "
          f"second call {second:.3f} ms", flush=True)
    if sink:
        sink.write(json.dumps(line) + "\n")
    ctx = Context(0, torch.cuda.current_stream().cuda_stream)
    lib = _lib.lib()
    print(f"{'log2 n':>6} {'ms':>9} {'rows/s':>10} {'GB/s':>8} {'of 3.35 TB/s':>13}")
    for lg in (int(v) for v in args.log_ns.split(",")):
        n = 1 << lg
        gen = torch.Generator(device="cuda").manual_seed(lg)
        idx = torch.randint(0, Cg.shape[0], (n,), device="cuda", generator=gen)
        C, V, want = Cg[idx].contiguous(), Vg[idx].contiguous(), okg[idx]
        Q = qd.repeat(n)
        Z = torch.full((n,), z, dtype=torch.uint8, device="cuda")
        ok = torch.empty(n, dtype=torch.uint8, device="cuda")

        def call():
            ctx.check(lib.ronk_kzg_check_pluto_ext_batch(ctx._h, C.data_ptr(), Q.data_ptr(), Z.data_ptr(), V.data_ptr(), n,
                                                          g1d.data_ptr(), 7, g2d.data_ptr(), 2, ok.data_ptr()))
        for _ in range(args.warmup):
            call()
        assert torch.equal(ok, want), "check mismatch against the oracle's rows"
        ts = []
        for _ in range(args.iters):
            torch.cuda.synchronize()
            t = time.perf_counter()
            call()
            ts.append((time.perf_counter() - t) * 1e3)
        ms = statistics.median(ts)
        rows = n / (ms * 1e-3)
        bps = rows * BYTES_PER_ROW
        print(f"{lg:6d} {ms:9.4f} {rows:10.3e} {bps / 1e9:8.1f} {100 * bps / HBM_BYTES_PER_S:12.1f}%", flush=True)
        if sink:
            sink.write(json.dumps({"n": n, "ms": ms, "rows_per_s": rows, "bytes_per_s": bps,
                                   "share_of_hbm": bps / HBM_BYTES_PER_S}) + "\n")
        del C, V, Q, Z, ok, want, idx
    print(f"# {card()}")


if __name__ == "__main__":
    main()
