#!/usr/bin/env python3
"""Small invocation of every kernel family for compute-sanitizer (memcheck / racecheck / synccheck):
   compute-sanitizer --tool racecheck python tools/sanitize_smoke.py"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
import oracle
from gpu_util import GL, ctx, dev, host, msm_inputs
from ronkathon_b200 import ops, kzg, curve, Polynomial, PlutoBaseField, PlutoScalarField

c = ctx()
ok = True
# (16, 1): the cluster kernel; (16, 3): the one-group-per-thread two-launch tile passes; (20, 1): passes A1 / A2 / C
for lg, batch in ((3, 5), (6, 3), (10, 2), (13, 1), (14, 1), (16, 1), (16, 3), (20, 1)):
    a = oracle.splitmix(GL, lg, batch << lg)
    d = dev(a); ops.ntt_(c, d, lg, batch); X = host(d)
    ok &= all(np.array_equal(X[b << lg:(b + 1) << lg], oracle.ntt_fast(GL, a[b << lg:(b + 1) << lg])) for b in range(batch))
    ops.ntt_(c, d, lg, batch, inverse=True); ok &= np.array_equal(host(d), a)
a = np.array([1, 2, 3, 4], dtype=np.uint64); d = dev(a); ops.ntt_(c, d, 2, 1, p=101, g=2); ok &= list(host(d)) == [10, 79, 99, 18]
A, B = oracle.splitmix(GL, 1, 700), oracle.splitmix(GL, 2, 900)
ok &= np.array_equal(host(ops.poly_mul(c, dev(A), dev(B))), oracle.poly_mul(GL, A, B))
ok &= np.array_equal(host(ops.poly_mul(c, dev(A[:20]), dev(B[:30]))), oracle.poly_mul(GL, A[:20], B[:30]))
xs = oracle.splitmix(GL, 3, 5)
ok &= list(host(ops.poly_eval(c, dev(A), dev(xs)))) == [oracle.poly_eval_horner(GL, A, int(x)) for x in xs]
q, r = Polynomial([5, 6, 7, 8, 9], PlutoBaseField).quotient_and_remainder(Polynomial([1, 2, 3, 4], PlutoBaseField))
ok &= list(q.coefficients) == [95, 78, 0, 0, 0]
ok &= Polynomial([1, 2, 3, 4], PlutoBaseField).dft().evaluate(PlutoBaseField(2)).value == 49
pts, sc = msm_inputs(5000)
ok &= ops.msm(c, torch.from_numpy(pts).cuda(), torch.from_numpy(sc).cuda()) == oracle.commit(sc, pts, fast=True)
g1, _ = kzg.setup(); ok &= kzg.commit([7, 16, 1, 11, 1], g1).raw == bytes([32, 0, 59, 0])
g1, g2 = kzg.setup()
cm, pf = kzg.commit([3, 2, 1], g1), kzg.open_([3, 2, 1], 5, g1)
ok &= kzg.check_batch([cm] * 3, [pf] * 3, [5] * 3, [4, 10, 4], g1, g2) == [True, False, True]
ok &= curve.pairing(curve.AffinePoint(bytes([9, 37, 19, 93])), curve.AffinePoint(bytes([63, 0, 0, 35]))) == (26, 97)
import poseidon_oracle as po
from ronkathon_b200.hashes import PoseidonConfig
orc = po.Config(GL, 5, 7, 3, 4, oracle.splitmix(GL, 4, 7 * 5).tolist(), oracle.splitmix(GL, 5, 25).reshape(5, 5).tolist())
pcfg = PoseidonConfig(5, 7, 3, 4, orc.rc.tolist(), orc.mds.reshape(5, 5).tolist())
st = oracle.splitmix(GL, 6, 300 * 5).reshape(300, 5)
ok &= np.array_equal(host(ops.poseidon_permute_(c, dev(st).view(300, 5), pcfg)).reshape(300, 5), po.permute(orc, st))
ok &= np.array_equal(host(ops.poseidon_sponge(c, dev(st).view(300, 5), 7, 3, pcfg)).reshape(300, 7), po.sponge_rows(orc, 3, st, 7))
import hashlib
import merkle_oracle as mo
leaves = [bytes(range(i % 5, i % 5 + i % 45)) for i in range(1100)]   # ragged, misaligned; two build launches
lo = np.concatenate([[0], np.cumsum([len(x) for x in leaves])]).astype(np.uint64)
ld = torch.frombuffer(bytearray(b"".join(leaves)), dtype=torch.uint8).cuda()
dig = ops.sha256(c, ld, dev(lo)).cpu().numpy()
ok &= all(dig[i].tobytes() == hashlib.sha256(leaves[i]).digest() for i in range(1100))
nodes, _ = ops.merkle_build(c, ld, dev(lo))
mt = mo.Tree(leaves)
ok &= nodes.cpu().numpy().tobytes() == mt.nodes()
picks = list(range(0, 1024, 9))
sib, sides = ops.merkle_proofs(c, nodes, 1100, dev(np.array(picks, np.uint64)))
items = [leaves[i] for i in picks]
io = np.concatenate([[0], np.cumsum([len(x) for x in items])]).astype(np.uint64)
ok &= bool(ops.merkle_verify(c, nodes[-1].contiguous(), torch.frombuffer(bytearray(b"".join(items)), dtype=torch.uint8).cuda(),
                             dev(io), sib, sides).all())
print("sanitize_smoke", "OK" if ok else "MISMATCH")
sys.exit(0 if ok else 1)
