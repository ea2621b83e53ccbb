"""The full launch sequence of each polynomial path built on the transforms: the profile names one warmed call records,
in order, and the launch count it adds, for ronk_poly_mul_u64 (schoolbook, single-tile, two-pass and bounded three-pass
transforms, the multi-modular path at one, two and three auxiliary primes, Goldilocks with a generator other than 7),
ronk_poly_mul_batch_u64 on the multi-modular path, ronk_poly_divrem_u64 on the Newton path in each remainder branch,
multipoint evaluation and interpolation on the subproduct tree, and Bluestein's transform.

tests/golden/poly_launch_sequences.json holds the sequences; `python tests/test_gpu_poly_launch_sequences.py` on an H100
rewrites it.  The host code that plans these launches (transform sizes, scratch, reversals, recombination) is shared
between the paths, and a change to it must leave every sequence as it is.  Each case also checks its words against
the oracle."""
import json
import os
import sys

import numpy as np
import pytest

_HERE = os.path.dirname(os.path.abspath(__file__))
for _d in (_HERE, os.path.dirname(_HERE)):   # run as a script: the helpers here and the package at the root
    if _d not in sys.path:
        sys.path.insert(0, _d)

import oracle  # noqa: E402
from gpu_util import BABYBEAR, GL, MONT_PRIMES, ctx, dev  # noqa: E402

FIXTURE = os.path.join(_HERE, "golden", "poly_launch_sequences.json")
BB_G = MONT_PRIMES["babybear"][1]
GL_G5 = MONT_PRIMES["gl_g5"][1]
M31 = (1 << 31) - 1
BETWEEN = 0xFFFFFFFF0000002F   # prime, q1 = Goldilocks < p < q2 = 0xFFFFFFFF70000001: reductions for q1 and q3 only
ABOVE = (1 << 64) - 279        # prime above every auxiliary prime: a reduction for each
_tree = None


def tree_ctx():
    """A context on the suite's stream that takes the subproduct tree wherever its transforms fit."""
    global _tree
    if _tree is None:
        import torch
        from ronkathon_b200 import Context
        ctx()
        old = os.environ.get("RONK_TREE_MIN")
        os.environ["RONK_TREE_MIN"] = "1"
        try:
            _tree = Context(0, torch.cuda.current_stream().cuda_stream)
        finally:
            if old is None:
                del os.environ["RONK_TREE_MIN"]
            else:
                os.environ["RONK_TREE_MIN"] = old
    return _tree


def _host(c, t):
    from ronkathon_b200 import ops
    c.sync()
    return ops.to_host(t)


def _product(p, g, a, b):
    """a·b: the oracle's schoolbook product, or above 2^22 multiplies its transforms (g of order p - 1)."""
    if len(a) * len(b) <= 1 << 22:
        return oracle.poly_mul(p, a, b)
    L = len(a) + len(b) - 1
    n = 1 << (L - 1).bit_length()
    A, B = np.zeros(n, np.uint64), np.zeros(n, np.uint64)
    A[:len(a)], B[:len(b)] = a, b
    spectrum = oracle.vec_mul(p, oracle.ntt_fast(p, A, g=g), oracle.ntt_fast(p, B, g=g))
    return oracle.ntt_fast(p, spectrum, inverse=True, g=g)[:L]


def _mul(p, g, da, db, seed):
    from ronkathon_b200 import ops
    a, b = oracle.splitmix(p, seed, da), oracle.splitmix(p, seed + 1, db)
    A, B = dev(a), dev(b)

    def check(c, out):
        assert np.array_equal(_host(c, out), _product(p, g, a, b))
    return (lambda c: ops.poly_mul(c, A, B, p=p, g=g)), check


def _mul_batch(p, g, rows, da, db, shared, seed):
    from ronkathon_b200 import ops
    a = oracle.splitmix(p, seed, rows * da).reshape(rows, da)
    b = oracle.splitmix(p, seed + 1, db if shared else rows * db).reshape((db,) if shared else (rows, db))
    A, B = dev(a), dev(b)

    def check(c, out):
        got = _host(c, out).reshape(rows, da + db - 1)
        for r in range(rows):
            assert np.array_equal(got[r], oracle.poly_mul(p, a[r], b if shared else b[r])), r
    return (lambda c: ops.poly_mul_batch(c, A, B, p=p, g=g)), check


def _divrem(p, g, da, db, seed):
    from ronkathon_b200 import ops
    a, b = oracle.splitmix(p, seed, da), oracle.splitmix(p, seed + 1, db)
    b[-1] = b[-1] or 1   # a nonzero top word: the Newton path
    A, B = dev(a), dev(b)

    def check(c, out):
        q, r = oracle.poly_divrem(p, a, b)
        assert np.array_equal(_host(c, out[0]), q) and np.array_equal(_host(c, out[1]), r)
    return (lambda c: ops.poly_divrem(c, A, B, p=p, g=g)), check


def _points(p, k, seed):
    xs = oracle.splitmix(p, seed, k)
    assert len(set(xs.tolist())) == k
    return xs


def _multieval(p, g, d, m, seed):
    """Checked at up to 512 of the m points (the oracle's Horner takes d steps per point)."""
    from ronkathon_b200 import ops
    coeffs, xs = oracle.splitmix(p, seed, d), _points(p, m, seed + 1)
    Cf, X = dev(coeffs), dev(xs)

    def check(c, out):
        got = _host(c, out)
        for i in sorted(set(range(0, m, max(1, m // 512))) | {m - 1}):
            assert int(got[i]) == oracle.poly_eval(p, coeffs, int(xs[i])), i
    return (lambda c: ops.poly_multieval(c, Cf, X, p=p, g=g)), check


def _interpolate(p, g, k, seed):
    """The interpolant has k coefficients, so agreeing with ys at the k distinct points pins every word."""
    from ronkathon_b200 import ops
    xs, ys = _points(p, k, seed), oracle.splitmix(p, seed + 1, k)
    X, Y = dev(xs), dev(ys)

    def check(c, out):
        got = _host(c, out)
        assert all(oracle.poly_eval(p, got, int(xs[i])) == int(ys[i]) for i in range(k))
    return (lambda c: ops.poly_interpolate(c, X, Y, p=p, g=g)), check


def _ntt_any(p, g, n, inverse, seed):
    """X_k = a(ω^k), ω = g^((p-1)/n); the inverse n^-1·a(ω^-k).  Checked with the oracle's evaluation at up to 512 of the
    n indices (its dft takes n² modular powers)."""
    from ronkathon_b200 import ops
    a = oracle.splitmix(p, seed, n)
    A = dev(a)
    w = pow(g, (p - 1) // n, p)
    w, scale = (pow(w, p - 2, p), pow(n, p - 2, p)) if inverse else (w, 1)

    def check(c, out):
        got = _host(c, out)
        for k in sorted(set(range(0, n, max(1, n // 512))) | {1, n - 1}):
            assert int(got[k]) == scale * oracle.poly_eval(p, a, pow(w, k, p)) % p, k
    return (lambda c: ops.ntt_any_(c, A.clone(), n, inverse=inverse, p=p, g=g)), check


CASES = {
    # id: (context: "default" or "tree", factory of (call, check))
    "mul_schoolbook_gl": ("default", lambda: _mul(GL, 7, 64, 64, 100)),
    "mul_schoolbook_gl_g5": ("default", lambda: _mul(GL, GL_G5, 64, 64, 102)),
    "mul_schoolbook_babybear": ("default", lambda: _mul(BABYBEAR, BB_G, 64, 64, 104)),
    "mul_single_gl": ("default", lambda: _mul(GL, 7, 256, 256, 106)),
    "mul_single_gl_g5": ("default", lambda: _mul(GL, GL_G5, 256, 256, 108)),
    "mul_single_babybear": ("default", lambda: _mul(BABYBEAR, BB_G, 256, 256, 110)),
    "mul_two_pass_babybear_2^20": ("default", lambda: _mul(BABYBEAR, BB_G, 1 << 19, (1 << 19) + 1, 112)),
    "mul_three_pass_gl_2^21x2^21": ("default", lambda: _mul(GL, 7, 1 << 21, 1 << 21, 114)),
    "mul_crt_k1_f101": ("default", lambda: _mul(101, 2, 256, 256, 116)),
    "mul_crt_k2_m31": ("default", lambda: _mul(M31, 7, 1024, 1024, 118)),
    "mul_crt_k3_between_q1_q2": ("default", lambda: _mul(BETWEEN, 3, 1024, 1024, 120)),
    "mul_crt_k3_above_all": ("default", lambda: _mul(ABOVE, 5, 1024, 1024, 122)),
    "mul_batch_crt_f101_shared": ("default", lambda: _mul_batch(101, 2, 64, 64, 64, True, 130)),
    "mul_batch_crt_f101": ("default", lambda: _mul_batch(101, 2, 64, 64, 64, False, 132)),
    "mul_batch_crt_above_all_long": ("default", lambda: _mul_batch(ABOVE, 5, 2, 2048, 2048, False, 134)),
    # L = da - db + 1 against rw = db - 1 and the remainder transform's N = 2^⌈log2 rw⌉
    "divrem_low_product": ("default", lambda: _divrem(GL, 7, 3000, 1000, 140)),
    "divrem_low_product_babybear": ("default", lambda: _divrem(BABYBEAR, BB_G, 3000, 1000, 142)),
    "divrem_cyclic_db_above_n": ("default", lambda: _divrem(GL, 7, 1500, 1025, 144)),
    "divrem_cyclic_da_above_n": ("default", lambda: _divrem(GL, 7, 1500, 1000, 146)),
    "divrem_cyclic_no_fold": ("default", lambda: _divrem(GL, 7, 1010, 1000, 148)),
    "divrem_constant_divisor": ("default", lambda: _divrem(GL, 7, 3000, 1, 150)),
    "multieval_tree_d_above_k": ("tree", lambda: _multieval(GL, 7, 300, 100, 160)),
    "multieval_tree_d_below_k": ("tree", lambda: _multieval(GL, 7, 100, 300, 162)),
    "multieval_tree_babybear": ("tree", lambda: _multieval(BABYBEAR, BB_G, 1000, 700, 164)),
    "multieval_default_d_above_k": ("default", lambda: _multieval(GL, 7, 40000, 1 << 15, 166)),
    "multieval_default_d_below_k": ("default", lambda: _multieval(GL, 7, 1 << 15, 40000, 168)),
    "interpolate_tree": ("tree", lambda: _interpolate(GL, 7, 300, 170)),
    "interpolate_default": ("default", lambda: _interpolate(GL, 7, 2048, 172)),
    "ntt_any_bluestein_gl": ("default", lambda: _ntt_any(GL, 7, 4080, False, 180)),
    "ntt_any_bluestein_gl_inverse": ("default", lambda: _ntt_any(GL, 7, 4080, True, 182)),
    "ntt_any_bluestein_babybear": ("default", lambda: _ntt_any(BABYBEAR, BB_G, 15 << 9, False, 184)),
}


def record(c, run):
    """Warm `run` once, then (profile names of one profiled call, launches of one unprofiled call, its output)."""
    run(c)
    c.sync()
    c.prof_fetch()
    c.prof_enable(True)
    try:
        run(c)
        names = [n for n, _ in c.prof_fetch()]
    finally:
        c.prof_enable(False)
    before = c.launches
    out = run(c)
    c.sync()
    return names, c.launches - before, out


def _run_case(case):
    kind, factory = CASES[case]
    c = tree_ctx() if kind == "tree" else ctx()
    run, check = factory()
    names, launches, out = record(c, run)
    check(c, out)
    return names, launches


def test_fixture_lists_every_case():
    with open(FIXTURE) as f:
        assert sorted(json.load(f)) == sorted(CASES)


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_launch_sequence(case):
    with open(FIXTURE) as f:
        want = json.load(f)[case]
    names, launches = _run_case(case)
    assert names == want["names"]
    assert launches == want["launches"]


if __name__ == "__main__":
    seqs = {}
    for case in CASES:
        names, launches = _run_case(case)
        seqs[case] = {"names": names, "launches": launches}
        print(f"{case}: {launches} launches", flush=True)
    with open(FIXTURE, "w") as f:
        json.dump(seqs, f, indent=1)
        f.write("\n")
