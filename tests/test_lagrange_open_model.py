"""CPU tier of the Lagrange-basis evaluation and opening (ronk_poly_lagrange_eval_u64 / _open_u64): the Python-integer
model of both formulas against the oracle's literal Lagrange evaluate, the oracle's division by [-z, 1] and Horner's rule,
the reference's kzg opening KAT through the Lagrange route, and the device batch inversion (batch_inv.cuh) run on the
CPU by tests/emu/bary_emu.cpp."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

import lagrange_model as lm
import oracle
from gpu_util import BABYBEAR, lagrange_closed_form

GL = oracle.GOLDILOCKS
_HERE = os.path.dirname(os.path.abspath(__file__))

# name → (p, g): g generates F_p*, so ω = g^((p-1)/n) has order n for every n | p - 1
FIELDS = {"f17": (17, 3), "f101": (101, 2), "f127": (127, 3), "babybear": (BABYBEAR, 31), "goldilocks": (GL, 7)}


def small_ns(p, cap=48):
    return [n for n in range(1, cap + 1) if (p - 1) % n == 0]


def points(p, g, n, s, rng):
    xs = lm.nodes(p, g, n, s)
    pts = {0, 1, p - 1, s % p, xs[0], xs[-1], xs[min(1, n - 1)]}
    pts |= {rng.randrange(p) for _ in range(3)}
    return sorted(pts)


@pytest.mark.parametrize("name", FIELDS)
def test_eval_matches_the_oracle_and_horner(name):
    p, g = FIELDS[name]
    rng = random.Random(p)
    for n in small_ns(p)[:12]:
        for s in (1, rng.randrange(1, p)):
            y = [rng.randrange(p) for _ in range(n)]
            a = lm.coefficients(p, g, y, s)
            assert [lm.horner(p, a, x) for x in lm.nodes(p, g, n, s)] == y
            for x in points(p, g, n, s, rng):
                got = lm.closed_form(p, g, y, x, s)
                on = x in lm.nodes(p, g, n, s)
                assert got == (0 if on else lm.horner(p, a, x)), (n, s, x)
                if s == 1:
                    assert got == lagrange_closed_form(p, g, y, x)
                    assert got == oracle.lagrange_eval(p, np.array(y, dtype=np.uint64), x, g=g), (n, x)


@pytest.mark.parametrize("name", FIELDS)
def test_quotient_matches_the_oracle_division(name):
    p, g = FIELDS[name]
    rng = random.Random(p + 1)
    for n in small_ns(p)[:12]:
        for s in (1, rng.randrange(1, p)):
            y = [rng.randrange(p) for _ in range(n)]
            a = lm.coefficients(p, g, y, s)
            xs = lm.nodes(p, g, n, s)
            for z in points(p, g, n, s, rng):
                v, q = lm.quotient(p, g, y, z, s)
                assert v == lm.horner(p, a, z)
                qm, r = oracle.poly_divrem(p, np.array(a, dtype=np.uint64), np.array([(p - z) % p, 1], dtype=np.uint64))
                assert int(r[0]) == v and not any(int(u) for u in r[1:])
                assert int(qm[-1]) == 0  # degree ≤ n - 2
                assert q == [lm.horner(p, qm, x) for x in xs], (n, s, z)


def test_node_rule_is_the_derivative():
    """q_k = f'(x_k) where z = x_k, on F_17 at n = 4, 8, 16 for every node."""
    p, g = 17, 3
    rng = random.Random(5)
    for n in (4, 8, 16):
        y = [rng.randrange(p) for _ in range(n)]
        a = lm.coefficients(p, g, y)
        da = [i * int(c) % p for i, c in enumerate(a)][1:]
        for k, xk in enumerate(lm.nodes(p, g, n)):
            assert lm.quotient(p, g, y, xk)[1][k] == lm.horner(p, da, xk)


def test_reference_kzg_opening_through_the_lagrange_route():
    """kzg/tests.rs:157-181: p(x) = (x-1)(x-2)(x-3) = [11, 11, 11, 1] over F_17 opened at z = 4 commits to (26, 45).
    Here 4 = ω_4^3 is a node, so the quotient's node rule decides the answer."""
    p = 17
    g = oracle.generator(p)
    coeffs = [11, 11, 11, 1]
    evals = [int(v) for v in oracle.fft(p, np.array(coeffs, dtype=np.uint64), g=g)]
    assert 4 in lm.nodes(p, g, 4)
    v, q = lm.quotient(p, g, evals, 4)
    assert v == lm.horner(p, coeffs, 4)
    qc = oracle.ifft(p, np.array(q, dtype=np.uint64), g=g)
    assert [int(c) for c in qc] == [3, 15, 1, 0]  # x^2 - 2x + 3
    g1, _ = oracle.setup()
    assert oracle.commit(np.array(qc, dtype=np.uint8), g1[:4]) == bytes([26, 0, 45, 0])


@pytest.fixture(scope="module")
def emu():
    csrc = os.path.join(_HERE, "..", "ronkathon_b200", "csrc")
    src = os.path.join(_HERE, "emu", "bary_emu.cpp")
    so = os.path.join(_HERE, "emu", "libbary_emu.so")
    deps = [src] + [os.path.join(csrc, h) for h in ("batch_inv.cuh", "field.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(x) for x in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", so, src])
    lib = C.CDLL(so)
    lib.emu_batch_invert.argtypes = [C.c_uint64, C.c_int, C.POINTER(C.c_uint64), C.c_size_t]
    return lib


@pytest.mark.parametrize("p,gl", [(GL, 1), (GL, 0), (BABYBEAR, 0), (0xFFFFFFFF70000001, 0), (17, 0), (101, 0)],
                         ids=["goldilocks", "goldilocks_mont", "babybear", "pbig", "f17", "f101"])
def test_batch_inversion_with_zeros_anywhere(emu, p, gl):
    K = emu.emu_bi_k()
    rng = np.random.default_rng(p % 1000)
    rows = []
    for pos in range(K):  # a zero at every position of a chunk
        r = [int(v) % (p - 1) + 1 for v in rng.integers(0, 2**63, K)]
        r[pos] = 0
        rows.append(r)
    rows.append([0] * K)
    rows.append([0 if i % 2 else int(rng.integers(1, min(p, 2**62))) for i in range(K)])
    rows.append([1] * (K - 1) + [p - 1])
    rows.append([int(v) % (p - 1) + 1 for v in rng.integers(0, 2**63, K)])
    vals = [v for r in rows for v in r]
    a = np.array(vals, dtype=np.uint64)
    assert emu.emu_batch_invert(p, gl, a.ctypes.data_as(C.POINTER(C.c_uint64)), len(a)) == 0
    assert [int(u) for u in a] == [pow(v, -1, p) if v else 0 for v in vals]
