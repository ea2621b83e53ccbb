"""ronk_poly_divrem_u64 / ops.poly_divrem: quotient_and_remainder on device pointers.

A divisor with a nonzero top word makes the division Euclidean, and where every transform of the plan divides p - 1
it runs as Newton iteration on the transforms (csrc/poly_div.cu).  Every other case keeps the path
ronk_poly_divrem_u64_host takes.  Results must equal the CPU oracle word for word, panics included."""
import ctypes as C

import numpy as np
import pytest

import oracle
from gpu_util import BABYBEAR, GL, MONT_PRIMES, ctx, dev, host

pytestmark = pytest.mark.gpu

# (p, g) whose 2-adicity covers every plan below (p2adic3 has only 8-point transforms)
NEWTON_PRIMES = {"gl": (GL, 7), **{n: (p, g) for n, (p, g, s) in MONT_PRIMES.items() if s >= 16}}
_DIV_LINEAR = ["div_linear_fold", "div_linear_carry", "div_linear_apply"]


def _generator(p):
    from ronkathon_b200 import _lib
    g = C.c_uint64()
    assert _lib.lib().ronk_field_generator(p, C.byref(g)) == 0
    return g.value


def _divisor(p, seed, db):
    b = oracle.splitmix(p, seed, db)
    b[-1] = b[-1] % (p - 1) + 1  # nonzero top word
    return b


def _dividends(p, seed, da):
    a = oracle.splitmix(p, seed, da)
    top0 = a.copy()
    top0[-min(da, 3):] = 0
    return {"random": a, "zero_top_words": top0, "zero": np.zeros(da, np.uint64)}


def _device(p, g, a, b, prof=False):
    """(q, r) as host arrays, or "panic"; with prof also the launch names of the call."""
    from ronkathon_b200 import RonkPanic, ops
    c = ctx()
    A, B = dev(a), dev(b)
    c.sync()
    if prof:
        c.prof_fetch()
        c.prof_enable(True)
    try:
        q, r = ops.poly_divrem(c, A, B, p=p, g=g)
        out = (host(q), host(r))
    except RonkPanic:
        out = "panic"
    finally:
        if prof:
            c.prof_enable(False)
    return (out, [n for n, _ in c.prof_fetch()]) if prof else out


def _host_variant(p, a, b):
    from ronkathon_b200 import RonkPanic, _lib
    q, r = np.empty(len(a), np.uint64), np.empty(len(a), np.uint64)
    try:
        ctx().call("ronk_poly_divrem_u64_host", p, _lib._ptr(a), len(a), _lib._ptr(b), len(b), _lib._ptr(q), _lib._ptr(r))
    except RonkPanic:
        return "panic"
    return q, r


def _oracle(p, a, b):
    try:
        return oracle.poly_divrem(p, a, b)
    except oracle.OraclePanic:
        return "panic"


def _same(got, exp):
    if isinstance(exp, str) or isinstance(got, str):
        return got == exp
    return np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1])


@pytest.mark.parametrize("name", list(NEWTON_PRIMES))
def test_newton_parity(name):
    """Random, zero-top-word and zero dividends against divisors of 1 … 4097 terms, quotient lengths at the doubling
    edges 2^k - 1, 2^k, 2^k + 1.  Wherever da >= db the call must run without the literal kernel, and with one Newton
    step per doubling of the inverse."""
    p, g = NEWTON_PRIMES[name]
    cases = {(da, db) for db in (1, 3, 17, 255, 256, 257, 4097) for da in (db - 1, db, db + 1, 2 * db, 5000, (1 << 14) + 3)}
    cases |= {(L + 16, 17) for k in (1, 2, 5, 10, 13) for L in ((1 << k) - 1, 1 << k, (1 << k) + 1)}
    for i, (da, db) in enumerate(sorted(cases)):
        b = _divisor(p, 1000 + i, db)
        for aname, a in _dividends(p, 2000 + i, da).items():
            got, names = _device(p, g, a, b, prof=True)
            assert _same(got, oracle.poly_divrem(p, a, b)), (name, da, db, aname)
            if da >= db:
                L = da - db + 1
                assert "poly_divrem" not in names, (name, da, db)
                assert names.count("divrem_newton_step") == (L - 1).bit_length(), (name, da, db, names)
            else:
                assert names == [], (name, da, db, names)


def test_non_newton_cases():
    """Divisors with a zero top word (a partly reduced remainder, the index panic, all zero), da < db, linear
    divisors, and g = 0: the same results as ronk_poly_divrem_u64_host and the oracle, panics included."""
    seen = set()
    for p, g in ((GL, 7), (BABYBEAR, MONT_PRIMES["babybear"][1]), (101, 2)):
        cases = [
            (oracle.splitmix(p, 1, 40), np.array([3, 5, 0], np.uint64)),        # trailing zero, reduces fully
            (oracle.splitmix(p, 2, 40), np.array([3, 5, 7, 0, 0], np.uint64)),  # trailing zeros
            (np.array([0, 0, 0, 0, 9], np.uint64), np.array([0, 0, 4, 0], np.uint64)),
            (oracle.splitmix(p, 3, 300), np.concatenate([oracle.splitmix(p, 4, 257), np.zeros(3, np.uint64)])),
            (oracle.splitmix(p, 5, 40), np.zeros(4, np.uint64)),                # all-zero divisor: panics
            (np.zeros(40, np.uint64), np.zeros(4, np.uint64)),                  # … unless the dividend is zero
            (oracle.splitmix(p, 6, 5), _divisor(p, 7, 9)),                      # da < db
            (oracle.splitmix(p, 8, 5000), np.array([p - 5, 1], np.uint64)),     # linear
            (oracle.splitmix(p, 9, 5000), _divisor(p, 10, 2)),
            (oracle.splitmix(p, 11, 1), _divisor(p, 12, 2)),
        ]
        for j, (a, b) in enumerate(cases):
            exp = _oracle(p, a, b)
            seen.add("panic" if isinstance(exp, str) else "ok")
            assert _same(_host_variant(p, a, b), exp), (p, j)
            assert _same(_device(p, g, a, b), exp), (p, j)
        # g = 0 (no transforms): the literal kernel, even where Newton iteration would fit
        a, b = oracle.splitmix(p, 13, 600), _divisor(p, 14, 70)
        got, names = _device(p, 0, a, b, prof=True)
        assert names == ["poly_divrem"] and _same(got, oracle.poly_divrem(p, a, b))
    assert seen == {"ok", "panic"}


def test_reference_kats(kats):
    """polynomial/tests.rs: b / a, b % a, a / b and (x² + 2x + 1) / (x + 1) in F_101, with g a generator (Newton
    iteration where the 4-point transforms of F_101 suffice) and with g = 0 (literal kernel); then the same
    generator-and-literal comparison with the oracle at p = 17 and 127, whose 2-adicity takes only small plans."""
    k = kats["polynomial"]
    p, a, b = k["p"], np.array(k["a"], np.uint64), np.array(k["b"], np.uint64)
    for g in (_generator(p), 0):
        q, r = _device(p, g, b, a)
        assert list(q) == k["b_div_a"] and list(r) == k["b_rem_a"]
        q, r = _device(p, g, a, b)
        assert list(q) == k["a_div_b"] and list(r) == k["a_rem_b"]
        q, r = _device(p, g, np.array([1, 2, 1], np.uint64), np.array([1, 1], np.uint64))
        assert list(q) == k["p121_div_11"] and list(r) == k["p121_rem_11"]
    for p in (101, 17, 127):
        paths = set()
        for g in (_generator(p), 0):
            for da, db in ((3, 3), (4, 3), (5, 3), (9, 3), (20, 3), (40, 5), (300, 17)):
                a, b = oracle.splitmix(p, da, da), _divisor(p, db, db)
                got, names = _device(p, g, a, b, prof=True)
                assert _same(got, oracle.poly_divrem(p, a, b)), (p, g, da, db)
                paths.add("literal" if names == ["poly_divrem"] else "newton")
        assert paths == {"literal", "newton"}, p


@pytest.mark.parametrize("p,g,da,db", [
    (GL, 7, 1 << 20, (1 << 19) + 1),
    (GL, 7, 1 << 24, (1 << 23) + 1),
    (GL, 7, 1 << 24, (1 << 12) + 1),
    (GL, 7, 1 << 22, 3),
    (BABYBEAR, MONT_PRIMES["babybear"][1], 1 << 22, (1 << 21) + 1),
], ids=["gl_2^20_2^19+1", "gl_2^24_2^23+1", "gl_2^24_2^12+1", "gl_2^22_3", "babybear_2^22_2^21+1"])
def test_identity_at_size(p, g, da, db):
    """a = b·q0 + r0 built on the device with poly_mul and poly_add; the division must return q0‖0 and r0‖0."""
    import torch
    from ronkathon_b200 import _lib, ops
    c = ctx()
    L = da - db + 1
    q0 = ops.splitmix_fill(c, L, 31, p)
    r0 = ops.splitmix_fill(c, db - 1, 32, p)
    b = ops.splitmix_fill(c, db, 33, p)
    b[-1] = 5
    prod = ops.poly_mul(c, b, q0, p=p, g=g)
    a = torch.empty_like(prod)
    c.call("ronk_poly_add_u64", p, _lib._ptr(prod), da, _lib._ptr(r0), db - 1, _lib._ptr(a))
    del prod
    q, r = ops.poly_divrem(c, a, b, p=p, g=g)
    c.sync()
    assert torch.equal(q[:L], q0) and not q[L:].any()
    assert torch.equal(r[:db - 1], r0) and not r[db - 1:].any()


def record(run):
    """Warm `run` once, then return (profile names of one profiled call, launches of one unprofiled call) — the method
    of test_gpu_launch_record.record."""
    c = ctx()
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
    run(c)
    c.sync()
    return names, c.launches - before


def _divrem_call(p, g, a, b):
    from ronkathon_b200 import ops
    A, B = dev(a), dev(b)
    return lambda c: ops.poly_divrem(c, A, B, p=p, g=g)


@pytest.mark.parametrize("name", ["gl", "babybear"])
def test_launch_record(name):
    p, g = NEWTON_PRIMES[name]
    a = oracle.splitmix(p, 27, 3000)
    names, launches = record(_divrem_call(p, g, a, _divisor(p, 28, 17)))
    assert launches == len(names)
    assert "poly_divrem" not in names
    assert names[:2] == ["divrem_reverse", "divrem_reverse"] and names.count("divrem_newton_step") == 12
    assert names[-1] == "poly_sub"
    low = np.zeros(3000, np.uint64)
    low[:2] = a[:2]  # degree below the divisor's: the reference's loop stops before it indexes out of range
    names, launches = record(_divrem_call(p, g, low, np.array([5, 2, 1, 0], np.uint64)))
    assert names == ["poly_divrem"] and launches == 1
    names, launches = record(_divrem_call(p, g, a, np.array([5, 1], np.uint64)))
    assert names == _DIV_LINEAR and launches == 3
    names, launches = record(_divrem_call(p, g, a[:10], _divisor(p, 29, 17)))  # da < db: copies only
    assert names == [] and launches == 0


def test_argument_checks():
    """Null pointers and q / r overlapping a, b or each other are refused before anything is written."""
    import torch
    from ronkathon_b200 import RonkPanic, _lib
    c = ctx()
    da, db = 64, 5
    a, b = dev(oracle.splitmix(GL, 40, da)), dev(_divisor(GL, 41, db))
    q, r = torch.full((da,), 77, dtype=torch.int64, device="cuda"), torch.full((da,), 88, dtype=torch.int64, device="cuda")
    a0, b0 = a.clone(), b.clone()
    buf = torch.full((2 * da,), 99, dtype=torch.int64, device="cuda")

    def refused(aa, bb, qq, rr, ddb=db):
        with pytest.raises(RonkPanic):
            c.call("ronk_poly_divrem_u64", GL, 7, _lib._ptr(aa), da, _lib._ptr(bb), ddb, _lib._ptr(qq), _lib._ptr(rr))

    refused(None, b, q, r)
    refused(a, None, q, r)
    refused(a, b, None, r)
    refused(a, b, q, None)
    refused(a, b, a, r)            # q aliases a
    refused(a, b, q, b)            # r aliases b
    refused(a, b, q, q)            # r aliases q
    refused(a, b, buf, buf[da // 2:])  # q and r overlap
    refused(a, b, a[1:], r)        # q overlaps a
    c.sync()
    assert torch.equal(a, a0) and torch.equal(b, b0)
    assert not (q != 77).any() and not (r != 88).any() and not (buf != 99).any()
    # da == 0: nothing to do, nothing written
    c.call("ronk_poly_divrem_u64", GL, 7, None, 0, _lib._ptr(b), db, None, None)
