"""The host-pointer (`_host`) entry points that run a device twin on staged copies of their arguments: the exact return
code of each argument check, and which check wins when several fail; outputs left unwritten when a call fails; the MSM
against its device twin; and a context's staging buffer growing for one large call and then serving smaller ones."""
import numpy as np
import pytest

import oracle
from gpu_util import BABYBEAR, GL, ctx, dev, msm_inputs

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5A5A5A5A5A5A5A5
TOO_LONG = 0x7FFFFFF1                      # one word past the division's length limit


def _raw(h, name, *args):
    """The return code of one call on context handle h (Context.call raises instead)."""
    from ronkathon_b200 import _lib
    return getattr(_lib.lib(), name)(h, *args)


def _rc(name, *args):
    return _raw(ctx()._h, name, *args)


def _p(x):
    from ronkathon_b200 import _lib
    return _lib._ptr(x)


def _codes():
    from ronkathon_b200 import _lib
    return _lib.OK, _lib.EINVAL, _lib.EUNSUPPORTED


def _untouched(*arrays):
    return all(np.all(a == SENTINEL) for a in arrays)


def test_field_host_return_codes():
    """ronk_field_{binop,unop,pow}_u64_host: null → EINVAL; n == 0 → OK before the modulus or the op is looked at;
    an unknown op → EINVAL before the modulus is; then the device checks.  A failed call leaves out unwritten."""
    OK, EINVAL, EUNSUP = _codes()
    n = 8
    a, b = oracle.splitmix(GL, 1, n), oracle.splitmix(GL - 1, 2, n) + 1
    out = np.full(n, SENTINEL, np.uint64)
    assert _raw(None, "ronk_field_binop_u64_host", 0, GL, _p(a), _p(b), _p(out), n) == EINVAL
    assert _rc("ronk_field_binop_u64_host", 0, GL, None, _p(b), _p(out), n) == EINVAL
    assert _rc("ronk_field_binop_u64_host", 0, GL, _p(a), _p(b), None, n) == EINVAL
    assert _rc("ronk_field_unop_u64_host", 0, GL, None, _p(out), n) == EINVAL
    assert _rc("ronk_field_pow_u64_host", GL, _p(a), 3, None, n) == EINVAL
    for p in (4, 2):                                                    # n == 0: no modulus check, no op check
        assert _rc("ronk_field_binop_u64_host", 0, p, None, None, None, 0) == OK
        assert _rc("ronk_field_binop_u64_host", 9, p, _p(a), _p(b), _p(out), 0) == OK
        assert _rc("ronk_field_unop_u64_host", 9, p, None, None, 0) == OK
        assert _rc("ronk_field_pow_u64_host", p, None, 3, None, 0) == OK
    for p in (GL, 2):                                                   # unknown op, before the modulus
        for op in (4, -1):
            assert _rc("ronk_field_binop_u64_host", op, p, _p(a), _p(b), _p(out), n) == EINVAL
        assert _rc("ronk_field_unop_u64_host", 2, p, _p(a), _p(out), n) == EINVAL
    for p, code in ((4, EINVAL), (2, EUNSUP)):                          # the device checks
        assert _rc("ronk_field_binop_u64_host", 2, p, _p(a), _p(b), _p(out), n) == code
        assert _rc("ronk_field_unop_u64_host", 0, p, _p(a), _p(out), n) == code
        assert _rc("ronk_field_pow_u64_host", p, _p(a), 3, _p(out), n) == code
    z = b.copy()
    z[-1] = 0
    assert _rc("ronk_field_binop_u64_host", 3, GL, _p(a), _p(z), _p(out), n) == EINVAL     # division by zero
    assert _rc("ronk_field_unop_u64_host", 1, GL, _p(z), _p(out), n) == EINVAL             # inverse of zero
    assert _untouched(out)
    assert _rc("ronk_field_binop_u64_host", 2, GL, _p(a), _p(b), _p(out), n) == OK
    assert np.array_equal(out, oracle.vec_mul(GL, a, b))


def test_poly_mul_host_return_codes():
    """ronk_poly_mul_u64_host: null → EINVAL; an empty operand → EINVAL, before the modulus; then the device checks."""
    OK, EINVAL, EUNSUP = _codes()
    a, b = oracle.splitmix(GL, 3, 5), oracle.splitmix(GL, 4, 3)
    c = np.full(7, SENTINEL, np.uint64)
    assert _raw(None, "ronk_poly_mul_u64_host", GL, 7, _p(a), 5, _p(b), 3, _p(c)) == EINVAL
    assert _rc("ronk_poly_mul_u64_host", GL, 7, None, 5, _p(b), 3, _p(c)) == EINVAL
    assert _rc("ronk_poly_mul_u64_host", GL, 7, _p(a), 5, _p(b), 3, None) == EINVAL
    for p in (GL, 2):
        assert _rc("ronk_poly_mul_u64_host", p, 7, _p(a), 0, _p(b), 3, _p(c)) == EINVAL
        assert _rc("ronk_poly_mul_u64_host", p, 7, _p(a), 5, _p(b), 0, _p(c)) == EINVAL
    assert _rc("ronk_poly_mul_u64_host", 4, 0, _p(a), 5, _p(b), 3, _p(c)) == EINVAL
    assert _rc("ronk_poly_mul_u64_host", 2, 0, _p(a), 5, _p(b), 3, _p(c)) == EUNSUP
    assert _untouched(c)
    assert _rc("ronk_poly_mul_u64_host", GL, 7, _p(a), 5, _p(b), 3, _p(c)) == OK
    assert np.array_equal(c, oracle.poly_mul(GL, a, b))


def test_poly_eval_and_dft_host_return_codes():
    """ronk_poly_eval_u64_host and ronk_dft_u64_host: null → EINVAL, then the device checks — m == 0 is OK for a
    prime and EINVAL for a composite p; a DFT of 0 points, of n ∤ p - 1 points or with g == 0 is EINVAL."""
    OK, EINVAL, EUNSUP = _codes()
    co, xs = oracle.splitmix(GL, 5, 6), oracle.splitmix(GL, 6, 3)
    out = np.full(15, SENTINEL, np.uint64)
    assert _raw(None, "ronk_poly_eval_u64_host", GL, _p(co), 6, _p(xs), 3, _p(out)) == EINVAL
    assert _rc("ronk_poly_eval_u64_host", GL, None, 6, _p(xs), 3, _p(out)) == EINVAL
    assert _rc("ronk_poly_eval_u64_host", GL, _p(co), 6, None, 3, _p(out)) == EINVAL
    assert _rc("ronk_poly_eval_u64_host", GL, None, 0, None, 0, None) == OK
    assert _rc("ronk_poly_eval_u64_host", 4, _p(co), 6, _p(xs), 0, _p(out)) == EINVAL
    assert _rc("ronk_poly_eval_u64_host", 2, _p(co), 6, _p(xs), 0, _p(out)) == EUNSUP
    a = oracle.splitmix(GL, 7, 15)
    assert _raw(None, "ronk_dft_u64_host", GL, 7, _p(a), 15, _p(out)) == EINVAL
    assert _rc("ronk_dft_u64_host", GL, 7, None, 15, _p(out)) == EINVAL
    assert _rc("ronk_dft_u64_host", GL, 7, _p(a), 15, None) == EINVAL
    assert _rc("ronk_dft_u64_host", GL, 7, _p(a), 0, _p(out)) == EINVAL
    assert _rc("ronk_dft_u64_host", GL, 7, _p(a), 7, _p(out)) == EINVAL   # 7 ∤ p - 1
    assert _rc("ronk_dft_u64_host", GL, 0, _p(a), 15, _p(out)) == EINVAL
    assert _rc("ronk_dft_u64_host", 4, 3, _p(a), 3, _p(out)) == EINVAL
    assert _rc("ronk_dft_u64_host", 2, 1, _p(a), 1, _p(out)) == EUNSUP
    assert _untouched(out)
    assert _rc("ronk_poly_eval_u64_host", GL, _p(co), 6, _p(xs), 3, _p(out)) == OK
    assert [int(v) for v in out[:3]] == [oracle.poly_eval_horner(GL, co, int(x)) for x in xs]
    assert _rc("ronk_dft_u64_host", GL, 7, _p(a), 15, _p(out)) == OK
    assert np.array_equal(out, oracle.dft(GL, a, g=7))


def test_divrem_host_return_codes():
    """ronk_poly_divrem_u64_host: null, then the modulus, then lengths above 0x7FFFFFF0, then da == 0 → OK; then the
    device checks.  A divisor the reference panics on leaves q and r unwritten; da < db with a nonzero top word
    launches nothing."""
    OK, EINVAL, EUNSUP = _codes()
    c = ctx()
    a, b = oracle.splitmix(GL, 8, 6), np.array([5, 2, 1], np.uint64)
    q, r = np.full(6, SENTINEL, np.uint64), np.full(6, SENTINEL, np.uint64)

    def rc(p, da, db, A=a, B=b, Q=q, R=r):
        return _rc("ronk_poly_divrem_u64_host", p, _p(A), da, _p(B), db, _p(Q), _p(R))

    assert _raw(None, "ronk_poly_divrem_u64_host", GL, _p(a), 6, _p(b), 3, _p(q), _p(r)) == EINVAL
    assert rc(GL, 6, 3, A=None) == EINVAL
    assert rc(GL, 6, 3, B=None) == EINVAL
    assert rc(GL, 6, 3, R=None) == EINVAL
    assert rc(4, 6, 3) == EINVAL
    assert rc(2, 6, 3) == EUNSUP
    assert rc(4, TOO_LONG, 3) == EINVAL                                 # the modulus before the length
    assert rc(GL, TOO_LONG, 3) == EUNSUP
    assert rc(GL, 0, TOO_LONG) == EUNSUP                                # the length before da == 0
    assert rc(GL, 0, 3, A=None, Q=None, R=None) == OK
    assert rc(4, 0, 3) == EINVAL                                        # the modulus before da == 0
    assert rc(GL, 6, 3, B=np.zeros(3, np.uint64)) == EINVAL             # all-zero divisor: the reference panics
    assert _untouched(q, r)
    assert rc(GL, 6, 3) == OK
    eq, er = oracle.poly_divrem(GL, a, b)
    assert np.array_equal(q, eq) and np.array_equal(r, er)
    before = c.launches
    for B in (b, np.array([5, 1], np.uint64)):                          # da < db, nonzero top word
        q1, r1 = np.full(1, SENTINEL, np.uint64), np.full(1, SENTINEL, np.uint64)
        assert rc(GL, 1, len(B), B=B, Q=q1, R=r1) == OK
        assert q1[0] == 0 and r1[0] == a[0]
    assert c.launches == before


@pytest.mark.parametrize("n", [1, 5, 4097])
def test_msm_host_equals_device(n):
    """ronk_msm_pluto_ext_host on the first n of n + 3 points equals ops.msm and the oracle on the same terms."""
    import torch
    from ronkathon_b200 import ops
    c = ctx()
    pts, sc = msm_inputs(n + 3)
    sc = np.ascontiguousarray(sc[:n])
    out = np.zeros(4, np.uint8)
    c.call("ronk_msm_pluto_ext_host", _p(pts), n + 3, _p(sc), n, _p(out))
    P, S = torch.from_numpy(pts.reshape(-1)).cuda(), torch.from_numpy(sc).cuda()
    assert out.tobytes() == ops.msm(c, P, S) == oracle.commit(sc, pts, fast=True)


def test_msm_host_return_codes():
    """ronk_msm_pluto_ext_host: null → EINVAL; n_points < n_scalars → EINVAL; n_scalars == 0 → Infinity; an off-curve
    point → EINVAL with out unwritten."""
    OK, EINVAL, _ = _codes()
    pts, sc = msm_inputs(4)
    out = np.zeros(4, np.uint8)
    assert _raw(None, "ronk_msm_pluto_ext_host", _p(pts), 4, _p(sc), 4, _p(out)) == EINVAL
    assert _rc("ronk_msm_pluto_ext_host", _p(pts), 4, _p(sc), 4, None) == EINVAL
    assert _rc("ronk_msm_pluto_ext_host", None, 4, _p(sc), 4, _p(out)) == EINVAL
    assert _rc("ronk_msm_pluto_ext_host", _p(pts), 3, _p(sc), 4, _p(out)) == EINVAL
    assert _rc("ronk_msm_pluto_ext_host", None, 0, None, 0, _p(out)) == OK
    assert out.tobytes() == oracle.INF
    out[:] = 0
    bad = pts.copy()
    bad[2] = (1, 0, 3, 0)                                               # x = 1: y² = 4, so y = 3 is off the curve
    assert not oracle.on_curve(bytes(bad[2]))
    assert _rc("ronk_msm_pluto_ext_host", _p(bad), 4, _p(sc), 4, _p(out)) == EINVAL
    assert not out.any()


def test_staging_buffer_grows_then_serves_smaller_calls():
    """On a fresh context: a small call, a 2^22-word call that grows the staging buffer, then small calls of other
    entry points and a second large one — every result exact."""
    import torch
    from ronkathon_b200 import Context
    c = Context(0, torch.cuda.current_stream().cuda_stream)
    try:
        def binop(op, p, a, b):
            out = np.empty(len(a), np.uint64)
            c.call("ronk_field_binop_u64_host", op, p, _p(a), _p(b), _p(out), len(a))
            return out

        a, b = oracle.splitmix(GL, 9, 1000), oracle.splitmix(GL, 10, 1000)
        assert np.array_equal(binop(2, GL, a, b), oracle.vec_mul(GL, a, b))
        big_a, big_b = oracle.splitmix(GL, 11, 1 << 22), oracle.splitmix(GL, 12, 1 << 22)
        assert np.array_equal(binop(2, GL, big_a, big_b), oracle.vec_mul(GL, big_a, big_b))
        pa, pb = oracle.splitmix(BABYBEAR, 13, 300), oracle.splitmix(BABYBEAR, 14, 200)
        prod = np.empty(499, np.uint64)
        c.call("ronk_poly_mul_u64_host", BABYBEAR, 31, _p(pa), 300, _p(pb), 200, _p(prod))
        assert np.array_equal(prod, oracle.poly_mul(BABYBEAR, pa, pb))
        q, r = np.empty(300, np.uint64), np.empty(300, np.uint64)
        c.call("ronk_poly_divrem_u64_host", BABYBEAR, _p(pa), 300, _p(pb[:7]), 7, _p(q), _p(r))
        eq, er = oracle.poly_divrem(BABYBEAR, pa, pb[:7])
        assert np.array_equal(q, eq) and np.array_equal(r, er)
        pts, sc = msm_inputs(5)
        out = np.empty(4, np.uint8)
        c.call("ronk_msm_pluto_ext_host", _p(pts), 5, _p(sc), 5, _p(out))
        assert out.tobytes() == oracle.commit(sc, pts, fast=True)
        neg = np.empty(1 << 22, np.uint64)
        c.call("ronk_field_unop_u64_host", 0, GL, _p(big_b), _p(neg), 1 << 22)
        assert np.array_equal(neg, oracle.poly_neg(GL, big_b))
    finally:
        c.close()
