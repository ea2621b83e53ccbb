"""ronk_poly_mul_u64's multi-modular path (poly_crt.cu) on the device.

A product over a prime whose p - 1 has no power-of-two root of the product's length is convolved modulo k ≤ 3
auxiliary NTT primes and rebuilt by the Chinese remainder theorem.  Its words must be the schoolbook kernel's.  The
checks: the oracle's schoolbook product where that is cheap; all-(p - 1) operands, whose integer coefficients reach the
bound min(da, db)·(p - 1)² exactly and whose product is count_j mod p in closed form, since (p - 1)² ≡ 1; and the end
coefficients with c(x) = a(x)·b(x) at random points.  A context created with RONK_CRT_MUL_MIN=1 takes the path wherever
it fits; the suite's context uses the measured crossovers."""
import os

import numpy as np
import pytest

import oracle
from gpu_util import GL, MONT_PRIMES, ctx, dev, host
from test_crt_mul_model import Q, is_prime, prime_count

pytestmark = pytest.mark.gpu

EINVAL, EUNSUPPORTED = 1, 5
REFERENCE = {"f101": (101, 2), "f17": (17, 3), "f127": (127, 3)}
_forced = None


def _context(env, stream=None):
    import torch
    from ronkathon_b200 import Context
    ctx()
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return Context(0, (stream or torch.cuda.current_stream()).cuda_stream)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def forced():
    """A context on the suite's stream that takes the multi-modular path wherever it fits."""
    global _forced
    if _forced is None:
        _forced = _context({"RONK_CRT_MUL_MIN": "1"})
    return _forced


def profiled(c, fn):
    """(fn(), the profile names of the launches it made on c)."""
    c.sync()
    c.prof_fetch()
    c.prof_enable(True)
    try:
        out = fn()
        names = [n for n, _ in c.prof_fetch()]
    finally:
        c.prof_enable(False)
    return out, names


def trapezoid(p, da, db):
    """The product of all-(p - 1) operands: coefficient j is the number of index pairs summing to j, mod p."""
    L = da + db - 1
    i = np.arange(L, dtype=np.uint64)
    return np.minimum(np.minimum(i + np.uint64(1), np.uint64(min(da, db))), np.uint64(L) - i) % np.uint64(p)


def mul_const(c, p, g, da, db, va, vb):
    from ronkathon_b200 import ops
    return host(ops.poly_mul(c, dev(np.full(da, va, dtype=np.uint64)), dev(np.full(db, vb, dtype=np.uint64)), p, g))


def check_trapezoid(c, p, g, da, db):
    got = mul_const(c, p, g, da, db, p - 1, p - 1)
    assert len(got) == da + db - 1 and np.array_equal(got, trapezoid(p, da, db)), (p, da, db)


def check_random(c, p, g, da, db, seed, points=4):
    """Random operands: the length, both end coefficients and c(x) = a(x)·b(x) at random points (oracle Horner)."""
    from ronkathon_b200 import ops
    A, B = ops.splitmix_fill(ctx(), da, seed, p), ops.splitmix_fill(ctx(), db, seed + 1, p)
    got, a, b = host(ops.poly_mul(c, A, B, p, g)), host(A), host(B)
    assert len(got) == da + db - 1
    assert int(got[0]) == oracle.mul(p, int(a[0]), int(b[0])) and int(got[-1]) == oracle.mul(p, int(a[-1]), int(b[-1]))
    for x in oracle.splitmix(p, seed + 2, points):
        x = int(x)
        assert oracle.poly_eval_horner(p, got, x) == oracle.mul(p, oracle.poly_eval_horner(p, a, x),
                                                                oracle.poly_eval_horner(p, b, x)), (p, da, db, x)


def _prime_3_mod_4_below(x):
    """The largest prime p < x with p ≡ 3 (mod 4): 2-adicity 1, so no transform of the product fits p - 1."""
    p = x - 1 - ((x - 1 - 3) % 4)
    while not is_prime(p):
        p -= 4
    return p


def _prime_between(lo, hi):
    p = lo + 2
    while p < hi and not (is_prime(p) and (p - 1) % 512):
        p += 2
    assert p < hi
    return p


# ---- the reference's fields -------------------------------------------------------------------------------------------
SMALL_SHAPES = [(1, 5000), (5000, 1), (3, 17), (100, 7), (3001, 8191), (8192, 8192)]   # L = 20 > 16: no 2-power root of 17 either


@pytest.mark.parametrize("da,db", SMALL_SHAPES, ids=[f"{a}x{b}" for a, b in SMALL_SHAPES])
@pytest.mark.parametrize("field", list(REFERENCE))
def test_reference_fields_match_the_oracle(field, da, db):
    from ronkathon_b200 import ops
    p, g = REFERENCE[field]
    a, b = oracle.splitmix(p, 1, da), oracle.splitmix(p, 2, db)
    got, names = profiled(forced(), lambda: host(ops.poly_mul(forced(), dev(a), dev(b), p, g)))
    assert names[-1] == "crt_combine" and "poly_mul_schoolbook" not in names
    assert np.array_equal(got, oracle.poly_mul(p, a, b))


@pytest.mark.parametrize("log_m", [20, 25])
@pytest.mark.parametrize("field", list(REFERENCE))
def test_reference_fields_at_the_bound(field, log_m):
    """2^20 and 2^25 squared (L = 2^26 - 1, the longest product the path takes), on the measured crossover too."""
    p, g = REFERENCE[field]
    check_trapezoid(forced(), p, g, 1 << log_m, 1 << log_m)
    if log_m == 20:
        check_trapezoid(ctx(), p, g, 1 << log_m, (1 << log_m) - 3)
        check_random(forced(), p, g, 1 << log_m, (1 << log_m) + 17, 10)


# ---- the prime count at its edges ---------------------------------------------------------------------------------------
# A prime near 2^25 (resp. 2^57) with 2-adicity 1, and the largest min(da, db) that one (resp. two) auxiliary primes
# cover: about 2^14 terms either way.  With one prime too few, the middle coefficients wrap.
B1 = _prime_3_mod_4_below(1 << 25)
B2 = _prime_3_mod_4_below(1 << 57)
EDGES = {"1to2": (B1, (Q[0] - 1) // (B1 - 1) ** 2, 1), "2to3": (B2, (Q[0] * Q[1] - 1) // (B2 - 1) ** 2, 2)}


@pytest.mark.parametrize("edge", list(EDGES))
def test_prime_count_boundary(edge):
    p, m, k = EDGES[edge]
    assert 1 << 12 < m < 1 << 16
    assert prime_count(p, m) == k and prime_count(p, m + 1) == k + 1
    for da, db in ((m, m), (m + 1, m + 1), (m, m + 7), (m + 1, 3 * m)):
        check_trapezoid(forced(), p, 3, da, db)
        check_trapezoid(ctx(), p, 3, da, db)


# ---- moduli above the auxiliary primes ----------------------------------------------------------------------------------
ABOVE = {"2^64-279": ((1 << 64) - 279, 5), "2^64-59": ((1 << 64) - 59, 2)}


@pytest.mark.parametrize("name", list(ABOVE))
def test_moduli_above_every_auxiliary_prime(name):
    """Operands near p - 1, so that every reduction kernel has words to reduce (p > q1, q2, q3)."""
    from ronkathon_b200 import ops
    p, g = ABOVE[name]
    rng = np.random.default_rng(3)
    for da, db in ((3000, 2500), (1, 4000), (4097, 2)):
        a = np.uint64(p - 1) - rng.integers(0, 1 << 20, da, dtype=np.uint64)
        b = np.uint64(p - 1) - rng.integers(0, 1 << 40, db, dtype=np.uint64)
        got, names = profiled(forced(), lambda: host(ops.poly_mul(forced(), dev(a), dev(b), p, g)))
        assert names.count("crt_reduce") == 3 and names[-1] == "crt_combine"
        assert np.array_equal(got, oracle.poly_mul(p, a, b)), (da, db)
    check_trapezoid(forced(), p, g, (1 << 18) + 3, 1 << 17)
    check_random(ctx(), p, g, 1 << 19, (1 << 19) + 1, 20)


# ---- NTT primes past their two-adicity ----------------------------------------------------------------------------------
def test_p32_past_its_two_adicity():
    """4295294977 has 2^16: (2^15 + 1)² needs 2^17 points."""
    p, g, s = MONT_PRIMES["p32"]
    assert s == 16
    check_trapezoid(ctx(), p, g, (1 << 15) + 1, (1 << 15) + 1)
    _, names = profiled(ctx(), lambda: check_random(ctx(), p, g, (1 << 15) + 1, (1 << 15) + 1, 30))
    assert "crt_combine" in names and "poly_mul_schoolbook" not in names
    check_random(ctx(), p, g, 1 << 20, (1 << 20) + 3, 31)


def test_koalabear_past_its_two_adicity():
    """127·2^24 + 1: products of 2^24 + 1 … 2^26 - 1 coefficients."""
    p, g, s = MONT_PRIMES["koalabear"]
    assert s == 24
    check_random(ctx(), p, g, (1 << 23) + 1, (1 << 23) + 1, 40)
    check_trapezoid(ctx(), p, g, 1 << 25, 1 << 25)
    check_trapezoid(forced(), p, g, (1 << 24) + 5, 1 << 20)


def test_three_primes_at_the_bound():
    """k = 3 at the longest product (2^25 × 2^25, L = 2^26 - 1) over a modulus above every auxiliary prime: three reductions
    and nine bounded transforms of 2^26 points, with the largest scratch the path takes."""
    p, g = ABOVE["2^64-59"]
    assert prime_count(p, 1 << 25) == 3
    check_trapezoid(ctx(), p, g, 1 << 25, 1 << 25)


# ---- the output over an operand ---------------------------------------------------------------------------------------
ALIAS = {"direct_gl": (GL, 7, 3000, 2000), "crt_k1_f101": (101, 2, 3000, 2000),
         "crt_k3_reduced": ((1 << 64) - 59, 2, 3000, 2000)}


@pytest.mark.parametrize("over", ["a", "b"])
@pytest.mark.parametrize("case", list(ALIAS))
def test_output_may_alias_an_operand(case, over):
    """On the transform paths (the direct one and the multi-modular one, with and without reductions) c may start where a
    or b does: both are consumed before the last launch writes c."""
    import torch
    from ronkathon_b200 import _lib
    p, g, da, db = ALIAS[case]
    a, b = oracle.splitmix(p, 95, da), oracle.splitmix(p, 96, db)
    L = da + db - 1
    buf = dev(np.concatenate([a if over == "a" else b, np.zeros(L - (da if over == "a" else db), dtype=np.uint64)]))
    other = dev(b if over == "a" else a)
    pa, pb = (buf, other) if over == "a" else (other, buf)
    _, names = profiled(ctx(), lambda: ctx().call("ronk_poly_mul_u64", p, g, _lib._ptr(pa), da, _lib._ptr(pb), db,
                                                  _lib._ptr(buf)))
    assert "poly_mul_schoolbook" not in names and (case == "direct_gl") == ("crt_combine" not in names)
    assert isinstance(buf, torch.Tensor) and np.array_equal(host(buf), oracle.poly_mul(p, a, b))


# ---- launch sequences ---------------------------------------------------------------------------------------------------
_PER_PRIME = ["ntt_single", "ntt_single", "intt_single"]
M31, M61 = (1 << 31) - 1, (1 << 61) - 1
BETWEEN = _prime_between(Q[0], Q[1])   # q1 < p < q2: reductions for q1 and q3 only
SEQUENCES = {
    "k1_f101": (101, 2, _PER_PRIME),
    "k2_m31": (M31, 7, _PER_PRIME * 2),
    "k3_m61": (M61, 37, _PER_PRIME * 3),
    "k3_above_q3": ((1 << 63) + 29, 2, _PER_PRIME * 2 + ["crt_reduce"] + _PER_PRIME),
    "k3_between_q1_q2": (BETWEEN, 3, ["crt_reduce"] + _PER_PRIME * 2 + ["crt_reduce"] + _PER_PRIME),
    "k3_above_all": ((1 << 64) - 59, 2, (["crt_reduce"] + _PER_PRIME) * 3),
}


def record(c, run):
    """Warm run once; then (profile names of one profiled call, launches of one unprofiled call)."""
    run()
    _, names = profiled(c, run)
    before = c.launches
    run()
    c.sync()
    return names, c.launches - before


@pytest.mark.parametrize("case", list(SEQUENCES))
def test_launch_sequence(case):
    """200 × 200 (512-point transforms): per auxiliary prime the reduction where q_i < p and three transforms, then one
    crt_combine.  The words are the oracle's."""
    from ronkathon_b200 import ops
    p, g, per = SEQUENCES[case]
    a, b = oracle.splitmix(p, 5, 200), oracle.splitmix(p, 6, 200)
    a[:3], b[:3] = p - 1, p - 1
    A, B = dev(a), dev(b)
    out = []
    names, launches = record(forced(), lambda: out.append(ops.poly_mul(forced(), A, B, p, g)))
    assert names == per + ["crt_combine"] and launches == len(names)
    assert np.array_equal(host(out[-1]), oracle.poly_mul(p, a, b))


SCHOOLBOOK = ["g0", "below_crossover", "short_operand_f101", "short_operand_k3", "longer_than_2^26"]


@pytest.mark.parametrize("case", SCHOOLBOOK)
def test_schoolbook_stays(case):
    """g = 0, a product below the measured da·db crossover, products whose da·db passes it but whose shorter operand is
    below the measured short-side crossover (255 × 2^16 over F_101, 2 × 2^20 over 2^64 - 279), and L > 2^26 launch only
    the schoolbook kernel."""
    from ronkathon_b200 import ops
    p = 101
    if case == "g0":
        c, g, da, db = forced(), 0, 300, 300
    elif case == "below_crossover":
        c, g, da, db = ctx(), 2, 8, 8
    elif case == "short_operand_f101":
        c, g, da, db = ctx(), 2, 255, 1 << 16
    elif case == "short_operand_k3":
        c, g, da, db, p = ctx(), 5, 2, 1 << 20, (1 << 64) - 279
    else:
        c, g, da, db = forced(), 2, 1 << 26, 2
    A, B = ops.splitmix_fill(ctx(), da, 7, p), ops.splitmix_fill(ctx(), db, 8, p)
    out = []
    names, launches = record(c, lambda: out.append(ops.poly_mul(c, A, B, p, g)))
    assert names == ["poly_mul_schoolbook"] and launches == 1
    got, a, b = host(out[-1]), host(A), host(B)
    if da * db <= 1 << 24:
        assert np.array_equal(got, oracle.poly_mul(p, a, b))
    else:
        j = da // 2
        assert int(got[j]) == (int(a[j]) * int(b[0]) + int(a[j - 1]) * int(b[1])) % p
        assert int(got[-1]) == int(a[-1]) * int(b[-1]) % p


# ---- interfaces ---------------------------------------------------------------------------------------------------------
def test_host_variant():
    from ronkathon_b200 import _lib
    p, g = 101, 2
    for da, db in ((4000, 3000), (1, 1 << 16)):
        a, b = oracle.splitmix(p, 50, da), oracle.splitmix(p, 51, db)
        out = np.empty(da + db - 1, dtype=np.uint64)
        _, names = profiled(forced(), lambda: forced().call("ronk_poly_mul_u64_host", p, g, _lib._ptr(a), da, _lib._ptr(b),
                                                            db, _lib._ptr(out)))
        assert names[-1] == "crt_combine"
        assert np.array_equal(out, oracle.poly_mul(p, a, b))


def test_polynomial_mul_over_f101():
    """Polynomial.__mul__ over PrimeField(101) (g = 2) at 2^16 terms, on the suite's default context."""
    from ronkathon_b200 import Polynomial, PrimeField
    F = PrimeField(101)
    p = 101
    a, b = oracle.splitmix(p, 60, 1 << 16), oracle.splitmix(p, 61, 1 << 16)
    pa, pb = Polynomial([int(v) for v in a], F), Polynomial([int(v) for v in b], F)
    assert pa.g == 2
    prod, names = profiled(ctx(), lambda: pa * pb)
    assert names[-1] == "crt_combine"
    got = np.asarray(prod.coefficients, dtype=np.uint64)
    assert len(got) == (1 << 17) - 1
    assert int(got[0]) == int(a[0]) * int(b[0]) % p and int(got[-1]) == int(a[-1]) * int(b[-1]) % p
    for x in (3, 50, 97):
        assert oracle.poly_eval_horner(p, got, x) == oracle.poly_eval_horner(p, a, x) * oracle.poly_eval_horner(p, b, x) % p


def test_error_codes():
    """The checks before any path is chosen answer as they always have, on sizes the multi-modular path would take."""
    from ronkathon_b200 import RonkError, _lib
    c = forced()
    a = dev(oracle.splitmix(101, 70, 5000))
    out = dev(np.zeros(9999, dtype=np.uint64))
    cases = [((101, 2, None, 5000, _lib._ptr(a), 5000, _lib._ptr(out)), EINVAL),      # null operand
             ((101, 2, _lib._ptr(a), 0, _lib._ptr(a), 5000, _lib._ptr(out)), EINVAL),  # empty operand
             ((100, 2, _lib._ptr(a), 5000, _lib._ptr(a), 5000, _lib._ptr(out)), EINVAL),  # composite modulus
             ((2, 1, _lib._ptr(a), 5000, _lib._ptr(a), 5000, _lib._ptr(out)), EUNSUPPORTED)]
    for args, code in cases:
        with pytest.raises(RonkError) as e:
            c.call("ronk_poly_mul_u64", *args)
        assert e.value.code == code, args
    with pytest.raises(RonkError) as e:
        c.call("ronk_poly_mul_u64_host", 101, 2, None, 5, None, 5, None)
    assert e.value.code == EINVAL


def test_behind_the_gate():
    """One product on a gated non-blocking stream (test_gpu_streams.py's gate), with the path forced on the gated
    context and taken by the measured crossover on the reference context."""
    import torch
    from test_gpu_streams import _res, _through_gate
    p, g, da, db = 101, 2, 1 << 14, (1 << 14) + 9
    ins = [_res(da, 80, p), _res(db, 81, p)]

    def call(c, b, o):
        c.call("ronk_poly_mul_u64", p, g, b[0].data_ptr(), da, b[1].data_ptr(), db, o[0].data_ptr())

    got, _ = _through_gate(ins, [(da + db - 1, torch.int64)], call, env={"RONK_CRT_MUL_MIN": "1"})
    from ronkathon_b200 import ops
    assert np.array_equal(ops.to_host(got[2]), oracle.poly_mul(p, ops.to_host(ins[0]), ops.to_host(ins[1])))


def test_scratch_grows():
    """A fresh context: a small product, one that grows the scratch 2^12-fold, and the small one again."""
    c = _context({"RONK_CRT_MUL_MIN": "1"})
    try:
        from ronkathon_b200 import ops
        p, g = (1 << 64) - 59, 2
        a, b = oracle.splitmix(p, 90, 300), oracle.splitmix(p, 91, 200)
        small = oracle.poly_mul(p, a, b)
        for step in range(3):
            if step == 1:
                check_trapezoid(c, p, g, 1 << 20, (1 << 20) + 1)
            else:
                assert np.array_equal(host(ops.poly_mul(c, dev(a), dev(b), p, g)), small)
    finally:
        c.close()
