"""GPU parity: Polynomial arithmetic through the C ABI vs reference KATs / oracle
(src/polynomial/arithmetic.rs tests, src/polynomial/tests.rs)."""
import numpy as np
import pytest

import oracle
from gpu_util import BABYBEAR, GL, MONT_PRIMES, PBIG, ctx, dev, host

pytestmark = pytest.mark.gpu


def test_reference_kats(kats):
    from ronkathon_b200 import Lagrange, PlutoBaseField, Polynomial
    ctx()
    k = kats["polynomial"]
    F = PlutoBaseField
    P = lambda c: Polynomial(c, F)
    a, b = P(k["a"]), P(k["b"])
    a5 = Polynomial.from_array(k["a"], F, 5)
    assert (b + a) == P(k["b_plus_a"])
    assert (a5 - b) == P(k["a5_minus_b"])
    assert (b - a5) == P(k["b_minus_a5"])
    assert (-a) == P(k["neg_a"])
    assert (a * b) == P(k["a_times_b"])
    assert (P(k["c"]) * P(k["d"])) == P(k["c_times_d"])
    assert (a / b) == P(k["a_div_b"]) and (a % b) == P(k["a_rem_b"])
    assert (b / a) == P(k["b_div_a"]) and (b % a) == P(k["b_rem_a"])
    assert (P([1, 2, 1]) / P([1, 1])) == P(k["p121_div_11"])
    assert (P([1, 2, 1]) % P([1, 1])) == P(k["p121_rem_11"])
    assert a.evaluate(F(2)) == F(k["eval_a_at_2"])
    e = k["eval_103_at_0"]
    assert P(e["coeffs"]).evaluate(F(e["x"])) == F(e["y"])
    assert a.dft().evaluate(F(2)) == F(k["lagrange_eval_dft_a_at_2"])   # polynomial/tests.rs:35-44
    assert a.degree() == k["degree_a"] and a.leading_coefficient() == F(k["leading_a"])
    assert a.pow_mult(2, F(5)) == P(k["pow_mult_a_2_5"])
    assert a.dft().basis is Lagrange
    c1 = kats["config1_extra"]   # BASELINE config 1: degree-8 × degree-8 over F101
    assert (P(c1["a"]) * P(c1["b"])) == P(c1["out"])


def test_lagrange_evaluate_matches_oracle_including_node_quirk():
    from ronkathon_b200 import Lagrange, PlutoBaseField, Polynomial
    ctx()
    rng = np.random.default_rng(3)
    for n in (2, 4, 5, 10, 20):
        c = [int(v) for v in rng.integers(0, 101, n)]
        poly = Polynomial(c, PlutoBaseField, Lagrange)
        for x in [0, 1, 2, 10, 57, 100]:
            assert poly.evaluate(PlutoBaseField(x)).value == oracle.lagrange_eval(101, c, x), (n, x)


def test_divrem_random_and_panics():
    from ronkathon_b200 import PlutoBaseField, PlutoScalarField, Polynomial, PrimeField, RonkPanic
    ctx()
    rng = np.random.default_rng(4)
    for F, p in ((PlutoBaseField, 101), (PlutoScalarField, 17)):
        for da, db in ((9, 3), (6, 6), (12, 2), (4, 7), (40, 5)):
            a = [int(v) for v in rng.integers(0, p, da)]
            b = [int(v) for v in rng.integers(0, p, db)]
            b[-1] = b[-1] or 1  # non-zero top coefficient (trailing zeros panic in the reference)
            q, r = Polynomial(a, F).quotient_and_remainder(Polynomial(b, F))
            eq, er = oracle.poly_divrem(p, a, b)
            assert list(q.coefficients) == list(eq) and list(r.coefficients) == list(er)
    for p in (PBIG, BABYBEAR):                                  # Montgomery moduli above 2^63 and below 2^31
        F = PrimeField(p)
        for da, db in ((9, 3), (6, 6), (12, 2), (4, 7), (40, 5)):
            a, b = oracle.splitmix(p, 30 + da, da), oracle.splitmix(p, 40 + db, db)
            b[-1] = b[-1] or 1
            a[0], b[0] = p - 1, p - 2
            q, r = Polynomial(a, F).quotient_and_remainder(Polynomial(b, F))
            eq, er = oracle.poly_divrem(p, a, b)
            assert np.array_equal(q.coefficients, eq) and np.array_equal(r.coefficients, er), (p, da, db)
    with pytest.raises(RonkPanic):
        Polynomial([1, 2, 3], PlutoBaseField) / Polynomial([0, 0], PlutoBaseField)
    with pytest.raises(oracle.OraclePanic):
        oracle.poly_divrem(101, [1, 2, 3], [0, 0])
    # big field, long dividend
    a, b = oracle.splitmix(GL, 1, 500), oracle.splitmix(GL, 2, 37)
    from ronkathon_b200 import GoldilocksField
    q, r = Polynomial(a, GoldilocksField).quotient_and_remainder(Polynomial(b, GoldilocksField))
    eq, er = oracle.poly_divrem(GL, a, b)
    assert np.array_equal(q.coefficients, eq) and np.array_equal(r.coefficients, er)


def test_div_by_linear_factor_scan_vs_oracle_and_identity():
    """§8f row 1: Polynomial::div/rem by the divisor kzg::open builds (kzg/setup.rs:72-75) runs as a
    device-wide scan.  Bit-exact vs the literal long division of the oracle (mod.rs:170-225) at sizes
    it finishes, and a = q·(b0 + b1·x) + r coefficient by coefficient at 2^22."""
    from ronkathon_b200 import GoldilocksField, PlutoBaseField, PlutoScalarField, Polynomial, PrimeField
    c = ctx()
    rng = np.random.default_rng(11)
    for F, p in ((PlutoBaseField, 101), (PlutoScalarField, 17), (GoldilocksField, GL), (PrimeField(PBIG), PBIG),
                 (PrimeField(BABYBEAR), BABYBEAR)):
        for d in (1, 2, 3, 15, 16, 17, 255, 4095, 4096, 4097, 8193, 9001):
            a = oracle.splitmix(p, 100 + d, d)
            for b in ([int(rng.integers(0, p, dtype=np.uint64)), 1],
                      [int(rng.integers(0, p, dtype=np.uint64)), int(rng.integers(1, p, dtype=np.uint64))], [0, 1]):
                q, r = Polynomial(a, F).quotient_and_remainder(Polynomial(b, F))
                eq, er = oracle.poly_divrem(p, a, b)
                assert np.array_equal(q.coefficients, eq) and np.array_equal(r.coefficients, er), (p, d, b)
    # all-zero dividend, and a dividend the divisor divides exactly (remainder 0)
    z = Polynomial([0] * 5000, GoldilocksField).quotient_and_remainder(Polynomial([5, 7], GoldilocksField))
    assert not z[0].coefficients.any() and not z[1].coefficients.any()
    base = oracle.splitmix(GL, 9, 4999)
    exact = oracle.poly_mul(GL, base, [GL - 3, 1])                      # base·(x - 3), 5000 terms
    q, r = Polynomial(exact, GoldilocksField).quotient_and_remainder(Polynomial([GL - 3, 1], GoldilocksField))
    assert np.array_equal(q.coefficients[:-1], base) and q.coefficients[-1] == 0 and not r.coefficients.any()
    # device-pointer entry at 2^22 (1024 chunks): identity check, remainder = a(z) by the evaluate kernel
    d = 1 << 22
    for p in (GL, PBIG, BABYBEAR):
        a = oracle.splitmix(p, 77, d)
        b0, b1 = 1234567890123456789 % p, 987654321987654321 % p
        A, Q, R = dev(a), dev(np.zeros(d, np.uint64)), dev(np.zeros(1, np.uint64))
        c.call("ronk_poly_div_linear_u64", p, A.data_ptr(), d, b0, b1, Q.data_ptr(), R.data_ptr())
        q, r = host(Q), host(R)
        assert q[-1] == 0
        recomposed = oracle.poly_add(p, oracle.vec_mul(p, q, np.full(d, b0, np.uint64)),
                                     np.concatenate([np.zeros(1, np.uint64), oracle.vec_mul(p, q, np.full(d, b1, np.uint64))[:-1]]))
        recomposed[0] = oracle.add(p, int(recomposed[0]), int(r[0]))
        assert np.array_equal(recomposed, a), p
        zpt = oracle.mul(p, p - b0, oracle.inverse(p, b1))
        assert int(r[0]) == oracle.poly_eval_horner(p, a, zpt), p
    with pytest.raises(Exception):
        c.call("ronk_poly_div_linear_u64", GL, A.data_ptr(), d, b0, 0, Q.data_ptr(), R.data_ptr())
    with pytest.raises(Exception):
        c.call("ronk_poly_div_linear_u64", GL, A.data_ptr(), d, b0, b1, A.data_ptr(), R.data_ptr())


def test_reed_solomon_decode_interpolation(kats):
    """§8f row 2: Message::decode (codes/reed_solomon.rs:55-107) = interpolation through the first K
    coordinates.  Reference decode tests, the literal oracle at small K, the inverse transform on a full
    set of roots of unity, and evaluate∘interpolate = id at K = 4097."""
    from ronkathon_b200 import GoldilocksField, PlutoBaseField, Polynomial, PrimeField, RonkPanic, codes
    ctx()
    r = kats["reed_solomon_decode"]
    F127 = PrimeField(127)
    for msg in r["messages"]:                                            # reed_solomon.rs:177-219
        cw = codes.rs_encode(msg, r["n"], F127)
        assert [v.value for v in codes.rs_decode(cw, len(msg), F127)] == msg
    rng = np.random.default_rng(21)
    for F, p in ((F127, 127), (PlutoBaseField, 101), (GoldilocksField, GL)):
        for k in (1, 2, 3, 6, 10):
            xs = [int(v) for v in (rng.choice(p, size=k, replace=False) if p < 1000 else oracle.splitmix(p, 50 + k, k))]
            ys = [int(v) for v in oracle.splitmix(p, 60 + k, k)]
            got = codes.rs_decode(list(zip(xs, ys)), k, F)
            assert [v.value for v in got] == [int(v) for v in oracle.rs_decode(p, xs, ys, k)], (p, k)
    from ronkathon_b200 import _lib
    for p in (PBIG, BABYBEAR):                                           # Montgomery moduli, the C entry point directly
        for k in (1, 2, 3, 6, 10):
            xs, ys = oracle.splitmix(p, 50 + k, k), oracle.splitmix(p, 60 + k, k)
            ys[0] = p - 1
            out = np.empty(k, dtype=np.uint64)
            ctx().call("ronk_poly_interpolate_u64_host", p, _lib._ptr(xs), _lib._ptr(ys), k, _lib._ptr(out))
            assert np.array_equal(out, oracle.rs_decode(p, xs, ys, k)), (p, k)
    for n in (256, 2048):                                              # full root-of-unity set: ifft
        msg = oracle.splitmix(GL, n, n)
        w = oracle.root_of_unity(GL, n)
        xs = np.array([pow(w, i, GL) for i in range(n)], dtype=np.uint64)
        ys = oracle.ntt_fast(GL, msg)
        got = codes.rs_decode(list(zip(xs.tolist(), ys.tolist())), n, GoldilocksField)
        assert np.array_equal(np.array([v.value for v in got], dtype=np.uint64), msg), n
    k = 4097                                                             # multi-block, odd K
    xs, ys = oracle.splitmix(GL, 71, k), oracle.splitmix(GL, 72, k)
    assert len(set(xs.tolist())) == k
    coeffs = [v.value for v in codes.rs_decode(list(zip(xs.tolist(), ys.tolist())), k, GoldilocksField)]
    for i in (0, 1, 31, 32, 255, 256, 2048, 4095, 4096):
        assert oracle.poly_eval_horner(GL, coeffs, int(xs[i])) == int(ys[i]), i
    back = Polynomial(coeffs, GoldilocksField).evaluate_many(xs.tolist())
    assert [v.value for v in back] == ys.tolist()
    with pytest.raises(RonkPanic):
        codes.rs_decode([(1, 3), (1, 4), (2, 5)], 3, F127)               # repeated x: the reference divides by zero


def test_kzg_open_at_scale_matches_fast_oracle():
    """commit→open on the device at a size the reference's const-generic arrays cannot reach:
    2^16 F17 coefficients, quotient by the scan kernel, commitment by the bucket MSM."""
    from ronkathon_b200 import kzg
    from ronkathon_b200.curve import AffinePoint
    from gpu_util import msm_inputs
    ctx()
    n = 1 << 16
    pts, _ = msm_inputs(n)
    coeffs = oracle.splitmix(17, 5, n)
    zz = 4
    out = kzg.open_([int(v) for v in coeffs], zz, pts)
    q, _ = _synthetic(17, coeffs, zz)
    assert out.raw == oracle.commit(q, pts, fast=True)


def _synthetic(p, a, z):
    """h_j = a_j + z·h_{j+1}; q_{j-1} = h_j, remainder h_0 (python ints)."""
    hh, out = 0, [0] * len(a)
    for j in range(len(a) - 1, 0, -1):
        hh = (int(a[j]) + z * hh) % p
        out[j - 1] = hh
    return out, (int(a[0]) + z * hh) % p


def test_poly_mul_paths_vs_oracle(gold64):
    from ronkathon_b200 import ops
    c = ctx()
    a3, b3 = oracle.splitmix(GL, 42, 300), oracle.splitmix(GL, 43, 300)
    got = host(ops.poly_mul(c, dev(a3), dev(b3)))
    assert list(got) == gold64["poly_mul_300x300_seed42_seed43"]
    for da, db in ((1, 1), (1, 7), (2, 2), (33, 1), (64, 64), (1000, 3), (2000, 3000), (5000, 5000), (40000, 25000)):
        a, b = oracle.splitmix(GL, da, da), oracle.splitmix(GL, db + 1, db)
        got = host(ops.poly_mul(c, dev(a), dev(b)))
        if da * db <= 4_000_000:
            exp = oracle.poly_mul(GL, a, b)
        else:  # convolution theorem with the oracle's transforms
            L = da + db - 1
            lg = (L - 1).bit_length()
            pa, pb = np.zeros(1 << lg, np.uint64), np.zeros(1 << lg, np.uint64)
            pa[:da], pb[:db] = a, b
            exp = oracle.ntt_fast(GL, oracle.vec_mul(GL, oracle.ntt_fast(GL, pa), oracle.ntt_fast(GL, pb)), inverse=True)[:L]
        assert np.array_equal(got, exp), (da, db)
    # p = 101 cannot use a power-of-two NTT beyond n = 4: schoolbook kernel
    rng = np.random.default_rng(9)
    a, b = rng.integers(0, 101, 57).astype(np.uint64), rng.integers(0, 101, 91).astype(np.uint64)
    assert np.array_equal(host(ops.poly_mul(c, dev(a), dev(b), p=101, g=2)), oracle.poly_mul(101, a, b))


def test_config3_poly_mul_2_24():
    """BASELINE config 3: two 2^23-coefficient polynomials (NTT + fused pointwise + iNTT, n = 2^24).
    Checked bit-exactly against the oracle's convolution-theorem route, and through the
    size-independent property c(x) == a(x)·b(x) at random points evaluated on the GPU."""
    from ronkathon_b200 import ops
    c = ctx()
    d = 1 << 23
    a, b = oracle.splitmix(GL, 42, d), oracle.splitmix(GL, 43, d)
    A, B = dev(a), dev(b)
    C = ops.poly_mul(c, A, B)
    got = host(C)
    assert len(got) == 2 * d - 1
    n = 1 << 24
    pa, pb = np.zeros(n, np.uint64), np.zeros(n, np.uint64)
    pa[:d], pb[:d] = a, b
    exp = oracle.ntt_fast(GL, oracle.vec_mul(GL, oracle.ntt_fast(GL, pa), oracle.ntt_fast(GL, pb)), inverse=True)
    assert exp[-1] == 0 and np.array_equal(got, exp[:-1])
    xs = dev(oracle.splitmix(GL, 99, 4))
    ea, eb, ec = host(ops.poly_eval(c, A, xs)), host(ops.poly_eval(c, B, xs)), host(ops.poly_eval(c, C, xs))
    assert np.array_equal(ec, oracle.vec_mul(GL, ea, eb))


@pytest.mark.parametrize("la,lb", [((1 << 20) + 7, (1 << 19) + 1), ((1 << 21) - 5, 1 << 21), ((1 << 22) - 1, (1 << 22) - 3)])
def test_poly_mul_mid_sizes_identity_and_agreement(la, lb):
    """Products whose transforms have 2^21, 2^22 and 2^23 points: zero padding and clipping happen inside the bounded first /
    last tile passes.  c(x) = a(x)·b(x) at a point (oracle Horner), end coefficients, length — and bit-for-bit
    agreement with a context that keeps the two-pass kernel for these sizes (RONK_NTT3_MID=0)."""
    import os
    import torch
    from ronkathon_b200 import Context, ops
    c = ctx()
    a = ops.splitmix_fill(c, la, 142, GL)
    b = ops.splitmix_fill(c, lb, 143, GL)
    prod = ops.poly_mul(c, a, b)
    ah, bh, ph = host(a), host(b), host(prod)
    assert len(ph) == la + lb - 1
    assert int(ph[0]) == oracle.mul(GL, int(ah[0]), int(bh[0]))
    assert int(ph[-1]) == oracle.mul(GL, int(ah[-1]), int(bh[-1]))
    x = 0x0FEDCBA987654321 % GL
    assert oracle.poly_eval_horner(GL, ph, x) == oracle.mul(GL, oracle.poly_eval_horner(GL, ah, x), oracle.poly_eval_horner(GL, bh, x))
    os.environ["RONK_NTT3_MID"] = "0"
    try:
        c1 = Context(0, torch.cuda.current_stream().cuda_stream)
    finally:
        os.environ.pop("RONK_NTT3_MID")
    p1 = ops.poly_mul(c1, a, b)
    c1.sync()
    assert np.array_equal(host(p1), ph)
    c1.close()


def test_evaluate_vs_oracle(gold64):
    from ronkathon_b200 import GoldilocksField, Polynomial, ops
    c = ctx()
    a3 = oracle.splitmix(GL, 42, 300)
    e = gold64["eval_300_seed42_at_seed43_0"]
    assert Polynomial(a3, GoldilocksField).evaluate(e["x"]).value == e["y"]
    for p in (GL, PBIG, BABYBEAR):
        for d in (0, 1, 2, 255, 256, 257, 1000, 70000):
            co = oracle.splitmix(p, d + 5, d)
            if d:
                co[-1] = p - 1
            xs = np.concatenate([oracle.splitmix(p, 8, 5), np.array([0, 1, p - 1], dtype=np.uint64)])
            got = host(ops.poly_eval(c, dev(co) if d else dev(np.zeros(1, np.uint64))[:0], dev(xs), p))
            exp = [oracle.poly_eval_horner(p, co, int(x)) if d else 0 for x in xs]
            assert list(got) == exp, (p, d)
            if 0 < d <= 300:  # the reference's literal O(D²) form gives the same values
                assert exp == [oracle.poly_eval(p, co, int(x)) for x in xs]


def test_reed_solomon_encode_and_shamir_next_rows(kats):
    """§8f: RS encode (codes/reed_solomon.rs:136-154, P = 127) and Shamir-style multi-point evaluate."""
    from ronkathon_b200 import PrimeField, codes
    ctx()
    r = kats["reed_solomon"]
    F = PrimeField(r["p"])
    cw = codes.rs_encode(r["msg"], r["n"], F)
    assert [x.value for x, _ in cw] == r["x"] and [y.value for _, y in cw] == r["y"]
    xs, ys = oracle.rs_encode(127, [1, 2, 3], 7)                      # encode_larger_size: N = 7
    cw7 = codes.rs_encode([1, 2, 3], 7, F)
    assert [x.value for x, _ in cw7] == list(xs) and [y.value for _, y in cw7] == list(ys)
    from ronkathon_b200 import GoldilocksField
    msg = [int(v) for v in oracle.splitmix(GL, 3, 100)]
    xs, ys = oracle.rs_encode(GL, msg, 256)
    cw = codes.rs_encode(msg, 256, GoldilocksField)                    # power of two → NTT path
    assert [x.value for x, _ in cw] == list(xs) and [y.value for _, y in cw] == list(ys)
    shares = codes.shamir_shares([11, 5, 7, 3], 9, PrimeField(101))
    assert [(x, y.value) for x, y in shares] == [(x, oracle.poly_eval(101, [11, 5, 7, 3], x)) for x in range(1, 10)]


def _conv_oracle(p, g, a, b):
    """The product by the convolution theorem with the oracle's transforms."""
    L = len(a) + len(b) - 1
    n = 1 << (L - 1).bit_length()
    pa, pb = np.zeros(n, np.uint64), np.zeros(n, np.uint64)
    pa[:len(a)], pb[:len(b)] = a, b
    return oracle.ntt_fast(p, oracle.vec_mul(p, oracle.ntt_fast(p, pa, g=g), oracle.ntt_fast(p, pb, g=g)), inverse=True, g=g)[:L]


def _poly_mul_generic_cases():
    cases = [(name, 64, 64) for name in MONT_PRIMES] + [(name, 200, 200) for name in MONT_PRIMES]   # schoolbook | NTT
    for name in ("babybear", "pbig"):                       # transforms of 2^13 … 2^20 points: single tile, two-pass
        cases += [(name, (1 << (k - 2)) + 5, (1 << (k - 1)) - 17) for k in range(13, 21)]
    cases += [("koalabear", 5000, 9000), ("p32", 40000, 25000), ("p57", 30001, 2), ("gl_g5", 70000, 60000)]
    return cases


@pytest.mark.parametrize("name,da,db", _poly_mul_generic_cases())
def test_poly_mul_generic_primes_vs_oracle(name, da, db):
    """poly_mul with every (p, g) of the Montgomery table: both sides of the schoolbook / NTT crossover against the
    oracle's schoolbook product, and products whose transforms have 2^13 … 2^20 points (the bounded single-tile and
    bounded two-pass Montgomery kernels, fused multiply included) against the oracle's convolution-theorem route."""
    from ronkathon_b200 import ops
    c = ctx()
    p, g, _ = MONT_PRIMES[name]
    a, b = oracle.splitmix(p, 300 + da, da), oracle.splitmix(p, 400 + db, db)
    a[0], b[-1] = p - 1, p - 2
    got = host(ops.poly_mul(c, dev(a), dev(b), p, g))
    exp = oracle.poly_mul(p, a, b) if da * db <= 100_000 else _conv_oracle(p, g, a, b)
    assert np.array_equal(got, exp), (name, da, db)


@pytest.mark.parametrize("name,da,db", [("babybear", (1 << 22) + 3, (1 << 22) - 9), ("pbig", 1 << 23, 1 << 23),
                                        ("p32", (1 << 15) + 1, (1 << 15) + 1)])
def test_poly_mul_generic_primes_large_and_beyond_the_two_adicity(name, da, db):
    """Products of 2^23 and 2^24 points on the Montgomery two-pass kernels, and one too long for the prime's 2-adicity
    (2^15 + 1 squared needs 2^17 points, 4295294977 has 2^16), which falls back to schoolbook: the length, the end
    coefficients and c(x) = a(x)·b(x) at random points by the oracle's Horner evaluation."""
    from ronkathon_b200 import ops
    c = ctx()
    p, g, _ = MONT_PRIMES[name]
    A, B = ops.splitmix_fill(c, da, 500, p), ops.splitmix_fill(c, db, 501, p)
    got, a, b = host(ops.poly_mul(c, A, B, p, g)), host(A), host(B)
    assert len(got) == da + db - 1
    assert int(got[0]) == oracle.mul(p, int(a[0]), int(b[0])) and int(got[-1]) == oracle.mul(p, int(a[-1]), int(b[-1]))
    for x in oracle.splitmix(p, 502, 4):
        x = int(x)
        assert oracle.poly_eval_horner(p, got, x) == oracle.mul(p, oracle.poly_eval_horner(p, a, x),
                                                                oracle.poly_eval_horner(p, b, x)), (name, x)
