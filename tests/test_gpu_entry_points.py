"""GPU parity for the C ABI entry points outside the transforms, with every test prime, past one thread block or one
grid stride, and at each entry point's panic edges: the fused cross-rank stage, the strided cross-rank butterflies and
the twiddle column, field element-wise ops, the any-size DFT, Lagrange evaluation, interpolation, general polynomial
division, polynomial add/sub, and point add/neg/smul over the whole group E(F_101²).  Every comparison is bit-exact
against the CPU oracle or against an identity evaluated with Python integers or the oracle's field ops."""
import ctypes as C
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import oracle
from gpu_util import BABYBEAR, GL, MONT_PRIMES, PBIG, ctx, dev, host, lagrange_closed_form

pytestmark = pytest.mark.gpu

P64 = (1 << 64) - 59                       # the largest 64-bit prime; used where no root of unity is needed
GL_G5 = MONT_PRIMES["gl_g5"][1]
KOALABEAR = MONT_PRIMES["koalabear"][0]
# every (p, g) the kernels dispatch on: Goldilocks with g = 7 (its own policy) and the Montgomery table
ROOTED = [("gl", GL, 7)] + [(name, p, g) for name, (p, g, _) in MONT_PRIMES.items()]
# every distinct modulus, for the calls that take no root of unity
MODULI = sorted({p for _, p, _ in ROOTED} | {P64})
# the primes of the cross-rank stage and the strided butterflies: both policies, a prime below 2^31 and one above 2^63
CROSS_RANK = [("gl", GL, 7), ("babybear", BABYBEAR, 31), ("pbig", PBIG, 3), ("gl_g5", GL, GL_G5)]


def _edge(p):
    v = [0, 1, 2, 3, p - 1, p - 2, p // 2, p // 2 + 1]
    if p > (1 << 33):
        v += [(1 << 32) - 1, 1 << 32, (1 << 32) + 1, p - (1 << 32), p - (1 << 32) + 1, 1 << 63, 0xFFFFFFFF00000000,
              0xFFFFFFFE00000002]
    return sorted({x % p for x in v})


def _rand(p, seed, n, nonzero=False):
    r = oracle.splitmix(p, seed, n)
    if nonzero:
        r[r == 0] = 1
    return r


def _empty(n):
    import torch
    return torch.empty(n, dtype=torch.int64, device="cuda")


def _code(excinfo):
    return excinfo.value.code


def _pmap(fn, items):
    """The oracle's ctypes calls release the GIL: spread long runs of them over the host's cores."""
    with ThreadPoolExecutor(8) as ex:
        return list(ex.map(fn, items))


def _horner_all(p, coeffs, xs):
    coeffs = np.ascontiguousarray(coeffs, dtype=np.uint64)
    return np.array(_pmap(lambda x: oracle.poly_eval_horner(p, coeffs, int(x)), list(xs)), dtype=np.uint64)


# ---- 1. the distributed-transform building blocks on one device -------------------------------------------------------
@pytest.mark.parametrize("name,p,g", CROSS_RANK)
@pytest.mark.parametrize("log_g", [1, 2, 3, 4])
def test_cross_rank_fused_stage_reassembles_the_transform(name, p, g, log_g):
    """ronk_ntt_cross_rank_fused_u64, one call per rank with every peer buffer on this device: the G outputs, put back
    with the header's layout out_s[q·blk + k] = X[s·blk + k + m·q], are the whole n-point transform."""
    from ronkathon_b200 import RonkError, RonkPanic, _lib
    c = ctx()
    G = 1 << log_g
    for log_n in (2 * log_g, 12, 18):
        n = 1 << log_n
        m = n // G
        blk = m // G
        a = _rand(p, 1000 + 10 * log_n + log_g, n)
        a[0], a[-1] = p - 1, p - 1
        ys = [dev(a[r::G]) for r in range(G)]
        for y in ys:                                                     # Y_r = the n/G-point transform of a[r::G]
            c.call("ronk_ntt_u64", p, g, y.data_ptr(), log_n - log_g, 1, 0)
        peers = (C.c_void_p * G)(*[y.data_ptr() for y in ys])
        got = np.zeros((G, m), np.uint64)
        out = _empty(m)
        for s in range(G):
            c.call("ronk_ntt_cross_rank_fused_u64", p, g, C.cast(peers, _lib.vp), log_g, s, log_n, out.data_ptr())
            got[:, s * blk:(s + 1) * blk] = host(out).reshape(G, blk)
        assert np.array_equal(got.reshape(-1), oracle.ntt_fast(p, a, g=g)), (name, log_g, log_n)
    # documented error returns; none of them launches the butterfly kernel
    log_n = 2 * log_g + 2
    with pytest.raises(RonkPanic):                                      # rank >= G
        c.call("ronk_ntt_cross_rank_fused_u64", p, g, C.cast(peers, _lib.vp), log_g, G, log_n, out.data_ptr())
    holes = (C.c_void_p * G)(*[y.data_ptr() for y in ys])
    holes[G - 1] = None
    with pytest.raises(RonkPanic):                                      # a null peer
        c.call("ronk_ntt_cross_rank_fused_u64", p, g, C.cast(holes, _lib.vp), log_g, 0, log_n, out.data_ptr())
    with pytest.raises(RonkPanic):                                      # n/G² < 1
        c.call("ronk_ntt_cross_rank_fused_u64", p, g, C.cast(peers, _lib.vp), log_g, 0, 2 * log_g - 1, out.data_ptr())
    for bad_log_g in (0, 5):                                            # G = 1 and G = 32 are outside 2 … 16
        with pytest.raises(RonkError) as e:
            c.call("ronk_ntt_cross_rank_fused_u64", p, g, C.cast(peers, _lib.vp), bad_log_g, 0, 12, out.data_ptr())
        assert _code(e) == _lib.EUNSUPPORTED


def _strided_dft(p, x, w, scale):
    """Σ_j x[j]·w^(jq)·scale for every column of the G×count matrix x, with the oracle's element-wise ops."""
    G = len(x)
    out = []
    for q in range(G):
        acc = np.zeros(x.shape[1], np.uint64)
        for j in range(G):
            acc = oracle.poly_add(p, acc, oracle.vec_mul(p, x[j], np.full(x.shape[1], pow(w, j * q, p), np.uint64)))
        out.append(oracle.vec_mul(p, acc, np.full(x.shape[1], scale, np.uint64)))
    return np.stack(out)


@pytest.mark.parametrize("name,p,g", CROSS_RANK)
def test_strided_small_transform_past_one_grid(name, p, g):
    """ronk_ntt_strided_small_u64 with count = 1 056 CTAs × 128 threads + 7, so the grid-stride loop runs twice for
    some threads.  Forward against the G-point DFT with the words between the strided sets untouched, then the inverse
    back to the input."""
    c = ctx()
    count = 1056 * 128 + 7
    stride = count + 5
    for log_g in (1, 2, 3, 4):
        G = 1 << log_g
        a = _rand(p, 77 + log_g, G * stride)
        a[:count] = p - 1                                                # x_0 = p - 1 in every set
        d = dev(a)
        w = pow(g, (p - 1) >> log_g, p)
        x = a.reshape(G, stride)[:, :count]
        fwd = a.reshape(G, stride).copy()
        fwd[:, :count] = _strided_dft(p, x, w, 1)
        c.call("ronk_ntt_strided_small_u64", p, g, d.data_ptr(), log_g, stride, count, 0)
        assert np.array_equal(host(d), fwd.reshape(-1)), (name, log_g)
        c.call("ronk_ntt_strided_small_u64", p, g, d.data_ptr(), log_g, stride, count, 1)
        assert np.array_equal(host(d), a), (name, log_g)                 # ω^-1 and G^-1 undo the exact forward result


@pytest.mark.parametrize("p", MODULI, ids=hex)
def test_field_powers_every_prime(p):
    """ronk_field_powers_u64: out[i] = scale·base^i at n = 1, 2 and 8·270 336 + 5, where every thread of the full grid
    takes more than 8 steps.  The recurrence out[i+1] = out[i]·base over the whole vector, out[0] = scale, and sampled
    scale·base^i by the oracle's pow."""
    c = ctx()
    base, scale = int(_rand(p, 5, 1, True)[0]), int(_rand(p, 6, 1, True)[0])
    for b, s in ((base, scale), (p - 1, p - 1)):
        for n in (1, 2, 8 * 132 * 8 * 256 + 5):
            out = _empty(n)
            c.call("ronk_field_powers_u64", p, b, s, out.data_ptr(), n)
            o = host(out)
            assert int(o[0]) == s
            assert np.array_equal(o[1:], oracle.vec_mul(p, o[:-1], np.full(n - 1, b, np.uint64))), (hex(p), n)
            for i in sorted({0, n - 1, n // 2} | set(int(v) for v in _rand(n, 7, 32))):
                assert int(o[i]) == oracle.mul(p, s, oracle.pow_(p, b, i)), (hex(p), n, i)


# ---- 2. field element-wise ops --------------------------------------------------------------------------------------
@pytest.mark.parametrize("p", MODULI, ids=hex)
def test_field_div_inv_pow_edges_and_aliasing(p):
    """div / inv against the oracle on the edge × edge matrix and 20 000 random pairs; pow with the exponents where
    square-and-multiply goes wrong on every edge value (0^0 = 1); in-place add/sub/mul/neg; and the host variants
    against the device ones."""
    from ronkathon_b200 import _lib
    c = ctx()
    ev = _edge(p)
    rnd_a, rnd_b = _rand(p, 11, 20000), _rand(p, 12, 20000)
    a = np.concatenate([np.repeat(np.array(ev, np.uint64), len(ev)), rnd_a])
    b = np.concatenate([np.tile(np.array(ev, np.uint64), len(ev)), rnd_b])
    nz = b != 0
    an, bn = np.ascontiguousarray(a[nz]), np.ascontiguousarray(b[nz])
    out, d_an, d_bn = _empty(len(an)), dev(an), dev(bn)                 # named: a freed temporary's block is reused
    c.call("ronk_field_div_u64", p, d_an.data_ptr(), d_bn.data_ptr(), out.data_ptr(), len(an))
    assert np.array_equal(host(out), np.array([oracle.div(p, int(x), int(y)) for x, y in zip(an, bn)], np.uint64))
    c.call("ronk_field_inv_u64", p, d_bn.data_ptr(), out.data_ptr(), len(bn))
    assert np.array_equal(host(out), np.array([oracle.inverse(p, int(y)) for y in bn], np.uint64))
    evd = dev(np.array(ev, np.uint64))
    po = _empty(len(ev))
    for e in (0, 1, 2, p - 2, p - 1, p, p + 1, 1 << 63, (1 << 64) - 1):
        c.call("ronk_field_pow_u64", p, evd.data_ptr(), e, po.data_ptr(), len(ev))
        exp = [pow(x, e, p) for x in ev]                                  # Python's pow: 0^0 = 1, like pow(0) = ONE
        assert list(host(po)) == exp and exp == [oracle.pow_(p, x, e) for x in ev], (hex(p), e)
    # out = a and out = b, where the header allows the alias
    for fn, name in ((oracle.add, "ronk_field_add_u64"), (oracle.sub, "ronk_field_sub_u64"),
                     (oracle.mul, "ronk_field_mul_u64")):
        exp = np.array([fn(p, int(x), int(y)) for x, y in zip(a, b)], np.uint64)
        da, db = dev(a), dev(b)
        c.call(name, p, da.data_ptr(), db.data_ptr(), da.data_ptr(), len(a))
        assert np.array_equal(host(da), exp) and np.array_equal(host(db), b), name
        da = dev(a)
        c.call(name, p, da.data_ptr(), db.data_ptr(), db.data_ptr(), len(a))
        assert np.array_equal(host(db), exp) and np.array_equal(host(da), a), name
    da = dev(a)
    c.call("ronk_field_neg_u64", p, da.data_ptr(), da.data_ptr(), len(a))
    assert np.array_equal(host(da), np.array([oracle.neg(p, int(x)) for x in a], np.uint64))
    # host-pointer variants on 1 000 elements give what the device variants give
    h_a, h_b = np.ascontiguousarray(an[-1000:]), np.ascontiguousarray(bn[-1000:])
    h_out = np.empty(1000, np.uint64)
    dev_out, d_ha, d_hb = _empty(1000), dev(h_a), dev(h_b)
    for op, name in enumerate(("ronk_field_add_u64", "ronk_field_sub_u64", "ronk_field_mul_u64", "ronk_field_div_u64")):
        c.call("ronk_field_binop_u64_host", op, p, _lib._ptr(h_a), _lib._ptr(h_b), _lib._ptr(h_out), 1000)
        c.call(name, p, d_ha.data_ptr(), d_hb.data_ptr(), dev_out.data_ptr(), 1000)
        assert np.array_equal(h_out, host(dev_out)), name
    for op, name in enumerate(("ronk_field_neg_u64", "ronk_field_inv_u64")):
        c.call("ronk_field_unop_u64_host", op, p, _lib._ptr(h_b), _lib._ptr(h_out), 1000)
        c.call(name, p, d_hb.data_ptr(), dev_out.data_ptr(), 1000)
        assert np.array_equal(h_out, host(dev_out)), name
    c.call("ronk_field_pow_u64_host", p, _lib._ptr(h_a), p - 3, _lib._ptr(h_out), 1000)
    c.call("ronk_field_pow_u64", p, d_ha.data_ptr(), p - 3, dev_out.data_ptr(), 1000)
    assert np.array_equal(h_out, host(dev_out))


@pytest.mark.parametrize("p", MODULI, ids=hex)
def test_field_zero_divisor_at_the_end_of_a_long_vector(p):
    """A zero divisor, or a zero under inv, at index n - 1 of a 2^20 + 3 vector raises; the next clean call on the same
    context succeeds, and out·b = a (out·a = 1) holds at every index."""
    from ronkathon_b200 import RonkPanic
    c = ctx()
    n = (1 << 20) + 3
    a, b = _rand(p, 21, n), _rand(p, 22, n, nonzero=True)
    b[-1] = 0
    da, db, out = dev(a), dev(b), _empty(n)
    with pytest.raises(RonkPanic):
        c.call("ronk_field_div_u64", p, da.data_ptr(), db.data_ptr(), out.data_ptr(), n)
    with pytest.raises(RonkPanic):
        c.call("ronk_field_inv_u64", p, db.data_ptr(), out.data_ptr(), n)
    b[-1] = p - 1
    db = dev(b)
    c.call("ronk_field_div_u64", p, da.data_ptr(), db.data_ptr(), out.data_ptr(), n)
    assert np.array_equal(oracle.vec_mul(p, host(out), b), a)
    c.call("ronk_field_inv_u64", p, db.data_ptr(), out.data_ptr(), n)
    assert np.array_equal(oracle.vec_mul(p, host(out), b), np.ones(n, np.uint64))


# ---- 3. any-size DFT ------------------------------------------------------------------------------------------------
# p - 1 = 2^32·3·5·17·257·65537 (GL), 2^27·3·5 (BabyBear), 2^24·127 (KoalaBear), 2^28·11·23831·262147 (PBIG)
DFT_CASES = ([(GL, 7, n) for n in (3, 5, 15, 17, 255, 257, 771, 4096, 65537)]
             + [(BABYBEAR, 31, n) for n in (3, 15, 3 << 12)]
             + [(KOALABEAR, 3, n) for n in (127, 508)]
             + [(PBIG, 3, n) for n in (11, 23831, 11 << 10)]
             + [(GL, 49, 256), (GL, 49, 15)])                            # 49 = 7² is no generator: ω of order 128 at n = 256


@pytest.mark.parametrize("p,g,n", DFT_CASES, ids=lambda v: hex(v) if v > 1 << 20 else str(v))
def test_dft_any_size(p, g, n):
    """ronk_dft_u64 / _host: X[i] = a(ω^i) for n | p - 1.  The oracle's literal dft up to n = 1024; above, Horner at
    i ∈ {0, 1, n - 1} and 64 sampled i; powers of two with a generator also against ronk_ntt_u64."""
    from ronkathon_b200 import _lib
    c = ctx()
    assert (p - 1) % n == 0
    a = _rand(p, 31 + n, n)
    a[0], a[-1] = p - 1, p - 1
    out, d_a = _empty(n), dev(a)
    c.call("ronk_dft_u64", p, g, d_a.data_ptr(), n, out.data_ptr())
    got = host(out)
    h_out = np.empty(n, np.uint64)
    c.call("ronk_dft_u64_host", p, g, _lib._ptr(a), n, _lib._ptr(h_out))
    assert np.array_equal(h_out, got)
    if n <= 1024:
        assert np.array_equal(got, oracle.dft(p, a, g=g)), (hex(p), g, n)
    else:
        w = pow(g, (p - 1) // n, p)
        idx = sorted({0, 1, n - 1} | set(int(v) for v in _rand(n, 32, 64)))
        exp = _horner_all(p, a, [pow(w, i, p) for i in idx])
        assert np.array_equal(got[idx], exp), (hex(p), g, n)
    if n & (n - 1) == 0 and g != 49:                                    # the transform needs ω of order exactly n
        d = dev(a)
        c.call("ronk_ntt_u64", p, g, d.data_ptr(), n.bit_length() - 1, 1, 0)
        assert np.array_equal(host(d), got)


# ---- 4. Lagrange evaluation -----------------------------------------------------------------------------------------
LAGRANGE_PRIMES = [("f101", 101, 2), ("gl", GL, 7), ("babybear", BABYBEAR, 31), ("pbig", PBIG, 3), ("gl_g5", GL, GL_G5)]


@pytest.mark.parametrize("name,p,g", LAGRANGE_PRIMES)
def test_lagrange_eval_past_one_block(name, p, g):
    """ronk_poly_lagrange_eval_u64_host at n up to 2^14, where each of the 256 threads owns up to 64 nodes: x = 0, g,
    p - 1, a random x and the nodes ω, ω^(n-1).  The oracle for n ≤ 256 and the closed form for every n; with g = 7^5
    and 5 | n the nodes repeat and the call raises."""
    from ronkathon_b200 import RonkPanic, _lib
    c = ctx()
    out = C.c_uint64()
    for n in (1, 2, 3, 255, 256, 257, 1024, 3 << 10, 1 << 14):
        if (p - 1) % n:
            continue
        co = _rand(p, 41 + n, n)
        co[-1] = p - 1
        w = pow(g, (p - 1) // n, p)
        distinct = len({pow(w, i, p) for i in range(n)}) == n           # g = 7^5: ω has order n/5 when 5 | n
        for x in (0, g, p - 1, int(_rand(p, 42 + n, 1)[0]), w, pow(w, n - 1, p)):
            if not distinct:                                             # the reference divides by zero
                with pytest.raises(RonkPanic):
                    c.call("ronk_poly_lagrange_eval_u64_host", p, g, _lib._ptr(co), n, x, C.byref(out))
                continue
            c.call("ronk_poly_lagrange_eval_u64_host", p, g, _lib._ptr(co), n, x, C.byref(out))
            exp = lagrange_closed_form(p, g, co, x)
            assert out.value == exp, (name, n, x)
            if n <= 256:
                assert exp == oracle.lagrange_eval(p, co, x, g=g), (name, n, x)


def test_lagrange_eval_panics():
    """A g whose ω has order below n repeats a node, which the reference divides by (GL, g = 49: ω_2 = 1, ω_256 of
    order 128); n ∤ p - 1 and a non-canonical x are refused."""
    from ronkathon_b200 import RonkPanic, _lib
    c = ctx()
    out = C.c_uint64()
    for n in (2, 256):
        co = _rand(GL, n, n)
        with pytest.raises(RonkPanic):
            c.call("ronk_poly_lagrange_eval_u64_host", GL, 49, _lib._ptr(co), n, 12345, C.byref(out))
        with pytest.raises(oracle.OraclePanic):
            oracle.lagrange_eval(GL, co, 12345, g=49)
    co = _rand(GL, 7, 7)
    with pytest.raises(RonkPanic):                                      # 7 ∤ p - 1
        c.call("ronk_poly_lagrange_eval_u64_host", GL, 7, _lib._ptr(co), 7, 5, C.byref(out))
    co = _rand(GL, 8, 8)
    with pytest.raises(RonkPanic):
        c.call("ronk_poly_lagrange_eval_u64_host", GL, 7, _lib._ptr(co), 8, GL, C.byref(out))
    c.call("ronk_poly_lagrange_eval_u64_host", GL, 7, _lib._ptr(co), 8, 5, C.byref(out))   # the context still works
    assert out.value == lagrange_closed_form(GL, 7, co, 5)


# ---- 5. interpolation -----------------------------------------------------------------------------------------------
def _distinct(p, seed, k):
    if p < 1 << 20:
        return np.random.default_rng(seed).choice(p, size=k, replace=False).astype(np.uint64)
    xs = oracle.splitmix(p, seed, k)
    assert len(np.unique(xs)) == k
    return xs


@pytest.mark.parametrize("p", [101] + MODULI, ids=hex)
def test_interpolation_every_size(p):
    """ronk_poly_interpolate_u64_host for k from one node to 8 192 (one to 32 warps, partial warps, the cap): k terms
    whose Horner value at every x_i is y_i, which pins the unique interpolant; the oracle's decode at k ≤ 12."""
    from ronkathon_b200 import _lib
    c = ctx()
    for k in (1, 12, 31, 32, 33, 255, 256, 257, 1025, 8192):
        if k > p:
            continue
        xs, ys = _distinct(p, 50 + k, k), _rand(p, 60 + k, k)
        ys[k // 2] = p - 1
        if p - 1 not in xs:
            xs[-1] = p - 1
        out = np.full(k + 1, 0xA5A5A5A5A5A5A5A5, np.uint64)                # one guard word after the k terms
        c.call("ronk_poly_interpolate_u64_host", p, _lib._ptr(xs), _lib._ptr(ys), k, _lib._ptr(out))
        assert out[k] == 0xA5A5A5A5A5A5A5A5
        assert np.array_equal(_horner_all(p, out[:k], xs), ys), (hex(p), k)
        if k <= 12:
            assert np.array_equal(out[:k], oracle.rs_decode(p, xs, ys, k)), (hex(p), k)


def test_interpolation_panics_and_cap():
    """At the 8 192 cap a repeated x at positions 0 and k - 1 raises; 8 193 nodes are unsupported; a non-canonical x
    is refused."""
    from ronkathon_b200 import RonkError, RonkPanic, _lib
    c = ctx()
    k = 8192
    xs, ys = _distinct(GL, 99, k + 1), _rand(GL, 98, k + 1)
    out = np.empty(k + 1, np.uint64)
    rep = xs[:k].copy()
    rep[-1] = rep[0]
    with pytest.raises(RonkPanic):
        c.call("ronk_poly_interpolate_u64_host", GL, _lib._ptr(rep), _lib._ptr(ys), k, _lib._ptr(out))
    with pytest.raises(RonkError) as e:
        c.call("ronk_poly_interpolate_u64_host", GL, _lib._ptr(xs), _lib._ptr(ys), k + 1, _lib._ptr(out))
    assert _code(e) == _lib.EUNSUPPORTED
    bad = xs[:33].copy()
    bad[17] = GL
    with pytest.raises(RonkPanic):
        c.call("ronk_poly_interpolate_u64_host", GL, _lib._ptr(bad), _lib._ptr(ys), 33, _lib._ptr(out))
    c.call("ronk_poly_interpolate_u64_host", GL, _lib._ptr(xs), _lib._ptr(ys), 33, _lib._ptr(out))
    assert np.array_equal(_horner_all(GL, out[:33], xs[:33]), ys[:33])


# ---- 6. general polynomial division ---------------------------------------------------------------------------------
def _divisors(p, db, seed):
    r = _rand(p, seed, db)
    top = r.copy()
    top[-1] = p - 1
    low0 = top.copy()
    low0[0] = 0
    xk = np.zeros(db, np.uint64)
    xk[-1] = 1
    out = {"random_top_p-1": top, "b0=0": low0, "x^k": xk}
    if db >= 3:
        tz = r.copy()
        tz[-2:] = 0
        tz[-3] = tz[-3] or 1
        out["trailing_zeros"] = tz
    return out


def _dividends(p, da, seed):
    r = _rand(p, seed, da)
    r[-1] = p - 1
    tz = r.copy()
    if da > 1:
        tz[-min(da - 1, 3):] = 0
    return {"random": r, "zero": np.zeros(da, np.uint64), "trailing_zeros": tz}


@pytest.mark.parametrize("p", [101, 17, GL, BABYBEAR, PBIG], ids=hex)
def test_divrem_general_divisor(p):
    """ronk_poly_divrem_u64_host with divisors that take the general kernel, up to 1 000 terms (past one 256-thread
    CTA): random with top coefficient p - 1, b[0] = 0, x^k, trailing zeros, and [c, 0]; dividends random, all zero and
    with trailing zeros, shorter than, as long as and longer than the divisor.  Where the oracle panics (the
    reference indexes out of range) the library raises."""
    from ronkathon_b200 import RonkPanic, _lib
    c = ctx()

    def check(a, b, tag):
        q, r = np.empty(len(a), np.uint64), np.empty(len(a), np.uint64)
        try:
            eq, er = oracle.poly_divrem(p, a, b)
        except oracle.OraclePanic:
            with pytest.raises(RonkPanic):
                c.call("ronk_poly_divrem_u64_host", p, _lib._ptr(a), len(a), _lib._ptr(b), len(b), _lib._ptr(q),
                       _lib._ptr(r))
            return "panic"
        c.call("ronk_poly_divrem_u64_host", p, _lib._ptr(a), len(a), _lib._ptr(b), len(b), _lib._ptr(q), _lib._ptr(r))
        assert np.array_equal(q, eq) and np.array_equal(r, er), (hex(p), len(a), len(b), tag)
        return "ok"

    seen = set()
    for da, db in ((3, 3), (300, 257), (5000, 256), (5000, 257), (20000, 300), (1000, 1000), (999, 1000)):
        for bname, b in _divisors(p, db, 70 + db).items():
            for aname, a in _dividends(p, da, 80 + da).items():
                if da == 20000 and (aname, bname) not in (("random", "random_top_p-1"), ("trailing_zeros", "x^k")):
                    continue
                seen.add((bname, aname, check(a, b, (bname, aname))))
    for cst in (1, p - 1):                                               # [c, 0]: linear in length, constant in value
        for da in (1, 2, 700):
            a = _rand(p, 90 + da, da)
            seen.add(("[c,0]", "random", check(a, np.array([cst, 0], np.uint64), "[c,0]")))
    a = _rand(p, 91, 700)
    a[-3:] = 0
    b = _rand(p, 92, 5, nonzero=True)
    b[-2:] = 0                                                           # as many trailing zeros in a as b: divides for a while
    seen.add(("trailing_zeros", "trailing_zeros_more", check(a, b, "tz/tz")))
    assert ("trailing_zeros", "random", "panic") in seen                 # both outcomes of a trailing-zero divisor ran
    assert any(s[0] == "trailing_zeros" and s[2] == "ok" for s in seen)


# ---- 7. polynomial add / sub ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("p", MODULI, ids=hex)
def test_poly_add_sub_every_prime_past_one_grid_stride(p):
    """ronk_poly_add_u64 / _sub_u64: out has da terms, b zero-extended or truncated; lengths past one grid stride
    (132·8·256 = 270 336 terms) on either side; all-(p - 1) and random operands."""
    c = ctx()
    for da, db in ((1, 1), (5, 1), (1, 5), (300000, 7), (7, 300000), ((1 << 20) + 3, (1 << 20) + 3)):
        for kind in ("p-1", "random"):
            if kind == "p-1":
                a, b = np.full(da, p - 1, np.uint64), np.full(db, p - 1, np.uint64)
            else:
                a, b = _rand(p, da, da), _rand(p, db + 1, db)
            A, B, out = dev(a), dev(b), _empty(da)
            for name, fn in (("ronk_poly_add_u64", oracle.poly_add), ("ronk_poly_sub_u64", oracle.poly_sub)):
                c.call(name, p, A.data_ptr(), da, B.data_ptr(), db, out.data_ptr())
                assert np.array_equal(host(out), fn(p, a, b)), (hex(p), da, db, kind, name)
            out = _empty(da)                                             # neg = 0 - a, as Polynomial.__neg__ runs it
            Z = dev(np.zeros(da, np.uint64))
            c.call("ronk_poly_sub_u64", p, Z.data_ptr(), da, A.data_ptr(), da, out.data_ptr())
            assert np.array_equal(host(out), oracle.poly_neg(p, a)), (hex(p), da, kind)


# ---- 8. point ops over the whole group ------------------------------------------------------------------------------
def _all_points():
    """E(F_101²): y² = x³ + 3 by a table of squares, Infinity first."""
    q = 101

    def gmul(a, b):
        return ((a[0] * b[0] - 2 * a[1] * b[1]) % q, (a[0] * b[1] + a[1] * b[0]) % q)

    roots = {}
    for y0 in range(q):
        for y1 in range(q):
            roots.setdefault(gmul((y0, y1), (y0, y1)), []).append((y0, y1))
    pts = [oracle.INF]
    for x0 in range(q):
        for x1 in range(q):
            r = gmul(gmul((x0, x1), (x0, x1)), (x0, x1))
            for y in roots.get(((r[0] + 3) % q, r[1]), []):
                pts.append(bytes([x0, x1, y[0], y[1]]))
    assert len(pts) == 102 * 102
    return pts


def _oracle_point_op(fn, *args):
    """One oracle point op through ctypes with no numpy round trip: several hundred thousand of them run here."""
    o = (C.c_uint8 * 4)()
    rc = fn(*[(C.c_uint8 * 4).from_buffer_copy(a) if isinstance(a, bytes) else a for a in args], o)
    assert not rc
    return bytes(o)


def _bytes(points):
    return np.frombuffer(b"".join(points), dtype=np.uint8).copy()


def _split(arr):
    return [bytes(arr[i:i + 4]) for i in range(0, len(arr), 4)]


def _point_call(name, *arrays):
    from ronkathon_b200 import _lib
    out = np.empty(len(arrays[0]) if name != "ronk_point_smul_pluto_ext_host" else 4 * len(arrays[1]), np.uint8)
    n = len(out) // 4
    ctx().call(name, *[_lib._ptr(a) for a in arrays], _lib._ptr(out), n)
    return _split(out)


def test_point_ops_over_the_whole_group():
    """add / neg / smul of ronk_point_*_pluto_ext_host against the oracle for every point of E(F_101²) and Infinity:
    neg of all; every point times every scalar 0 … 16; P + P, P + (-P), P + ∞, ∞ + P for every P; each 2- and
    3-torsion point against every point; 200 000 random pairs; a raw scalar of 17 or 255 raises."""
    from ronkathon_b200 import RonkPanic
    ctx()
    lib = oracle.lib()
    pts = _all_points()
    N = len(pts)
    negs = [oracle.point_neg(P) for P in pts]
    assert _point_call("ronk_point_neg_pluto_ext_host", _bytes(pts)) == negs
    assert negs[0] == oracle.INF and all(oracle.point_add(P, Q) == oracle.INF for P, Q in zip(pts[:50], negs[:50]))
    sm_pts = [P for P in pts for _ in range(17)]
    sm_sc = list(range(17)) * N
    assert _point_call("ronk_point_smul_pluto_ext_host", _bytes(sm_pts), np.array(sm_sc, np.uint8)) == \
        [_oracle_point_op(lib.orc_point_smul, P, s) for P, s in zip(sm_pts, sm_sc)]
    two = [P for P in pts[1:] if P[2] == 0 and P[3] == 0]
    three = [P for P, nP in zip(pts[1:], negs[1:]) if oracle.point_add(P, P) == nP]
    assert len(two) == 3 and len(three) == 8                            # E[2] ≅ (Z/2)², E[3] ≅ (Z/3)²
    lhs = pts + pts + pts + [oracle.INF] * N
    rhs = pts + negs + [oracle.INF] * N + pts
    for T in two + three:
        lhs += [T] * N + pts
        rhs += pts + [T] * N
    rng = np.random.default_rng(8)
    ia, ib = rng.integers(0, N, 200000), rng.integers(0, N, 200000)
    lhs += [pts[i] for i in ia]
    rhs += [pts[i] for i in ib]
    got = _point_call("ronk_point_add_pluto_ext_host", _bytes(lhs), _bytes(rhs))
    assert got == [_oracle_point_op(lib.orc_point_add, P, Q) for P, Q in zip(lhs, rhs)]
    for s in (17, 255):
        sc = np.zeros(300, np.uint8)
        sc[-1] = s
        with pytest.raises(RonkPanic):
            _point_call("ronk_point_smul_pluto_ext_host", _bytes(pts[1:301]), sc)
