"""The device half of ronkathon_b200/csrc/field.cuh, primitive by primitive, through tests/cuda/field_harness.cu:
Goldilocks (inline PTX) add / sub / neg / mul / mul_tw / pow, mul_pow2<S> for every S < 192, w16 / w16_sub in both
directions and the radix-16 butterfly network; MontField add / sub / neg / mul / redc_mul / to_tw / mul_tw / pow,
w16 / w16_sub and the network for every test prime.  Each runs on the structured corpus of tests/field_corpus.py
(which reaches every carry and borrow case) and on random words, bit-exact against exact integers, and where the
CPU emulator has the same primitive, against that host twin too: a result that differs from the exact one while
the host twin is right points at the PTX, not at the formula.  The Goldilocks tests run again on every build of
the harness with an alternative formulation (RONK_FMA_TAIL, RONK_REDUCE_V2=0, RONK_SHIFT_V2=0)."""
import ctypes as C
import functools
import os

import numpy as np
import pytest

import field_corpus as fc
import oracle

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GL = fc.GL
R64 = fc.R64
VARIANTS = ("default", "fma0", "fma11", "fma19", "fma31", "reduce_v1", "shift_v1")
OP = {"add": 0, "sub": 1, "neg": 2, "mul": 3, "mul_tw": 4, "pow": 5, "redc_mul": 6, "to_tw": 7}
P64 = C.POINTER(C.c_uint64)
u64, i32 = C.c_uint64, C.c_int


@functools.lru_cache(maxsize=None)
def harness(variant):
    name = "libfield_harness.so" if variant == "default" else f"libfield_harness_{variant}.so"
    path = os.path.join(HERE, "cuda", name)
    assert os.path.exists(path), f"{name} is missing: run __graft_entry__.build() first"
    lib = C.CDLL(path)
    lib.fh_gl_op.argtypes = [i32, P64, P64, P64, u64]
    lib.fh_gl_mul_pow2.argtypes = [i32, P64, P64, u64]
    lib.fh_gl_w16.argtypes = [i32, i32, i32, P64, P64, P64, u64]
    lib.fh_gl_radix.argtypes = [i32, i32, P64, P64, u64]
    lib.fh_mont_op.argtypes = [u64, i32, P64, P64, P64, u64]
    lib.fh_mont_w16.argtypes = [u64, u64, i32, i32, i32, P64, P64, P64, u64]
    lib.fh_mont_radix.argtypes = [u64, u64, i32, i32, P64, P64, u64]
    return lib


def _arr(x):
    return np.ascontiguousarray(x, dtype=np.uint64)


def call(fn, *head, a, b=None):
    """fn(*head, a, b, out, n) for the element-wise exports (b omitted where fn takes none)."""
    a = _arr(a)
    out = np.full_like(a, 0xDEADBEEFDEADBEEF)
    args = head + ((fc.ptr(a),) if b is False else (fc.ptr(a), fc.ptr(None if b is None else _arr(b))))
    assert fn(*args, fc.ptr(out), len(a)) == 0
    return out


def check(got, exp, what, inputs, twin=None):
    """got == exp bit for bit; on a mismatch, show the first inputs and whether the host twin got them right."""
    if twin is not None and np.array_equal(got, exp) and not np.array_equal(twin, exp):
        bad = np.flatnonzero(twin != exp)[:4]
        pytest.fail(f"{what}: the device is right but the host twin is not at {[hex(int(inputs[0][i])) for i in bad]}")
    if np.array_equal(got, exp):
        return
    bad = np.flatnonzero(got != exp)
    lines = []
    for i in bad[:6]:
        ins = ", ".join(hex(int(x[i])) for x in inputs)
        tw = "" if twin is None else ("  host twin right" if twin[i] == exp[i] else f"  host twin {int(twin[i]):#x}")
        lines.append(f"({ins}) → {int(got[i]):#x}, expected {int(exp[i]):#x}{tw}")
    pytest.fail(f"{what}: {len(bad)} of {len(got)} wrong\n" + "\n".join(lines))


def np_add(p, a, b):
    """(a + b) mod p on uint64 arrays of residues, exactly: a wrap past 2^64 or a sum ≥ p subtracts p."""
    with np.errstate(over="ignore"):
        s = a + b
        return np.where((s < a) | (s >= np.uint64(p)), s - np.uint64(p), s)


def np_sub(p, a, b):
    with np.errstate(over="ignore"):
        return np.where(a >= b, a - b, a - b + np.uint64(p))


# ---- Goldilocks (the inline-PTX path), on every build ---------------------------------------------------------
@functools.lru_cache(maxsize=None)
def gl_random(seed):
    return fc.random_words(GL, seed)


@pytest.mark.parametrize("variant", VARIANTS)
def test_goldilocks_add_sub_neg_mul(variant):
    lib = harness(variant)
    sa, sb = fc.gl_pairs()
    for op, host_op in (("add", 0), ("sub", 1), ("mul", 2), ("mul_tw", 2)):
        got = call(lib.fh_gl_op, OP[op], a=sa, b=sb)
        check(got, fc.exact("mul" if op == "mul_tw" else op, GL, sa, sb), op, (sa, sb), fc.host_field_op(GL, host_op, sa, sb))
    v = np.array(fc.gl_values(), dtype=np.uint64)
    check(call(lib.fh_gl_op, OP["neg"], a=v), fc.exact("neg", GL, v), "neg", (v,), fc.host_field_op(GL, 3, v))
    ra, rb = gl_random(1), gl_random(2)
    check(call(lib.fh_gl_op, OP["add"], a=ra, b=rb), np_add(GL, ra, rb), "add (random)", (ra, rb))
    check(call(lib.fh_gl_op, OP["sub"], a=ra, b=rb), np_sub(GL, ra, rb), "sub (random)", (ra, rb))
    check(call(lib.fh_gl_op, OP["neg"], a=ra), np_sub(GL, np.zeros_like(ra), ra), "neg (random)", (ra,))
    rm = oracle.vec_mul(GL, ra, rb)
    check(call(lib.fh_gl_op, OP["mul"], a=ra, b=rb), rm, "mul (random)", (ra, rb))
    check(call(lib.fh_gl_op, OP["mul_tw"], a=ra, b=rb), rm, "mul_tw (random)", (ra, rb))


@functools.lru_cache(maxsize=None)
def gl_shift_expected(S):
    x = np.array(fc.gl_shift_inputs(S), dtype=np.uint64)
    return x, fc.exact("mul", GL, x, [pow(2, S, GL)] * len(x)), fc.host_gl_shift(0, S, False, x)


@pytest.mark.parametrize("variant", VARIANTS)
def test_goldilocks_mul_pow2_every_shift(variant):
    """mul_pow2<S> for every S in [0, 192): the structured inputs of S (preimages that put shl_a / shl_b / shl_c's
    words on the 32-bit boundaries) and 2^20 random words."""
    lib = harness(variant)
    r = gl_random(3)
    for S in range(192):
        x, exp, twin = gl_shift_expected(S)
        check(call(lib.fh_gl_mul_pow2, S, a=x, b=False), exp, f"mul_pow2<{S}>", (x,), twin)
        check(call(lib.fh_gl_mul_pow2, S, a=r, b=False), oracle.vec_mul(GL, r, np.full(len(r), pow(2, S, GL), np.uint64)),
              f"mul_pow2<{S}> (random)", (r,))


@pytest.mark.parametrize("variant", VARIANTS)
def test_goldilocks_w16_and_w16_sub(variant):
    """w16<E, INV>(a) = a·ω16^±E and w16_sub<E, INV>(a, b) = (a − b)·ω16^±E for E < 8, both directions, ω16 = 7^((p−1)/16),
    on the shift corpus of each E's shift (reached through the subtraction for w16_sub) and on random words."""
    lib = harness(variant)
    w16 = oracle.root_of_unity(GL, 16)
    ra, rb = gl_random(4), gl_random(5)
    for inverse in (False, True):
        for e in range(8):
            w = pow(w16, -e if inverse else e, GL)
            S = fc.w16_shift(e, inverse)
            assert pow(2, S, GL) == w
            what = f"w16<{e}, {inverse}>"
            x = np.array(fc.gl_shift_inputs(S), dtype=np.uint64)
            check(call(lib.fh_gl_w16, e, int(inverse), 0, a=x), fc.exact("mul", GL, x, [w] * len(x)), what, (x,),
                  gl_shift_expected(S)[2])
            a, b = fc.gl_w16_sub_operands(S)
            check(call(lib.fh_gl_w16, e, int(inverse), 1, a=a, b=b), fc.exact("mul", GL, fc.exact("sub", GL, a, b), [w] * len(a)),
                  "w16_sub" + what[3:], (a, b), fc.host_gl_shift(1, e, inverse, a, b))
            wv = np.full(len(ra), w, np.uint64)
            check(call(lib.fh_gl_w16, e, int(inverse), 0, a=ra), oracle.vec_mul(GL, ra, wv), what + " (random)", (ra,))
            check(call(lib.fh_gl_w16, e, int(inverse), 1, a=ra, b=rb), oracle.vec_mul(GL, np_sub(GL, ra, rb), wv),
                  "w16_sub" + what[3:] + " (random)", (ra, rb))


POW_EXPONENTS = (0, 1, 2, 3, 7, 2**32 - 1, 2**32, 2**63, 2**64 - 1, GL - 2, GL - 1, GL, (GL - 1) // 2, (GL - 1) // 16)


def pow_operands(p, values, seed, n_random):
    """Every structured value to each exponent of POW_EXPONENTS (and p − 2, p − 1, (p − 1)/2), then random bases to
    random 64-bit exponents."""
    exps = sorted(set(POW_EXPONENTS) | {p - 2, p - 1, (p - 1) // 2})
    a = [v for v in values for _ in exps]
    e = [x for _ in values for x in exps]
    rb = oracle.splitmix(p, seed, n_random)
    re = np.random.default_rng(seed).integers(0, 2**64 - 1, n_random, dtype=np.uint64, endpoint=True)
    return np.array(a, dtype=np.uint64), np.array(e, dtype=np.uint64), rb, re


@pytest.mark.parametrize("variant", VARIANTS)
def test_goldilocks_field_pow(variant):
    lib = harness(variant)
    a, e, rb, re = pow_operands(GL, fc.gl_values(), 6, 1 << 14)
    check(call(lib.fh_gl_op, OP["pow"], a=a, b=e), fc.exact("pow", GL, a, e), "field_pow", (a, e))
    exp = np.array([oracle.pow_(GL, int(x), int(y)) for x, y in zip(rb, re)], dtype=np.uint64)
    check(call(lib.fh_gl_op, OP["pow"], a=rb, b=re), exp, "field_pow (random)", (rb, re))


def bitrev(q, bits):
    return int(format(q, f"0{bits}b")[::-1], 2) if bits else 0


def radix_groups(p, values, seed, n_random):
    """16-word groups: all p − 1, alternating 0 / p − 1 (both phases), each value alone in a field of zeros at each of
    the 16 positions, then random groups."""
    groups = [[p - 1] * 16, [0, p - 1] * 8, [p - 1, 0] * 8]
    for v in values:
        for i in range(16):
            g = [0] * 16
            g[i] = v
            groups.append(g)
    out = np.concatenate([np.array(groups, dtype=np.uint64).reshape(-1), oracle.splitmix(p, seed, 16 * n_random)])
    return out


def radix_expected(p, g, x, nst, inverse):
    """radix_network<nst>: independent 2^nst-point DFTs on consecutive blocks of 2^nst registers (ω = g^((p−1)/2^nst),
    its inverse for INV, no scaling), each output at the bit-reversed position of its block."""
    n = 1 << nst
    gg = pow(g, -1, p) if inverse else g
    blocks = x.reshape(-1, n)
    out = np.empty_like(blocks)
    perm = [bitrev(q, nst) for q in range(n)]
    for i, blk in enumerate(blocks):
        out[i] = oracle.dft(p, blk, g=gg)[perm]
    return out.reshape(-1)


@functools.lru_cache(maxsize=None)
def gl_radix_case(nst, inverse):
    x = radix_groups(GL, fc.gl_values(), 7, 4096)
    return x, radix_expected(GL, 7, x, nst, inverse)


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("inverse", [False, True])
@pytest.mark.parametrize("nst", [1, 2, 3, 4])
def test_goldilocks_radix_network(variant, nst, inverse):
    """radix_network<NST, INV> with 16 values live per thread, as in the transform kernels: <4> is one 16-point DFT at
    bit-reversed positions, <3> two 8-point DFTs on x[0..7] and x[8..15], <2> four 4-point, <1> eight 2-point."""
    lib = harness(variant)
    x, exp = gl_radix_case(nst, inverse)
    got = np.full_like(x, 0xDEADBEEFDEADBEEF)
    assert lib.fh_gl_radix(nst, int(inverse), fc.ptr(x), fc.ptr(got), len(x) // 16) == 0
    check(got, exp, f"radix_network<{nst}, {inverse}>", (x,))


# ---- MontField, every test prime (the policy is plain C++: the switches do not touch it) ------------------------
MONT = list(fc.MONT_PRIMES.items())


@pytest.mark.parametrize("name,p", MONT, ids=[n for n, _ in MONT])
def test_mont_add_sub_neg_mul_redc_tw(name, p):
    lib = harness("default")
    sa, sb = fc.mont_pairs(p)
    ra, rb = oracle.splitmix(p, 11, 1 << 18), oracle.splitmix(p, 12, 1 << 18)
    rinv = pow(R64, -1, p)
    for op, host_op in (("add", 0), ("sub", 1), ("mul", 2)):
        got = call(lib.fh_mont_op, p, OP[op], a=sa, b=sb)
        check(got, fc.exact(op, p, sa, sb), f"{op} mod {name}", (sa, sb), fc.host_field_op(p, host_op, sa, sb, force_mont=True))
    v = np.array(fc.mont_values(p), dtype=np.uint64)
    check(call(lib.fh_mont_op, p, OP["neg"], a=v), fc.exact("neg", p, v), f"neg mod {name}", (v,),
          fc.host_field_op(p, 3, v, force_mont=True))
    redc = np.array([int(x) * int(y) * rinv % p for x, y in zip(sa, sb)], dtype=np.uint64)
    check(call(lib.fh_mont_op, p, OP["redc_mul"], a=sa, b=sb), redc, f"redc_mul mod {name}", (sa, sb))
    check(call(lib.fh_mont_op, p, OP["to_tw"], a=v), np.array([int(x) * R64 % p for x in v], dtype=np.uint64),
          f"to_tw mod {name}", (v,))
    b_mont = np.array([int(y) * R64 % p for y in sb], dtype=np.uint64)   # the twiddle form, supplied by the test
    check(call(lib.fh_mont_op, p, OP["mul_tw"], a=sa, b=b_mont), fc.exact("mul", p, sa, sb), f"mul_tw mod {name}", (sa, b_mont))
    check(call(lib.fh_mont_op, p, OP["add"], a=ra, b=rb), np_add(p, ra, rb), f"add mod {name} (random)", (ra, rb))
    check(call(lib.fh_mont_op, p, OP["sub"], a=ra, b=rb), np_sub(p, ra, rb), f"sub mod {name} (random)", (ra, rb))
    check(call(lib.fh_mont_op, p, OP["mul"], a=ra, b=rb), oracle.vec_mul(p, ra, rb), f"mul mod {name} (random)", (ra, rb))
    rb_mont = oracle.vec_mul(p, rb, np.full(len(rb), R64 % p, np.uint64))
    check(call(lib.fh_mont_op, p, OP["mul_tw"], a=ra, b=rb_mont), oracle.vec_mul(p, ra, rb), f"mul_tw mod {name} (random)",
          (ra, rb_mont))
    a, e, pb, pe = pow_operands(p, fc.mont_values(p)[:64], 13, 1 << 12)
    check(call(lib.fh_mont_op, p, OP["pow"], a=a, b=e), fc.exact("pow", p, a, e), f"field_pow mod {name}", (a, e))
    exp = np.array([oracle.pow_(p, int(x), int(y)) for x, y in zip(pb, pe)], dtype=np.uint64)
    check(call(lib.fh_mont_op, p, OP["pow"], a=pb, b=pe), exp, f"field_pow mod {name} (random)", (pb, pe))



@pytest.mark.parametrize("name,p", MONT, ids=[n for n, _ in MONT])
def test_mont_w16_and_radix_network(name, p):
    """w16 / w16_sub against the table make_mont_field builds (ω16^e where the 2-adicity k ≤ 4 allows it, 1 elsewhere),
    and radix_network<NST> for every NST ≤ k against the oracle's DFT."""
    lib = harness("default")
    g = fc.generator(p)
    k = min(fc.two_adicity(p), 4)
    stride = 16 >> k
    v = np.array(fc.mont_values(p), dtype=np.uint64)
    a, b = oracle.splitmix(p, 21, 1 << 14), oracle.splitmix(p, 22, 1 << 14)
    a = np.concatenate([v, np.zeros_like(v), a])
    b = np.concatenate([np.zeros_like(v), v, b])
    for inverse in (False, True):
        w = pow(g, (p - 1) >> k, p)
        if inverse:
            w = pow(w, -1, p)
        for e in range(8):
            f = pow(w, e // stride, p) if e % stride == 0 else 1
            what = f"w16<{e}, {inverse}> mod {name}"
            check(call(lib.fh_mont_w16, p, g, e, int(inverse), 0, a=a), fc.exact("mul", p, a, [f] * len(a)), what, (a,))
            check(call(lib.fh_mont_w16, p, g, e, int(inverse), 1, a=a, b=b),
                  fc.exact("mul", p, fc.exact("sub", p, a, b), [f] * len(a)), "w16_sub" + what[3:], (a, b))
        x = radix_groups(p, fc.mont_values(p)[:64], 23, 512)
        for nst in range(1, k + 1):
            got = np.full_like(x, 0xDEADBEEFDEADBEEF)
            assert lib.fh_mont_radix(p, g, nst, int(inverse), fc.ptr(x), fc.ptr(got), len(x) // 16) == 0
            check(got, radix_expected(p, g, x, nst, inverse), f"radix_network<{nst}, {inverse}> mod {name}", (x,))
