"""Inputs that reach every carry and borrow case of the field arithmetic in ronkathon_b200/csrc/field.cuh, and a
predicate per case its derivations name, so a test can show which cases a corpus reaches.  Shared by the CPU
emulator tests (the host twin of field.cuh) and the device tests (tests/cuda/field_harness.cu).  Importable
without a GPU.

Random data reaches some of these cases about once in 2^32 operations (a 32-bit word of all ones in the right
place), so the corpus is built from words on the 32-bit boundaries instead, and for the shift forms from
preimages that put the shifted words themselves on those boundaries."""
import ctypes as C
import functools
import os
import subprocess

import numpy as np

import oracle

GL = oracle.GOLDILOCKS
M32 = (1 << 32) - 1
M64 = (1 << 64) - 1
EPS = M32                       # 2^64 mod GL
R64 = 1 << 64                   # the Montgomery radix
MIN_HITS = 16                   # every case must be reached at least this often by the corpus handed to an op

# 32-bit words on either side of every boundary a carry chain can cross
BOUNDARY_WORDS = (0, 1, 2, 3, 2**31 - 1, 2**31, 2**31 + 1, 2**32 - 3, 2**32 - 2, 2**32 - 1)
# a wider set for the low word of a shift preimage, whose low S mod 32 bits are shifted out
LOW_WORDS = tuple(sorted(set(BOUNDARY_WORDS) | {1 << k for k in range(32)} | {(1 << 32) - (1 << k) for k in range(32)}))

# Test primes for MontField (name → p): tiny ones with every residue, both sides of 2^32 and 2^63, and the
# largest 64-bit primes.
MONT_PRIMES = {
    "3": 3, "5": 5, "17": 17, "101": 101, "127": 127, "65537": 65537, "m31": 2**31 - 1,
    "babybear": 2013265921, "koalabear": 2130706433, "2^32-5": 2**32 - 5, "2^32+15": 2**32 + 15,
    "p32": 0x100050001, "p57": 29 * 2**57 + 1, "m61": 2**61 - 1, "2^63-25": 2**63 - 25, "2^63+29": 2**63 + 29,
    "pbig": 0xFFFFFFFF70000001, "goldilocks": GL, "2^64-279": 2**64 - 279, "2^64-59": 2**64 - 59,
}
EXHAUSTIVE_BELOW = 128          # below this, the corpus holds every residue (and every pair of residues)


def is_prime(n):
    """Deterministic Miller–Rabin: these twelve bases decide every n < 3.3·10^24."""
    if n < 2:
        return False
    bases = (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37)
    for q in bases:
        if n % q == 0:
            return n == q
    d, r = n - 1, 0
    while d % 2 == 0:
        d, r = d // 2, r + 1
    for a in bases:
        x = pow(a, d, n)
        if x in (1, n - 1):
            continue
        for _ in range(r - 1):
            x = x * x % n
            if x == n - 1:
                break
        else:
            return False
    return True


def generator(p):
    """The smallest quadratic non-residue mod p: then g^((p-1)/2^k) has order exactly 2^k for every 2^k | p - 1."""
    return next(g for g in range(2, p) if pow(g, (p - 1) // 2, p) == p - 1)


def two_adicity(p):
    return ((p - 1) & -(p - 1)).bit_length() - 1


# ---- Goldilocks values --------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def gl_values():
    """hi·2^32 + lo for boundary words hi, lo; p − v for each; 2^j, 2^j ± 1 and p − 2^j.  All below p, sorted."""
    words = [(hi << 32) | lo for hi in BOUNDARY_WORDS for lo in BOUNDARY_WORDS]
    vals = set(words) | {GL - v for v in words}
    for j in range(64):
        vals |= {1 << j, (1 << j) + 1, (1 << j) - 1, GL - (1 << j)}
    return tuple(sorted(v for v in vals if 0 <= v < GL))


@functools.lru_cache(maxsize=None)
def gl_shift_preimages(s):
    """x = ⌊T / 2^s⌋ (s = S mod 32) for 96-bit patterns T = (t2 : t1 : t0) with t2 < 2^s on either side of 0 and
    2^s − 1, t1 a boundary word and t0 from LOW_WORDS: x·2^s = (y2 : y1 : y0) then has its words on the boundaries
    (y0 = t0 without its low s bits).  Kept if below p."""
    tops = ({w & ((1 << s) - 1) for w in BOUNDARY_WORDS} | {max((1 << s) - k, 0) for k in (1, 2, 3)}
            | set(range(min(1 << s, 32))))
    out = set()
    for t2 in tops:
        for t1 in BOUNDARY_WORDS:
            for t0 in LOW_WORDS:
                x = ((t2 << 64) | (t1 << 32) | t0) >> s
                if x < GL:
                    out.add(x)
    return tuple(sorted(out))


def gl_shift_inputs(S):
    """The structured inputs for mul_pow2<S>."""
    return tuple(sorted(set(gl_values()) | set(gl_shift_preimages(S % 32))))


@functools.lru_cache(maxsize=None)
def gl_pairs():
    """Every pair of gl_values(): the structured operands of add, sub and mul."""
    v = np.array(gl_values(), dtype=np.uint64)
    return np.repeat(v, len(v)), np.tile(v, len(v))


def random_words(p, seed, n=1 << 20):
    return oracle.splitmix(p, seed, n)


# ---- Goldilocks cases -----------------------------------------------------------------------------------------
def gl_add_cases(a, b):
    s = a + b
    return ("sum_lt_p",) if s < GL else ("sum_in_p_2_64",) if s < R64 else ("sum_carries_2_64",)


def sub_cases(a, b):
    return ("a_ge_b",) if a >= b else ("a_lt_b",)


def gl_mul_cases(a, b):
    """reduce_words on the product's words r0..r3: Y = r2·EPS + r0, t = Y − r3 (+p on a borrow), then
    t + (r1 : 2^32 − 1) carries or not."""
    x = a * b
    r0, r1, r2, r3 = x & M32, (x >> 32) & M32, (x >> 64) & M32, x >> 96
    y = r2 * EPS + r0
    t = y - r3 if y >= r3 else y - r3 + GL
    cases = ["Y_lt_r3" if y < r3 else "Y_ge_r3", "step2_carry" if t + ((r1 << 32) | M32) >= R64 else "step2_no_carry"]
    if r1 == 0:
        cases.append("r1_zero")
    if r1 == M32:
        cases.append("r1_max")
    if r3 == M32 - 1:
        cases.append("r3_max")
    return tuple(cases)


GL_MUL_CASES = ("Y_lt_r3", "Y_ge_r3", "step2_carry", "step2_no_carry", "r1_zero", "r1_max", "r3_max")


def gl_shift_form(S):
    """Which single-correction form of field.cuh computes mul_pow2<S> (S ≥ 96 is the negation of S − 96)."""
    s = S % 96
    return None if s == 0 else "shl_a" if s < 32 else "shl_b" if s < 64 else "shl_c"


SHIFT_CASES = {
    None: ("identity",),
    "shl_a": ("a_y10_ge_p", "a_y10_lt_p", "a_y2_zero", "a_y2_max"),
    "shl_b": ("b_c1", "b_c0", "b_b1_one", "b_b1_zero", "b_borrow", "b_no_borrow"),
    "shl_c": ("c_borrow", "c_no_borrow"),
}


def gl_shift_cases(S, x):
    s = S % 96
    form = gl_shift_form(S)
    if form is None:
        return ("identity",)
    if form == "shl_a":        # x·2^s = (y2 : y1 : y0), result (y1:y0) + y2·EPS
        y = x << s
        y0, y1, y2 = y & M32, (y >> 32) & M32, y >> 64
        cases = ["a_y10_ge_p" if ((y1 << 32) | y0) >= GL else "a_y10_lt_p"]
        if y2 == 0:
            cases.append("a_y2_zero")
        if y2 == (1 << s) - 1:
            cases.append("a_y2_max")
        return tuple(cases)
    if form == "shl_b":        # y = x·2^(s−32); ((y0 + y1 mod B) + c : 0) − (y1 + y2 + c)
        y = x << (s - 32)
        y0, y1, y2 = y & M32, (y >> 32) & M32, y >> 64
        c = (y0 + y1) >> 32
        hi = ((y0 + y1) & M32) + c
        b = y1 + y2 + c
        return ("b_c1" if c else "b_c0", "b_b1_one" if b >> 32 else "b_b1_zero",
                "b_borrow" if (hi << 32) < b else "b_no_borrow")
    k = 96 - s                 # shl_c: (v : 0) − ((x >> k) + v), v = x0·2^(32−k) mod B
    x0 = x & M32
    v = x0 if k == 32 else (x0 << (32 - k)) & M32
    return ("c_borrow" if (v << 32) < (x >> k) + v else "c_no_borrow",)


# Cases that fewer than MIN_HITS inputs below p reach at all: (case) → (how many inputs reach it, why).  The corpus
# holds every one of them, and the coverage test checks that it reaches each exactly that often.
GL_MUL_SMALL = {
    "r3_max": (3, "a·b ≥ (2^32 − 2)·2^96 = p² − 3·2^64 + 2^33 − 1 only for (p − 1)² and (p − 1)(p − 2) in both orders"),
}
_SHL_B_BORROW = ("the borrow needs hi = 0, i.e. y0 = y1 = 0: x = t·2^(64 − s') for 0 < t < 2^s', s' = S − 32")
GL_SHIFT_SMALL = {}
for _S0 in (32, 128):   # mul_pow2<128> = −mul_pow2<32>: the same shl_b<0>
    GL_SHIFT_SMALL[(_S0, "b_borrow")] = (0, "y2 = 0: hi·2^32 ≥ y1 + c whenever hi > 0, and hi = 0 forces y0 = y1 = 0")
    GL_SHIFT_SMALL[(_S0, "b_b1_one")] = (0, "y1 + c = 2^32 needs x1 = 2^32 − 1 and x0 ≥ 1, i.e. x ≥ p")
    for _sp in range(1, 5):
        GL_SHIFT_SMALL[(_S0 + _sp, "b_borrow")] = ((1 << _sp) - 1, _SHL_B_BORROW)


def w16_shift(e, inverse):
    """The shift of ω16^±e = 2^(±156·e mod 192) (field.cuh: ω16 = 2^156 for g = 7)."""
    fwd = (156 * e) % 192
    return (192 - fwd) % 192 if inverse else fwd


def gl_w16_sub_operands(S):
    """Operands (a, b) for w16_sub with shift S: (x, 0), (0, x) and (x + d, d) for x in the shift corpus of S, so
    that the difference reaching mul_pow2 (a − b, or b − a where the sign is folded in) runs over that corpus."""
    x = np.array(gl_shift_inputs(S), dtype=np.uint64)
    d = oracle.splitmix(GL, 1000 + S, len(x))
    zero = np.zeros_like(x)
    return np.concatenate([x, zero, exact("add", GL, x, d)]), np.concatenate([zero, x, d])


# ---- Montgomery -------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def mont_values(p):
    """Every residue below EXHAUSTIVE_BELOW; otherwise boundary words and their distance to p, 2^j (±1) mod p and
    p − 2^j, R mod p and R^-1 mod p, 1 and 2 either side of p/2."""
    if p < EXHAUSTIVE_BELOW:
        return tuple(range(p))
    base = set(BOUNDARY_WORDS) | {(hi << 32) | lo for hi in (0, 1, 2**31, M32) for lo in BOUNDARY_WORDS}
    vals = {v % p for v in base} | {(p - v) % p for v in base}
    for j in range(64):
        vals |= {(1 << j) % p, ((1 << j) + 1) % p, ((1 << j) - 1) % p, (p - (1 << j)) % p}
    vals |= {R64 % p, pow(R64, -1, p), p // 2 - 1, p // 2, p // 2 + 1, p // 2 + 2}
    return tuple(sorted(vals))


@functools.lru_cache(maxsize=None)
def mont_pairs(p):
    """Every pair of mont_values(p), plus pairs whose REDC lands next to 0 and next to p (a·b·R^-1 ≡ c for
    c ∈ {1, 2, p − 1, p − 2}): there hi − mp is small, or small below zero, so both sides of hi < mp are near."""
    v = mont_values(p)
    a = [x for x in v for _ in v]
    b = [y for _ in v for y in v]
    if p >= EXHAUSTIVE_BELOW:
        for x in [x for x in v if x][:64]:
            xinv = pow(x, -1, p)
            for c in (1, 2, p - 1, p - 2):
                a.append(x)
                b.append(c * R64 % p * xinv % p)
    return np.array(a, dtype=np.uint64), np.array(b, dtype=np.uint64)


def mont_add_cases(p, a, b):
    s = a + b
    return ("sum_carries_2_64",) if s >= R64 else ("sum_ge_p",) if s >= p else ("sum_lt_p",)


def redc_cases(p, a, b):
    """redc_mul: t = hi − mp with mp = ⌊m·p / 2^64⌋, m = lo·p^-1 mod 2^64; + p when hi < mp."""
    x = a * b
    lo, hi = x & M64, x >> 64
    m = lo * pow(p, -1, R64) & M64
    return ("hi_lt_mp",) if hi < (m * p) >> 64 else ("hi_ge_mp",)


def mont_add_expected_cases(p):
    """Cases of MontField::add a corpus can reach: a sum ≥ 2^64 needs p > 2^63."""
    return ("sum_lt_p", "sum_ge_p") + (("sum_carries_2_64",) if p > 2**63 else ())


def mont_redc_expected_cases(p):
    return ("hi_lt_mp", "hi_ge_mp")


def exact(op, p, a, b=None):
    """The exact residue of one field operation on Python integers."""
    a = [int(x) for x in a]
    b = None if b is None else [int(y) for y in b]
    if op == "add":
        out = [(x + y) % p for x, y in zip(a, b)]
    elif op == "sub":
        out = [(x - y) % p for x, y in zip(a, b)]
    elif op == "neg":
        out = [-x % p for x in a]
    elif op == "mul":
        out = [x * y % p for x, y in zip(a, b)]
    elif op == "pow":
        out = [pow(x, y, p) for x, y in zip(a, b)]
    else:
        raise ValueError(op)
    return np.array(out, dtype=np.uint64)


# ---- the host twin: field.cuh compiled for the CPU (tests/emu/ntt_emu.cpp) --------------------------------------
_HERE = os.path.dirname(os.path.abspath(__file__))
_P64 = C.POINTER(C.c_uint64)
_emu = None


def ptr(a):
    return None if a is None else a.ctypes.data_as(_P64)


def host_twin():
    """tests/emu/libntt_emu.so, built with g++ when older than its sources: field.cuh's portable host path and the
    kernel headers on the CPU."""
    global _emu
    if _emu is not None:
        return _emu
    csrc = os.path.join(_HERE, "..", "ronkathon_b200", "csrc")
    src = os.path.join(_HERE, "emu", "ntt_emu.cpp")
    so = os.path.join(_HERE, "emu", "libntt_emu.so")
    deps = [src] + [os.path.join(csrc, h) for h in ("ntt_kernel.cuh", "field.cuh", "ntt12_kernel.cuh", "ntt3_kernel.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(x) for x in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", so, src])
    lib = C.CDLL(so)
    lib.emu_ntt.argtypes = [C.c_uint64, C.c_uint64, _P64, _P64, C.c_uint32, C.c_uint32, C.c_int, C.c_uint32, C.c_uint32,
                            C.c_uint32]
    lib.emu_ntt_bounded.argtypes = [C.c_uint64, C.c_uint64, _P64, C.c_uint64, _P64, C.c_uint64, _P64, C.c_uint32, C.c_int,
                                    C.c_uint32, C.c_uint32, C.c_uint32]
    lib.emu_field_op.argtypes = [C.c_uint64, C.c_int, _P64, _P64, _P64, C.c_uint64, C.c_int]
    lib.emu_gl_w16.argtypes = [C.c_uint64, _P64]
    lib.emu_gl_shift_op.argtypes = [C.c_int, C.c_int, C.c_int, _P64, _P64, _P64, C.c_uint64]
    lib.emu_swizzle_worst_conflict.argtypes = [C.c_uint32, C.c_uint32]
    lib.emu_fast12_tiles.restype = C.c_uint64
    lib.emu_ntt3.argtypes = [_P64, _P64, C.c_uint32, C.c_uint32, C.c_int, C.c_int]
    lib.emu_ntt3_bounded.argtypes = [_P64, C.c_uint64, _P64, C.c_uint64, _P64, C.c_int]
    lib.emu_ntt16_cluster.argtypes = [_P64, _P64, C.c_uint32, C.c_int]
    lib.emu_ntt3_shared_mul.argtypes = [_P64, _P64, C.c_uint32, C.c_uint32]
    _emu = lib
    return lib


def host_field_op(p, op, a, b=None, force_mont=False):
    """emu_field_op: op 0 add, 1 sub, 2 mul, 3 neg; Goldilocks takes GoldilocksField unless force_mont."""
    a = np.ascontiguousarray(a, dtype=np.uint64)
    b = a if b is None else np.ascontiguousarray(b, dtype=np.uint64)
    out = np.empty_like(a)
    assert host_twin().emu_field_op(p, op, ptr(a), ptr(b), ptr(out), len(a), int(force_mont)) == 0
    return out


def host_gl_shift(op, k, inverse, a, b=None):
    """emu_gl_shift_op: op 0 mul_pow2<k>(a), op 1 w16_sub<k, inverse>(a, b)."""
    a = np.ascontiguousarray(a, dtype=np.uint64)
    b = None if b is None else np.ascontiguousarray(b, dtype=np.uint64)
    out = np.empty_like(a)
    assert host_twin().emu_gl_shift_op(op, k, int(inverse), ptr(a), ptr(b), ptr(out), len(a)) == 0
    return out


def count_cases(fn, *operands):
    counts = {}
    for ops in zip(*operands):
        for c in fn(*(int(o) for o in ops)):
            counts[c] = counts.get(c, 0) + 1
    return counts
