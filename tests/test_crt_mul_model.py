"""The multi-modular product of ronk_poly_mul_u64 (poly_crt.cu, crt.cuh) on the CPU.

The auxiliary primes are pinned here, and so are Garner's constants and the prime-count rule at its edges.  A Python
big-integer restatement of the whole path (reduce, convolve modulo each q_i by its power-of-two transform, Garner, mod
p) is checked against the oracle's schoolbook product.  The Garner step itself, crt.cuh compiled for the host
(tests/emu/crt_emu.cpp), is checked on edge residues against the Chinese remainder theorem in Python integers."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

import oracle

GL = oracle.GOLDILOCKS
Q = (GL, 0xFFFFFFFF70000001, 29 * 2**57 + 1)
G = (7, 3, 3)
MAX_LEN = 1 << 26                # the longest product the path takes
P64 = C.POINTER(C.c_uint64)
# test moduli: the reference's fields, primes without 2-power roots on both sides of 2^32 and 2^63, an NTT prime past its
# 2-adicity, and primes above every q_i
PRIMES = (101, 17, 127, 65537, 2**31 - 1, 4295294977, 2**61 - 1, 2**63 - 25, 2**63 + 29, 2**64 - 279, 2**64 - 59)

_HERE = os.path.dirname(os.path.abspath(__file__))


def is_prime(n):
    """Deterministic Miller–Rabin for n < 3.3·10^24 (the first 13 prime bases)."""
    if n < 2:
        return False
    bases = (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37, 41)
    for b in bases:
        if n % b == 0:
            return n == b
    d, s = n - 1, 0
    while d % 2 == 0:
        d, s = d // 2, s + 1
    for b in bases:
        x = pow(b, d, n)
        if x in (1, n - 1):
            continue
        for _ in range(s - 1):
            x = x * x % n
            if x == n - 1:
                break
        else:
            return False
    return True


def two_adicity(n):
    return ((n - 1) & -(n - 1)).bit_length() - 1


def prime_count(p, m):
    """The smallest k with q_1⋯q_k > m·(p - 1)², the bound on the integer product's coefficients (0: none)."""
    bound, Qk = m * (p - 1) ** 2, 1
    for k, q in enumerate(Q, 1):
        Qk *= q
        if Qk > bound:
            return k
    return 0


def crt(res, p):
    """The x < q_1⋯q_k with x ≡ res[i] (mod q_i), mod p: Python integers."""
    x, M = 0, 1
    for c, q in zip(res, Q):
        t = (c - x) * pow(M, -1, q) % q
        x, M = x + M * t, M * q
    return x % p


def ntt(a, q, g, n, inverse=False):
    """The n-point transform mod q with ω = g^((q-1)/n), by the O(n²) definition (sizes here are small)."""
    w = pow(g, (q - 1) // n, q)
    if inverse:
        w = pow(w, -1, q)
    a = list(a) + [0] * (n - len(a))
    out = [sum(x * pow(w, i * j, q) for j, x in enumerate(a)) % q for i in range(n)]
    if inverse:
        ninv = pow(n, -1, q)
        out = [x * ninv % q for x in out]
    return out


def model_mul(p, a, b, k=None):
    """The path of crt_mul_device in Python integers: a·b mod p from k residue products (default: the prime count)."""
    L = len(a) + len(b) - 1
    n = 1 << (L - 1).bit_length()
    k = prime_count(p, min(len(a), len(b))) if k is None else k
    residues = []
    for q, g in zip(Q[:k], G[:k]):
        ra, rb = [x % q for x in a], [x % q for x in b]      # crt_reduce when q < p; a no-op otherwise
        A, B = ntt(ra, q, g, n), ntt(rb, q, g, n)
        residues.append(ntt([x * y % q for x, y in zip(A, B)], q, g, n, inverse=True)[:L])
    return [crt([r[i] for r in residues], p) for i in range(L)]


@pytest.fixture(scope="module")
def emu():
    src = os.path.join(_HERE, "emu", "crt_emu.cpp")
    so = os.path.join(_HERE, "emu", "libcrt_emu.so")
    deps = [src] + [os.path.join(_HERE, "..", "ronkathon_b200", "csrc", h) for h in ("crt.cuh", "field.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(x) for x in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, src])
    lib = C.CDLL(so)
    lib.emu_crt_prime_count.argtypes = [C.c_uint64, C.c_uint64]
    lib.emu_crt_primes.argtypes = [P64]
    lib.emu_crt_consts.argtypes = [C.c_uint64, P64]
    lib.emu_crt_garner.argtypes = [C.c_uint64, C.c_int, P64, P64, P64, P64, C.c_uint64]
    lib.emu_crt_below.argtypes = [C.c_uint64, P64, P64, C.c_uint64]
    return lib


def _ptr(a):
    return a.ctypes.data_as(P64)


def test_the_primes():
    """Each q_i is prime, has 2-adicity ≥ 26 (every transform of the path), and its g is a quadratic non-residue, so
    g^((q-1)/2^s) has order exactly 2^s; the product of the three exceeds the largest bound the path can meet."""
    for q, g in zip(Q, G):
        assert is_prime(q), hex(q)
        assert two_adicity(q) >= 26, hex(q)
        assert pow(g, (q - 1) // 2, q) == q - 1, hex(q)
    assert [two_adicity(q) for q in Q] == [32, 28, 57]
    assert Q[0] < Q[1] and Q[2] < Q[0]
    assert Q[0] * Q[1] * Q[2] > (MAX_LEN // 2) * (2**64 - 2) ** 2


def test_emulator_primes_match(emu):
    out = np.zeros(6, dtype=np.uint64)
    emu.emu_crt_primes(_ptr(out))
    assert [int(v) for v in out] == list(Q) + list(G)


@pytest.mark.parametrize("p", (101, 4295294977, 2**64 - 279, GL))
def test_garner_constants(emu, p):
    out = np.zeros(6, dtype=np.uint64)
    emu.emu_crt_consts(p, _ptr(out))
    q1, q2, q3 = Q
    inv12 = pow(q1 * q2, -1, q3)
    assert [int(v) for v in out] == [pow(q1, -1, q2), inv12, q1 * inv12 % q3, 1 % p, q1 % p, q1 * q2 % p]


def test_prime_count_edges(emu):
    """For each k, the largest min(da, db) that k primes cover and one more, on primes across the whole range."""
    for p in PRIMES + (3, 5, 2**19 + 21, 2**20 + 7, 2**51 + 111, 2**52 + 21):
        Qk = 1
        for k, q in enumerate(Q, 1):
            Qk *= q
            m = (Qk - 1) // (p - 1) ** 2      # m·(p-1)² < Q_k  ⇔  m ≤ (Q_k - 1) / (p-1)²
            if m >= 1 and m < 2**64:
                assert prime_count(p, m) == k and emu.emu_crt_prime_count(p, m) == k, (p, k)
                if m + 1 < 2**64:
                    assert prime_count(p, m + 1) == k + 1 if k < 3 else prime_count(p, m + 1) == 0
                    assert emu.emu_crt_prime_count(p, m + 1) == prime_count(p, m + 1), (p, k, m)
    # the ranges each k covers at min(da, db) = 2^25
    m = MAX_LEN // 2
    for p in (17, 101, 127, 2**19 + 21):
        assert prime_count(p, m) == 1 and emu.emu_crt_prime_count(p, m) == 1
    assert prime_count(2**20 + 7, m) == 2 and prime_count(2**51 + 111, m) == 2
    assert prime_count(2**52 + 21, m) == 3 and prime_count(2**64 - 59, m) == 3
    for p in (17, 101, 127, 4295294977, 2**64 - 59):
        for m in (1, 2, 3, 1 << 12, (1 << 25) + 1, MAX_LEN):
            assert emu.emu_crt_prime_count(p, m) == prime_count(p, m), (p, m)


def test_model_matches_schoolbook():
    """Random operands at random sizes, on every test prime, with the prime count the path would choose."""
    rng = random.Random(1)
    for p in PRIMES:
        for _ in range(3):
            da, db = rng.randint(1, 40), rng.randint(1, 40)
            a = [rng.randrange(p) for _ in range(da)]
            b = [rng.randrange(p) for _ in range(db)]
            exp = [int(v) for v in oracle.poly_mul(p, np.array(a, dtype=np.uint64), np.array(b, dtype=np.uint64))]
            assert model_mul(p, a, b) == exp, (p, da, db)


@pytest.mark.parametrize("p", (101, 2**64 - 59))
def test_model_needs_every_prime(p):
    """All-(p - 1) operands make every integer coefficient reach min(da, db)·(p - 1)²: at the prime count the model is
    exact, with one prime fewer it is not.  At p = 101 and m = 40, one prime is needed and enough; 2^64 - 59 needs three."""
    m = 40
    a, b = [p - 1] * m, [p - 1] * (m + 3)
    exp = [int(v) for v in oracle.poly_mul(p, np.array(a, dtype=np.uint64), np.array(b, dtype=np.uint64))]
    k = prime_count(p, m)
    assert model_mul(p, a, b) == exp
    if k > 1:
        assert model_mul(p, a, b, k - 1) != exp


def _edges(bound):
    return [0, 1, 2, bound // 2, bound - 2, bound - 1]


@pytest.mark.parametrize("p", (101, 17, 4295294977, 2**61 - 1, 2**63 - 25, 2**63 + 29, 2**64 - 279, 2**64 - 59, GL))
def test_host_garner_on_edge_residues(emu, p):
    """crt_garner<k> compiled for the host on every combination of edge residues: 0, 1, q_i - 1, and residues ≥ q3 and
    ≥ p where they exist, against the CRT in Python integers."""
    c1v = _edges(Q[0]) + [Q[2], Q[2] + 1, 4 * Q[2] + 3] + [v for v in (p, p + 1, 2 * p - 1) if v < Q[0]]
    c2v = _edges(Q[1]) + [Q[0], Q[0] + 5, Q[2], 3 * Q[2]] + [v for v in (p, p + 1) if v < Q[1]]
    c3v = _edges(Q[2]) + [v for v in (p, p + 1) if v < Q[2]]
    combos = [(x, y, z) for x in c1v for y in c2v for z in c3v]
    rng = random.Random(p)
    combos += [(rng.randrange(Q[0]), rng.randrange(Q[1]), rng.randrange(Q[2])) for _ in range(2000)]
    c1, c2, c3 = (np.array(col, dtype=np.uint64) for col in zip(*combos))
    for k in (1, 2, 3):
        out = np.zeros(len(combos), dtype=np.uint64)
        assert emu.emu_crt_garner(p, k, _ptr(c1), _ptr(c2), _ptr(c3), _ptr(out), len(combos)) == 0
        exp = [crt(t[:k], p) for t in combos]
        bad = [i for i in range(len(combos)) if int(out[i]) != exp[i]]
        assert not bad, (p, k, combos[bad[0]], int(out[bad[0]]), exp[bad[0]])


@pytest.mark.parametrize("q", Q)
def test_host_reduction_edges(emu, q):
    """crt_below, the reduction of crt_reduce_kernel: x mod q_i for x up to 2^64 - 1 (four subtractions for q3)."""
    xs = sorted({v for v in (0, 1, q - 1, q, q + 1, 2 * q - 1, 2 * q, 3 * q + 7, 4 * q - 1, 4 * q, 2**64 - 1, 2**64 - 2)
                 if v < 2**64})
    x = np.array(xs, dtype=np.uint64)
    out = np.zeros_like(x)
    emu.emu_crt_below(q, _ptr(x), _ptr(out), len(x))
    assert [int(v) for v in out] == [v % q for v in xs]
