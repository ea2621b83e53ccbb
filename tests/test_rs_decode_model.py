"""CPU tier: a Python-integer model of the errors-and-erasures Reed–Solomon decoder of csrc/rs.cu, step for step
(inverse transform, syndromes, erasure locator, Berlekamp–Massey seeded with the erasures in its inversion-free
form, the degree check, Ω, Chien search on the forward transforms, Forney, the re-encoding check), checked against
brute-force nearest-codeword search, the oracle's rs_encode and its rs_decode (Message::decode)."""
import itertools
import random

import pytest

import oracle


def _dft(p, w, a, n):
    return [sum(int(a[j]) * pow(w, i * j % n, p) for j in range(len(a))) % p for i in range(n)]


def encode(p, g, msg, n):
    """codeword[i] = m(ω_n^i)"""
    return _dft(p, pow(g, (p - 1) // n, p), msg, n)


def decode(p, g, row, erased, k):
    """(message, errors), or (None, -1) when the row is not within the decoding radius of a codeword."""
    n = len(row)
    m = n - k
    w = pow(g, (p - 1) // n, p)
    wi = pow(w, p - 2, p)
    ninv = pow(n, p - 2, p)
    Y = [v * ninv % p for v in _dft(p, wi, row, n)]
    S = Y[k:]
    E = [i for i in range(n) if erased[i]]
    eps = len(E)
    if eps > m:
        return None, -1
    gam = [1] + [0] * m
    for i in E:                                            # Γ ← Γ · (1 − ω^-i z)
        x = pow(wi, i, p)
        gam = [(gam[j] - x * (gam[j - 1] if j else 0)) % p for j in range(m + 1)]
    psi, B, L, b, s = gam[:], gam[:], eps, 1, 1
    for r in range(eps, m):
        d = sum(psi[i] * S[r - i] for i in range(r + 1)) % p
        if d == 0:
            s += 1
            continue
        full = [(b * (psi[i] if i <= m else 0) - d * (B[i - s] if s <= i <= m + s else 0)) % p for i in range(m + s + 1)]
        assert not any(full[m + 1:]), "Ψ outgrew m + 1 coefficients"
        T, psi = psi, full[:m + 1]
        if 2 * L <= r + eps:
            L, B, b, s = r + 1 + eps - L, T, d, 1
        else:
            s += 1
    deg = max(i for i in range(m + 1) if psi[i])
    if 2 * deg - eps > m:
        return None, -1
    omega = [sum(psi[i] * S[j - i] for i in range(j + 1)) % p for j in range(m)]
    dpsi = [i * psi[i] % p for i in range(1, m + 1)]
    Pv, Dv, Ov = _dft(p, w, psi, n), _dft(p, w, dpsi, n), _dft(p, w, omega, n)
    corrected = list(row)
    roots = 0
    for i in range(n):
        if Pv[i]:
            continue
        roots += 1
        if Dv[i] == 0:
            return None, -1
        e = (-n * pow(w, i * (k - 1) % n, p) * Ov[i] * pow(Dv[i], p - 2, p)) % p
        corrected[i] = (corrected[i] - e) % p
    if roots != deg:
        return None, -1
    C = [v * ninv % p for v in _dft(p, wi, corrected, n)]
    if any(C[k:]):
        return None, -1
    return C[:k], deg - eps


def generator(p):
    """The smallest generator of F_p*.  (The reference's search returns elements of lower order for some primes,
    97 and 193 among them, and then ω_n has order below n.)"""
    q = [d for d in range(2, p) if (p - 1) % d == 0 and all(d % r for r in range(2, d))]
    return next(a for a in range(2, p) if all(pow(a, (p - 1) // r, p) != 1 for r in q))


def distance(a, b, erased):
    return sum(1 for x, y, e in zip(a, b, erased) if not e and x != y)


def nearest(p, g, row, erased, k):
    """Brute force: every codeword within distance n - k of the row agrees with it on k non-erased positions, so it is
    the interpolant through some k of them.  Returns {message: distance} over all k-subsets."""
    n = len(row)
    w = pow(g, (p - 1) // n, p)
    live = [i for i in range(n) if not erased[i]]
    found = {}
    for sub in itertools.combinations(live, k):
        xs = [pow(w, i, p) for i in sub]
        msg = tuple(int(v) for v in oracle.rs_decode(p, xs, [row[i] for i in sub], k))
        found[msg] = distance(encode(p, g, msg, n), row, erased)
    return found


def check_bounded(p, g, row, erased, k, got):
    """The decoder's promise: −1, or a message whose codeword lies within the radius of the row."""
    msg, st = got
    m, eps = len(row) - k, sum(1 for e in erased if e)
    if msg is None:
        assert st == -1
        return
    assert 2 * st + eps <= m
    assert distance(encode(p, g, msg, len(row)), row, erased) == st


TINY = [(17, 8, 2), (17, 8, 4), (17, 4, 1), (127, 7, 3), (127, 7, 5)]


@pytest.mark.parametrize("p,n,k", TINY, ids=[f"p{p}-n{n}-k{k}" for p, n, k in TINY])
def test_every_pattern_to_the_radius_matches_brute_force(p, n, k):
    """Every error pattern up to the radius on one codeword (for p = 127, n = 7, k = 3: every single error and a
    seeded sample of double errors), with no erasures and with erasure sets of every size ≤ n - k, against brute-force
    search; and a sample of words one error beyond the radius keeps the bounded-distance promise."""
    g = generator(p)
    m = n - k
    rng = random.Random(p * 1000 + n * 10 + k)
    msg = [rng.randrange(p) for _ in range(k)]
    cw = encode(p, g, msg, n)
    for eps in range(m + 1):
        for er_set in list(itertools.combinations(range(n), eps))[:3]:
            erased = [1 if i in er_set else 0 for i in range(n)]
            radius = (m - eps) // 2
            live = [i for i in range(n) if not erased[i]]
            base = [(v + 1 + rng.randrange(p - 1)) % p if erased[i] else v for i, v in enumerate(cw)]
            for e in range(radius + 1):
                patterns = [(pos, vals) for pos in itertools.combinations(live, e)
                            for vals in itertools.product(range(1, p), repeat=e)]
                if len(patterns) > 1500:
                    patterns = rng.sample(patterns, 1500)
                for pos, vals in patterns:
                    row = list(base)
                    for i, v in zip(pos, vals):
                        row[i] = (row[i] + v) % p
                    assert decode(p, g, row, erased, k) == (msg, e), (eps, pos, vals)
                    if e == radius and len(patterns) <= 200:
                        best = nearest(p, g, row, erased, k)
                        assert best[tuple(msg)] == e, (pos, vals)
                        assert all(d > e for mm, d in best.items() if mm != tuple(msg)), (pos, vals)
            for _ in range(60):
                e = min(radius + 1 + rng.randrange(2), len(live))
                row = list(base)
                for i in rng.sample(live, e):
                    row[i] = (row[i] + 1 + rng.randrange(p - 1)) % p
                got = decode(p, g, row, erased, k)
                check_bounded(p, g, row, erased, k, got)
                if got[0] is not None:
                    assert nearest(p, g, row, erased, k)[tuple(got[0])] == got[1]


@pytest.mark.parametrize("p", [17, 101, 127, 193, 257])
def test_encode_matches_the_oracle(p):
    g = generator(p)
    rng = random.Random(p)
    for n in [d for d in range(1, p) if (p - 1) % d == 0][:8]:
        k = rng.randrange(1, n + 1)
        msg = [rng.randrange(p) for _ in range(k)]
        xs, ys = oracle.rs_encode(p, msg, n, g)
        assert [int(v) for v in ys] == encode(p, g, msg, n)
        assert [int(v) for v in xs] == [pow(g, (p - 1) // n * i, p) for i in range(n)]


@pytest.mark.parametrize("p", [17, 101, 127, 193, 257])
def test_tail_erased_is_message_decode(p):
    """Any row with positions k..n-1 erased decodes, with no error, to Message::decode of its first k coordinates."""
    g = generator(p)
    rng = random.Random(p + 1)
    for n in [d for d in range(2, p) if (p - 1) % d == 0][:10]:
        for k in sorted({1, n // 2 or 1, n} & set(range(21))):   # the oracle's combination formula stops at k = 20
            row = [rng.randrange(p) for _ in range(n)]
            erased = [0] * k + [1] * (n - k)
            xs = [pow(g, (p - 1) // n * i, p) for i in range(n)]
            want = [int(v) for v in oracle.rs_decode(p, xs, row, k)]
            assert decode(p, g, row, erased, k) == (want, 0), (n, k)


@pytest.mark.parametrize("p", [97, 127, 193, 257])
def test_random_codes_and_words_beyond_the_radius(p):
    """Random n | p - 1, k, erasures and errors: exact at the radius; random words keep the bounded-distance promise."""
    g = generator(p)
    rng = random.Random(p + 2)
    divisors = [d for d in range(2, p) if (p - 1) % d == 0]
    for _ in range(60):
        n = rng.choice(divisors)
        k = rng.randrange(1, n + 1)
        m = n - k
        msg = [rng.randrange(p) for _ in range(k)]
        cw = encode(p, g, msg, n)
        eps = rng.randrange(m + 1)
        er = set(rng.sample(range(n), eps))
        erased = [1 if i in er else 0 for i in range(n)]
        e = (m - eps) // 2
        row = [rng.randrange(p) if erased[i] else v for i, v in enumerate(cw)]
        for i in rng.sample([i for i in range(n) if not erased[i]], e):
            row[i] = (row[i] + 1 + rng.randrange(p - 1)) % p
        assert decode(p, g, row, erased, k) == (msg, e), (n, k, eps, e)
        junk = [rng.randrange(p) for _ in range(n)]
        check_bounded(p, g, junk, erased, k, decode(p, g, junk, erased, k))


def test_edges_m1_and_k_equal_n():
    p, g = 127, 3
    rng = random.Random(5)
    for n in (2, 3, 6, 7, 9, 14):
        k = n - 1                                  # m = 1: radius 0 without erasures, one erasure is corrected
        msg = [rng.randrange(p) for _ in range(k)]
        cw = encode(p, g, msg, n)
        assert decode(p, g, cw, [0] * n, k) == (msg, 0)
        for i in range(n):
            row = list(cw)
            row[i] = (row[i] + 1 + rng.randrange(p - 1)) % p
            assert decode(p, g, row, [0] * n, k) == (None, -1), (n, i)
            assert decode(p, g, row, [int(j == i) for j in range(n)], k) == (msg, 0), (n, i)
        row = [rng.randrange(p) for _ in range(n)]   # k = n: every word is a codeword; any erasure fails
        assert decode(p, g, row, [0] * n, n) == (encode_inverse(p, g, row), 0)
        assert decode(p, g, row, [1] + [0] * (n - 1), n) == (None, -1)
    assert decode(p, g, [5], [0], 1) == ([5], 0)


def encode_inverse(p, g, row):
    n = len(row)
    wi = pow(pow(g, (p - 1) // n, p), p - 2, p)
    ninv = pow(n, p - 2, p)
    return [v * ninv % p for v in _dft(p, wi, row, n)]
