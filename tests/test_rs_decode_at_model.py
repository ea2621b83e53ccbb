"""CPU tier: a Python-integer model of ronk_rs_decode_at_u64 (csrc/rs.cu), the errors-and-erasures Reed–Solomon decoder
at any n distinct points, step for step: the syndromes through the interpolant (S = Ĩ·T mod z^m, T the reversed
quotient of X^(n+m-1) by M), Berlekamp–Massey seeded with the erasures in its inversion-free form, the reversed forms
σ, σ', Ω̂ with Berlekamp–Massey's length L, Chien search and Forney with M'(x_i), and the check by re-interpolation.
It is checked against brute-force nearest-codeword search at small primes (points, errors and erasures at x = 0
included, n = 1, k = n and k = 1), and word for word against the ω_n^i decoder's model at x_i = ω_n^i."""
import itertools
import random

import pytest

from test_rs_decode_model import decode as decode_omega
from test_rs_decode_model import generator


def _eval(p, c, x):
    acc = 0
    for v in reversed(c):
        acc = (acc * x + v) % p
    return acc


def _mul(p, a, b):
    out = [0] * (len(a) + len(b) - 1) if a and b else []
    for i, u in enumerate(a):
        for j, v in enumerate(b):
            out[i + j] = (out[i + j] + u * v) % p
    return out


def _from_roots(p, xs):
    out = [1]
    for x in xs:
        out = _mul(p, out, [(-x) % p, 1])
    return out


def _quotient(p, a, b):
    """quo(a, b) for a monic b, len(a) - len(b) + 1 words."""
    a = list(a)
    q = [0] * (len(a) - len(b) + 1)
    for i in range(len(q) - 1, -1, -1):
        q[i] = a[i + len(b) - 1]
        for j, v in enumerate(b):
            a[i + j] = (a[i + j] - q[i] * v) % p
    return q


def interpolate(p, xs, ys):
    """The interpolant through (xs[i], ys[i]): len(xs) coefficients."""
    n = len(xs)
    M = _from_roots(p, xs)
    out = [0] * n
    for i, x in enumerate(xs):
        q = _quotient(p, M, [(-x) % p, 1])
        c = ys[i] * pow(_eval(p, q, x), p - 2, p) % p
        for j in range(n):
            out[j] = (out[j] + c * q[j]) % p
    return out


def decode_at(p, xs, row, erased, k):
    """(message, errors), or (None, -1) when the row is not within the decoding radius of a codeword."""
    n = len(xs)
    m = n - k
    r0 = [0 if erased[i] else row[i] for i in range(n)]            # erased values are never read
    I = interpolate(p, xs, r0)
    M = _from_roots(p, xs)
    Md = [(i + 1) * M[i + 1] % p for i in range(n)]
    W = [_eval(p, Md, x) for x in xs]                              # M'(x_i)
    S = []
    if m:
        T = _quotient(p, [0] * (n + m - 1) + [1], M)[::-1]         # 1 / (z^n·M(1/z)) mod z^m
        It = [I[n - 1 - t] for t in range(m)]
        S = _mul(p, It, T)[:m]
    E = [i for i in range(n) if erased[i]]
    eps = len(E)
    if eps > m:
        return None, -1
    gam = [1] + [0] * m
    for i in E:                                                    # Γ ← Γ · (1 − x_i z)
        gam = [(gam[j] - xs[i] * (gam[j - 1] if j else 0)) % p for j in range(m + 1)]
    psi, B, L, b, s = gam[:], gam[:], eps, 1, 1
    for r in range(eps, m):
        d = sum(psi[i] * S[r - i] for i in range(r + 1)) % p
        if d == 0:
            s += 1
            continue
        full = [(b * (psi[i] if i <= m else 0) - d * (B[i - s] if s <= i <= m + s else 0)) % p for i in range(m + s + 1)]
        assert not any(full[m + 1:]), "Ψ outgrew m + 1 coefficients"
        old, psi = psi, full[:m + 1]
        if 2 * L <= r + eps:
            L, B, b, s = r + 1 + eps - L, old, d, 1
        else:
            s += 1
    if 2 * L - eps > m:
        return None, -1
    omega = [sum(psi[i] * S[j - i] for i in range(j + 1)) % p for j in range(m)]
    sigma = [psi[L - i] for i in range(L + 1)]                     # X^L·Ψ(1/X): a point at 0 is a root
    dsigma = [(i + 1) * sigma[i + 1] % p for i in range(L)]
    omh = [omega[L - 1 - i] for i in range(L)]                     # X^(L-1)·Ω(1/X)
    corrected = list(r0)
    roots = 0
    for i, x in enumerate(xs):
        if _eval(p, sigma, x):
            continue
        roots += 1
        dv = _eval(p, dsigma, x)
        if dv == 0:
            return None, -1
        corrected[i] = (corrected[i] - _eval(p, omh, x) * W[i] * pow(dv, p - 2, p)) % p
    if roots != L:
        return None, -1
    C = interpolate(p, xs, corrected)
    if any(C[k:]):
        return None, -1
    return C[:k], L - eps


def distance(p, xs, msg, row, erased):
    return sum(1 for x, y, e in zip(xs, row, erased) if not e and _eval(p, msg, x) != y)


def nearest(p, xs, row, erased, k):
    """Brute force: {message: distance} over the interpolants through every k non-erased positions, which include every
    codeword within distance n - k of the row."""
    live = [i for i in range(len(xs)) if not erased[i]]
    found = {}
    for sub in itertools.combinations(live, k):
        msg = tuple(interpolate(p, [xs[i] for i in sub], [row[i] for i in sub]))
        found[msg] = distance(p, xs, msg, row, erased)
    return found


def check_against_brute_force(p, xs, row, erased, k, got):
    """A complete bounded-distance decoder: the codeword within the radius when there is one, else (None, -1)."""
    m, eps = len(xs) - k, sum(1 for e in erased if e)
    within = {msg: d for msg, d in nearest(p, xs, row, erased, k).items() if 2 * d + eps <= m}
    assert len(within) <= 1
    if within:
        (msg, d), = within.items()
        assert got == (list(msg), d), (xs, row, erased, k, got, within)
    else:
        assert got == (None, -1), (xs, row, erased, k, got)


def _row(p, rng, xs, k, errors, erased_at):
    msg = [rng.randrange(p) for _ in range(k)]
    row = [_eval(p, msg, x) for x in xs]
    erased = [1 if i in erased_at else 0 for i in range(len(xs))]
    for i in erased_at:
        row[i] = rng.randrange(p)
    for i in errors:
        row[i] = (row[i] + 1 + rng.randrange(p - 1)) % p
    return msg, row, erased


@pytest.mark.parametrize("p", [17, 97, 101])
def test_within_the_radius_gives_the_message(p):
    """Random distinct points (0 among them in every other case), errors and erasures at 2e + ε ≤ m, x = 0 carrying an
    error or an erasure: the sent message and the error count."""
    rng = random.Random(p)
    for case in range(400):
        n = rng.randrange(1, 13)
        k = rng.choice([1, n, rng.randrange(1, n + 1)])
        m = n - k
        xs = rng.sample(range(1, p), n)
        if case % 2 and n > 1:
            xs[rng.randrange(n)] = 0
        eps = rng.randrange(m + 1)
        erased_at = set(rng.sample(range(n), eps))
        e = (m - eps) // 2 if case % 3 else rng.randrange((m - eps) // 2 + 1)
        live = [i for i in range(n) if i not in erased_at]
        msg, row, erased = _row(p, rng, xs, k, rng.sample(live, e), erased_at)
        assert decode_at(p, xs, row, erased, k) == (msg, e), (xs, row, erased, k)
    zero_cases = [({0}, set()), (set(), {0}), ({0, 3}, {5}), ({1}, {0, 4})]   # x = 0 at position 0
    for errs, ers in zero_cases:
        xs = [0] + rng.sample(range(1, p), 7)
        msg, row, erased = _row(p, rng, xs, 2, errs, ers)
        assert decode_at(p, xs, row, erased, 2) == (msg, len(errs))


@pytest.mark.parametrize("p", [17, 97, 101])
def test_agrees_with_brute_force_search(p):
    """Small rows at every distance, within the radius and beyond it, against brute-force nearest-codeword search."""
    rng = random.Random(p + 7)
    for case in range(150):
        n = rng.randrange(1, 9)
        k = rng.randrange(1, n + 1)
        xs = rng.sample(range(p), n)                         # 0 may be among them
        eps = rng.randrange(n - k + 2) if n > k else 0
        erased_at = set(rng.sample(range(n), min(eps, n)))
        live = [i for i in range(n) if i not in erased_at]
        errs = rng.sample(live, rng.randrange(len(live) + 1))
        _, row, erased = _row(p, rng, xs, k, errs, erased_at)
        if case % 5 == 0:
            row = [rng.randrange(p) for _ in range(n)]       # an arbitrary word
        check_against_brute_force(p, xs, row, erased, k, decode_at(p, xs, row, erased, k))


def test_single_point_and_full_rate():
    """n = 1 and k = n (m = 0): the interpolant, with status 0; an erasure with m = 0 is refused."""
    p = 97
    assert decode_at(p, [0], [5], [0], 1) == ([5], 0)
    assert decode_at(p, [3], [5], [1], 1) == (None, -1)
    xs, ys = [0, 4, 9], [1, 2, 3]
    assert decode_at(p, xs, ys, [0, 0, 0], 3) == (interpolate(p, xs, ys), 0)


@pytest.mark.parametrize("p", [17, 97, 193, 257])
def test_at_roots_of_unity_matches_the_omega_decoder(p):
    """At x_i = ω_n^i in order, word for word what the ω_n^i decoder's model gives, within the radius and beyond it."""
    g = generator(p)
    rng = random.Random(p + 11)
    divisors = [d for d in range(1, min(p, 40)) if (p - 1) % d == 0]
    for _ in range(250):
        n = rng.choice(divisors)
        k = rng.randrange(1, n + 1)
        m = n - k
        w = pow(g, (p - 1) // n, p)
        xs = [pow(w, i, p) for i in range(n)]
        eps = rng.randrange(m + 2) if m else 0
        erased_at = set(rng.sample(range(n), min(eps, n)))
        live = [i for i in range(n) if i not in erased_at]
        e = min(len(live), max(0, (m - eps) // 2 + rng.randrange(-1, 3)))
        _, row, erased = _row(p, rng, xs, k, rng.sample(live, e), erased_at)
        assert decode_at(p, xs, row, erased, k) == decode_omega(p, g, row, erased, k), (n, k, row, erased)
