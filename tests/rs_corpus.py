"""Structured received words for the Reed–Solomon decoder of ronkathon_b200/csrc/rs.cu, with what the decoder must
answer known by construction, so that no reference decoder is needed at the sizes the device runs.  Shared by the CPU
model tests (tests/test_rs_locator_model.py) and the device tests (tests/test_gpu_rs_decode_structured.py).
Importable without a GPU.

Random errors at the full radius, which is what the rest of the suite decodes, give Berlekamp–Massey a nonzero
discrepancy at every step and a length that grows by one every other step.  The rows here are built to leave that
path: few errors under a large parity budget (long runs of zero discrepancies after the locator is found), errors on
a coset of a subgroup (locator 1 - c·z^e: the syndromes vanish except every e-th, and the length jumps by e at once),
and syndrome sequences prescribed outright.

A row is described in the transform domain: row = forward transform of Y, plus errata.  Since the decoder's Y is the
scaled inverse transform of the row and its syndromes are S_j = Y[k + j], Y[0..k) is a message when Y[k..n) = 0, and
any syndrome sequence can be prescribed by writing it into Y[k..n).  `build` turns specs into rows with a forward
transform the caller supplies (the device encoder with k = n, or `forward_py`); `syndromes` gives a spec's syndromes
in O(errata · m) without any transform."""
from typing import NamedTuple, Optional

import numpy as np

ZERO = "zero"                     # an erratum that turns the received symbol into 0 (into 1 where it is 0 already)
FLAGS = (1, 2, 0x80, 0xFF)        # `erased` marks a position with any nonzero byte


class Code(NamedTuple):
    p: int
    g: int
    n: int
    k: int

    @property
    def m(self):
        return self.n - self.k

    @property
    def w(self):
        return pow(self.g, (self.p - 1) // self.n, self.p)

    @property
    def winv(self):
        return pow(self.w, self.p - 2, self.p)


class Expect(NamedTuple):
    """status -1: the row must be refused (zero message).  status ≥ 0: exactly that many errors; msg, when known, is
    the message.  status None: the row may decode or not, and must keep the bounded-distance promise either way."""
    status: Optional[int]
    msg: Optional[np.ndarray] = None


class Spec(NamedTuple):
    name: str
    base: np.ndarray              # Y, n words
    errata: dict                  # position → value added to the row there (an int, or ZERO)
    erased: dict                  # position → flag byte
    expect: Expect


def _rand(code, rng, count):
    return rng.integers(0, code.p, count, dtype=np.uint64)


def _nonzero(code, rng):
    return 1 + int(rng.integers(0, code.p - 1, dtype=np.uint64))


def _message(code, rng):
    base = np.zeros(code.n, dtype=np.uint64)
    base[:code.k] = _rand(code, rng, code.k)
    return base


def _erase(code, rng, eps, keep_off=()):
    """ε erased positions outside keep_off, flagged with every byte of FLAGS in turn, each holding a random value
    (so about one in p of them is correct, which an erased position may be)."""
    free = np.setdiff1d(np.arange(code.n), np.fromiter(keep_off, dtype=np.int64, count=len(keep_off)))
    pos = [int(i) for i in rng.choice(free, eps, replace=False)]
    return ({i: FLAGS[j % len(FLAGS)] for j, i in enumerate(pos)},
            {i: int(rng.integers(0, code.p, dtype=np.uint64)) for i in pos})


def erasure_counts(m):
    """ε ∈ {0, 1, m/3, m - 2}, those that fit: m - ε of both parities, a radius shared between errors and erasures, and
    a radius of one error under a long erasure locator"""
    return sorted({e for e in (0, 1, m // 3, m - 2) if 0 <= e <= m})


def error_counts(radius):
    """e ∈ {1, 2, 3, ⌊r/2⌋, r - 1} within the radius r"""
    return sorted({e for e in (1, 2, 3, radius // 2, radius - 1) if 1 <= e <= radius})


def _divisors(n, most):
    return [d for d in range(1, most + 1) if n % d == 0]


def genuine(code, rng):
    """Codewords with e errors within the radius r = ⌊(m - ε)/2⌋, e < r almost everywhere: the decoder must return
    the message and e.  Per (ε, e): random positions and values; positions 0 and n - 1 among them, value p - 1; a
    burst of e consecutive positions, value 1; random positions whose received symbol becomes 0.  Per ε: errors on
    cosets i₀ + j·n/e of the subgroups of order e | n, with equal values (error locator 1 - c·z^e) and random ones."""
    p, n, m = code.p, code.n, code.m
    out = []

    def add(name, eps, positions, values):
        base = _message(code, rng)
        flags, fill = _erase(code, rng, eps, positions)
        errata = dict(fill)
        errata.update({int(i): v for i, v in zip(positions, values)})
        out.append(Spec(f"{name}-eps{eps}-e{len(positions)}", base, errata, flags, Expect(len(positions), base[:code.k].copy())))

    for eps in erasure_counts(m):
        if n - eps < 1:
            continue
        radius = min((m - eps) // 2, n - eps)
        for e in error_counts(radius):
            add("random", eps, [int(i) for i in rng.choice(n, e, replace=False)], [_nonzero(code, rng) for _ in range(e)])
            ends = ([0, n - 1] + [int(i) for i in rng.choice(np.arange(1, n - 1), max(e - 2, 0), replace=False)])[:e]
            add("ends", eps, ends, [p - 1] * len(ends))
            start = int(rng.integers(0, n - e + 1))
            add("burst", eps, list(range(start, start + e)), [1] * e)
            add("tozero", eps, [int(i) for i in rng.choice(n, e, replace=False)], [ZERO] * e)
        divs = [d for d in _divisors(n, radius) if d > 1]
        for e in sorted(set(divs[-1:] + divs[len(divs) // 2:len(divs) // 2 + 1])):
            first = int(rng.integers(0, n // e))
            coset = [first + j * (n // e) for j in range(e)]
            v = _nonzero(code, rng)
            add("coset_equal", eps, coset, [v] * e)
            add("coset_random", eps, coset, [_nonzero(code, rng) for _ in range(e)])
    return out


def beyond_on_a_coset(code, rng):
    """e equal errors on a coset of the subgroup of order e | n, m/2 < e ≤ m, no erasures (the smallest and the largest
    such e): beyond the radius, with at most two nonzero syndromes in the window.  When the first of them is S_(e-1)
    Berlekamp–Massey finds the true locator 1 - c·z^e, all its roots are positions and Forney's values are the true
    errors, so every later check would pass and only the degree check 2·deg Ψ ≤ m refuses the row.  The row must be
    refused when e ≤ m - r: its codeword is e > r away, and every other one at least m + 1 - e > r."""
    n, m = code.n, code.m
    out = []
    divs = [d for d in _divisors(n, m) if 2 * d > m]
    for e in sorted(set(divs[:1] + divs[-1:])):
        first = int(rng.integers(0, n // e))
        v = _nonzero(code, rng)
        out.append(Spec(f"beyond_coset-e{e}", _message(code, rng), {first + j * (n // e): v for j in range(e)}, {},
                        Expect(-1 if e <= m - m // 2 else None)))
    return out


def _with_syndromes(code, rng, S):
    base = _rand(code, rng, code.n)
    base[code.k:] = np.array([int(v) % code.p for v in S], dtype=np.uint64)
    return base


def _power_sums(code, terms, m, linear=()):
    """S_j = Σ c·x^j over terms (x, c), plus Σ c·j·x^j over `linear`: the general solution of the recurrence whose
    connection polynomial is Π (1 - x z), with (1 - x z)² for the x of `linear`."""
    p = code.p
    S = [0] * m
    for lin, group in ((False, terms), (True, linear)):
        for x, c in group:
            cur = c % p
            for j in range(m):
                S[j] = (S[j] + (cur * j if lin else cur)) % p
                cur = cur * x % p
    return S


def deltas(code, rng):
    """S = c·δ_t, t ∈ {0, 1, ⌊m/2⌋ - 1, ⌊m/2⌋, m - 1}, without erasures and with a few.

    Without erasures every one must be refused (an errata pattern with this syndrome window has at least
    max(t + 1, m - t) > m/2 terms), and which check refuses it depends on t.  For t ≥ m/2 the length jumps to t + 1 and
    the degree check fires.  For t < m/2 it jumps to t + 1 as well, but the update at step 2t + 1 cancels the z^(t+1)
    term again: Ψ ends as a nonzero *constant*, which passes the degree check, has no roots and degree 0, so passes
    the root count too; only the re-encoding check C[k..n) = 0 refuses the row (tests/test_rs_locator_model.py
    shows that with the model).  With ε erasures the row must be refused when 2·max(t + 1, m - t) > m + ε; otherwise it
    may decode, within the radius."""
    n, m = code.n, code.m
    out = []
    for t in sorted({t for t in (0, 1, m // 2 - 1, m // 2, m - 1) if 0 <= t < m}):
        for eps in sorted({0, min(3, m - 1), m // 2}):
            if eps < 0 or eps > n:
                continue
            S = [0] * m
            S[t] = _nonzero(code, rng)
            flags, _ = _erase(code, rng, eps)
            refused = 2 * max(t + 1, m - t) > m + eps
            out.append(Spec(f"delta-t{t}-eps{eps}", _with_syndromes(code, rng, S), {}, flags, Expect(-1 if refused else None)))
    return out


def recurrences(code, rng, longest=24):
    """Syndromes generated by a chosen connection polynomial Ψ of degree L, 2L ≤ m + ε (so Berlekamp–Massey finds
    exactly Ψ), for L ∈ {1, 3, up to `longest`} and ε ∈ {0, 2} of its roots erased:
      genuine: Ψ = Π (1 - x z) over L distinct positions' x = ω^-i, every coefficient nonzero: an L-errata pattern on
        some codeword whose message is not Y[0..k) (the errata's spectrum runs on into 0..k-1), so the row decodes
        with exactly L - ε errors, to a message that re-encodes to the row at all but those positions;
      double: the same with one factor squared: a root where Ψ' vanishes, and fewer roots than the degree;
      offdomain: one x replaced by an element that is no n-th root of unity: deg Ψ - 1 roots among the positions."""
    p, n, m = code.p, code.n, code.m
    out = []
    off = next((x for x in (code.g, 2, 3, 5) if pow(x, n, p) != 1), None)
    for eps in (0, 2):
        for L in sorted({L for L in (1, 3, min((m + eps) // 2, longest)) if eps <= L and 2 * L <= m + eps and L <= n}):
            pos = [int(i) for i in rng.choice(n, L, replace=False)]
            xs = [pow(code.winv, i, p) for i in pos]
            cs = [_nonzero(code, rng) for _ in range(L)]
            flags = {i: FLAGS[j % len(FLAGS)] for j, i in enumerate(pos[:eps])}
            S = _power_sums(code, list(zip(xs, cs)), m)
            out.append(Spec(f"recur_genuine-L{L}-eps{eps}", _with_syndromes(code, rng, S), {}, flags, Expect(L - eps)))
            if 2 * (L + 1) <= m + eps and L > eps:
                S = _power_sums(code, list(zip(xs, cs)), m, linear=[(xs[-1], _nonzero(code, rng))])
                out.append(Spec(f"recur_double-L{L + 1}-eps{eps}", _with_syndromes(code, rng, S), {}, flags, Expect(-1)))
            if off is not None and L > eps:
                S = _power_sums(code, list(zip(xs[:-1] + [off], cs)), m)
                out.append(Spec(f"recur_offdomain-L{L}-eps{eps}", _with_syndromes(code, rng, S), {}, flags, Expect(-1)))
    return out


def too_many_erasures(code, rng):
    """ε = m + 1 on a clean codeword: refused before any syndrome is read."""
    if code.m + 1 > code.n:
        return []
    flags, _ = _erase(code, rng, code.m + 1)
    return [Spec("erasures-m+1", _message(code, rng), {}, flags, Expect(-1))]


def everything(code, rng, longest=24):
    return (genuine(code, rng) + beyond_on_a_coset(code, rng) + deltas(code, rng) + recurrences(code, rng, longest)
            + too_many_erasures(code, rng))


def mixed(code, rng, rows=300, longest=24):
    """At least `rows` specs of every kind, rows that must be refused placed between rows that decode."""
    specs = []
    while len(specs) < rows:
        specs += everything(code, rng, longest)
    bad = [s for s in specs if s.expect.status == -1]
    good = [s for s in specs if s.expect.status != -1]
    out = []
    stride = max(len(good) // max(len(bad), 1), 1)
    for i, s in enumerate(good):                       # a refused row after every stride-th decoding row
        out.append(s)
        if i % stride == 0 and bad:
            out.append(bad.pop())
    return out + bad


def forward_py(code):
    """The forward transform of each row of Y in Python integers, O(n²) per row."""
    p, n = code.p, code.n
    pw = [1] * n
    for i in range(1, n):
        pw[i] = pw[i - 1] * code.w % p

    def forward(Y):
        out = np.empty(Y.shape, dtype=np.uint64)
        for r, y in enumerate(Y):
            nz = [(j, int(v)) for j, v in enumerate(y) if v]
            out[r] = [sum(v * pw[i * j % n] for j, v in nz) % p for i in range(n)]
        return out
    return forward


def _value_at(code, base, i):
    x = pow(code.w, i, code.p)
    acc = 0
    for v in base[::-1]:
        acc = (acc * x + int(v)) % code.p
    return acc


def _erratum(code, v, symbol):
    if v is not ZERO:
        return v
    return (-symbol) % code.p if symbol else 1


def build(code, specs, forward):
    """(rows, erased, k, [Expect]) for the specs; forward(Y) transforms every row of a (batch, n) uint64 array."""
    p = code.p
    rows = np.array(forward(np.stack([s.base for s in specs])), dtype=np.uint64)
    erased = np.zeros(rows.shape, dtype=np.uint8)
    for r, s in enumerate(specs):
        for i, v in s.errata.items():
            rows[r, i] = (int(rows[r, i]) + _erratum(code, v, int(rows[r, i]))) % p
        for i, flag in s.erased.items():
            erased[r, i] = flag
    return rows, erased, code.k, [s.expect for s in specs]


def syndromes(code, spec):
    """S_j = Y[k + j] of the spec's row, without a transform: Y[t] = base[t] + n^-1 · Σ errata_i · ω^(-i·t)."""
    p, n, k, m = code.p, code.n, code.k, code.m
    S = [int(v) for v in spec.base[k:]]
    ninv = pow(n, p - 2, p)
    for i, v in spec.errata.items():
        if v is ZERO:
            v = _erratum(code, v, _value_at(code, spec.base, i))
        x = pow(code.winv, i, p)
        cur = v * ninv * pow(x, k, p) % p
        for j in range(m):
            S[j] = (S[j] + cur) % p
            cur = cur * x % p
    return S
