"""CPU tier: the locator kernel's bookkeeping, and the structured rows of tests/rs_corpus.py.

`mirror` restates rs_locator_kernel of csrc/rs.cu in Python integers *with* what the plain model
(tests/test_rs_decode_model.py) leaves out: the double-buffered erasure product, the degree bounds hi and hb, the
bound nh up to which a step updates Ψ, the `i <= r && i <= hi` limit of the discrepancy sum, the new B written in
full, and the coefficients a block of T threads owns.  It must agree with the plain algorithm after every step, on
rows that reach every branch of that bookkeeping; the tests below assert that the corpus does reach them, so a slip in
the kernel's copy of the same lines is met by tests/test_gpu_rs_decode_structured.py on the same rows."""
import functools
import itertools
import random
from unittest import mock

import numpy as np
import pytest

import oracle
import rs_corpus as rc
import test_rs_decode_model as model
from test_rs_decode_model import TINY, check_bounded, generator, nearest

GL = oracle.GOLDILOCKS
PER, MAX_THREADS = 8, 1024        # RS_LOC_PER, RS_LOC_MAX_THREADS


def threads_for(m):
    """The block rs_decode_device launches for m parity symbols."""
    return min(MAX_THREADS, max(32, ((m + 1 + PER - 1) // PER + 31) // 32 * 32))


def mirror(p, S, xs, m, T, plain=None, events=None):
    """(Ψ, deg Ψ, fail) as rs_locator_kernel computes them from the syndromes S and the erasures' ω^-i (xs), with T
    threads.  Thread t owns the coefficients t + j·T, j < PER, so the block owns exactly 0..PER·T-1 and the loops
    below run over that range.  plain: the plain model's steps, compared after every step; events: a set that
    receives the name of every branch taken."""
    events = set() if events is None else events
    eps, owned = len(xs), PER * T
    assert m < owned, "a coefficient of Ψ that no thread owns"
    B = [[0] * (m + 1), [0] * (m + 1)]
    B[0][0] = 1 % p
    fail = eps > m
    cur = 0
    if not fail:
        for l, x in enumerate(xs):
            src, dst = B[l & 1], B[(l & 1) ^ 1]
            for i in range(m + 1):
                dst[i] = (src[i] - x * src[i - 1]) % p if i else src[0]
        cur = eps & 1
    psi = [B[cur][i] if not fail and i <= m else 0 for i in range(owned)]
    if not fail:
        last = max((j for j in range(m) if S[j]), default=-1)
        L, bb, s, hi, hb = eps, 1 % p, 1, eps, eps
        for r in range(eps, m):
            d = sum(psi[i] * S[r - i] for i in range(owned) if i <= r and i <= hi) % p
            if d == 0:
                s += 1
                if r < last:
                    events.add("zero discrepancy before the last nonzero syndrome")
            else:
                Bc = B[cur]
                grow = 2 * L <= r + eps
                # s + hb = r + 1 + ε - L ≤ m - (L - ε) ≤ m: see test_the_clip_at_m_is_never_taken
                assert s + hb <= m, "nh is clipped at m"
                if s + hb < hi:
                    events.add("s + hb < hi")
                nh = hi if s + hb < hi else min(s + hb, m)
                for i in range(owned):
                    if i <= m:
                        old = psi[i]
                        if i <= nh:
                            psi[i] = (bb * old - (d * Bc[i - s] if i >= s else 0)) % p
                        if grow:
                            B[cur ^ 1][i] = old
                if grow:
                    hb = hi
                hi = nh
                if grow:
                    if r + 1 + eps - L > L + 1:
                        events.add("the length jumps by more than one")
                    cur ^= 1
                    L, bb, s = r + 1 + eps - L, d, 1
                else:
                    if s >= 3:
                        events.add("update without growth at s >= 3")
                    s += 1
            if plain is not None:
                pr, pd, ppsi, pL, ps = plain[r - eps]
                assert (pr, pd, pL, ps) == (r, d, L, s) and ppsi == psi[:m + 1], f"step {r}"
            assert not any(psi[m + 1:])
    deg = max((i for i in range(m + 1) if psi[i]), default=0)
    fail = fail or 2 * deg > m + eps
    return ([0] * (m + 1) if fail else psi[:m + 1]), deg, fail


def _dft_table(p, w, a, n):
    """The words of the model's _dft, which raises ω to a power for every term, from a table of the powers."""
    pw = [1] * n
    for i in range(1, n):
        pw[i] = pw[i - 1] * w % p
    nz = [(j, int(v)) for j, v in enumerate(a) if v]
    return [sum(v * pw[i * j % n] for j, v in nz) % p for i in range(n)]


def decode(p, g, row, erased, k):
    """The model's decode, several times faster at n in the hundreds."""
    with mock.patch.object(model, "_dft", _dft_table):
        return model.decode(p, g, row, erased, k)


def test_the_table_transform_is_the_models():
    rng = random.Random(7)
    for p, n in ((97, 96), (257, 64), (GL, 51), (GL, 1)):
        w = pow(generator(p) if p != GL else 7, (p - 1) // n, p)
        for length in (n, n // 3 + 1):
            a = [rng.randrange(p) * rng.randrange(2) for _ in range(length)]
            assert _dft_table(p, w, a, n) == model._dft(p, w, a, n)


def plain_steps(p, S, xs, m, steps=None):
    """Berlekamp–Massey seeded with the erasure locator, inversion-free, as the model's decode runs it and with nothing
    else: every step touches all m + 1 coefficients.  Returns Ψ; steps, when a list, receives (r, d, Ψ after the step,
    L, s) for every r."""
    eps = len(xs)
    gam = [1 % p] + [0] * m
    for x in xs:
        gam = [(gam[j] - x * (gam[j - 1] if j else 0)) % p for j in range(m + 1)]
    psi, B, L, b, s = gam[:], gam[:], eps, 1, 1
    for r in range(eps, m):
        d = sum(psi[i] * S[r - i] for i in range(r + 1)) % p
        if d:
            full = [(b * (psi[i] if i <= m else 0) - d * (B[i - s] if s <= i <= m + s else 0)) % p for i in range(m + s + 1)]
            assert not any(full[m + 1:]), "Ψ outgrew m + 1 coefficients"
            T, psi = psi, full[:m + 1]
        if d and 2 * L <= r + eps:
            L, B, b, s = r + 1 + eps - L, T, d, 1
        else:
            s += 1
        if steps is not None:
            steps.append((r, d, psi[:], L, s))
    return psi


def plain_locator(p, S, xs, m, steps):
    eps = len(xs)
    if eps > m:
        return [0] * (m + 1), 0, True
    psi = plain_steps(p, S, xs, m, steps)
    deg = max((i for i in range(m + 1) if psi[i]), default=0)
    fail = 2 * deg > m + eps
    return ([0] * (m + 1) if fail else psi), deg, fail


def _syndromes_of(code, row):
    p, n = code.p, code.n
    ninv = pow(n, p - 2, p)
    return [v * ninv % p for v in _dft_table(p, code.winv, row, n)[code.k:]]


def refused_by(code, row, erased):
    """The first of the decoder's checks, in its order, that refuses the row, or None when it decodes: the erasure
    count, the degree of Ψ, a root of Ψ where Ψ' vanishes, the number of roots among the positions, and, when all of
    those pass and the model still refuses the row, the re-encoding check C[k..n) = 0."""
    p, n, m = code.p, code.n, code.m
    E = [i for i in range(n) if erased[i]]
    got = decode(p, code.g, row, erased, code.k)
    why = None
    if len(E) > m:
        why = "erasures"
    else:
        psi = plain_steps(p, _syndromes_of(code, row), [pow(code.winv, i, p) for i in E], m)
        deg = max(i for i in range(m + 1) if psi[i])
        values = _dft_table(p, code.w, psi, n)
        slopes = _dft_table(p, code.w, [i * psi[i] % p for i in range(1, m + 1)], n)
        roots = [i for i in range(n) if values[i] == 0]
        if 2 * deg > m + len(E):
            why = "degree"
        elif any(slopes[i] == 0 for i in roots):
            why = "derivative"
        elif len(roots) != deg:
            why = "roots"
        elif got[0] is None:
            why = "reencode"
    assert (why is None) == (got[0] is not None), why
    return got, why


def compare(p, S, xs, m, events=None, T=None):
    steps = []
    want = plain_locator(p, S, xs, m, steps)
    assert mirror(p, S, xs, m, T or threads_for(m), steps, events) == want
    return want


def compare_spec(code, spec, events=None):
    xs = [pow(code.winv, i, code.p) for i in sorted(spec.erased)]
    return compare(code.p, rc.syndromes(code, spec), xs, code.m, events)


# ---- the mirror against the plain algorithm ----------------------------------------------------------------------------
PARITIES = [0, 1, 30, 31, 32, 254, 255, 256]     # m + 1 on both sides of 32 and 256: blocks of 32 and 64 threads, 8·T = m + 1
CODES = [(97, 32), (97, 96), (193, 64), (193, 192), (257, 128), (257, 256), (65537, 512), (GL, 255), (GL, 384), (GL, 512)]
CELLS = [(p, n, m) for p, n in CODES for m in PARITIES if m < n and (m < 64 or (p, n) in ((257, 256), (65537, 512), (GL, 384)))]


@functools.lru_cache(maxsize=None)
def corpus_events(p, n, m):
    """Every spec of the corpus for this code through both locators; the branches the mirror took."""
    code = rc.Code(p, generator(p) if p != GL else 7, n, n - m)
    rng = np.random.default_rng([p % (1 << 32), n, m])
    specs = rc.everything(code, rng)
    if m > 64:
        specs = specs[::3] + [s for s in specs if s.expect.status is None or s.expect.status < 0]
    events = set()
    for spec in specs:
        compare_spec(code, spec, events)
    return frozenset(events), len(specs)


@pytest.mark.parametrize("p,n,m", CELLS, ids=[f"p{p}-n{n}-m{m}" for p, n, m in CELLS])
def test_mirror_equals_the_plain_locator_on_the_corpus(p, n, m):
    _, count = corpus_events(p, n, m)
    assert count > 0


def test_thread_ownership_at_the_block_edges():
    """m + 1 = 8·T exactly, one less and one more, for every block size up to the cap: every coefficient is owned."""
    for T in range(32, MAX_THREADS + 1, 32):
        for m in (PER * T - 2, PER * T - 1, PER * T):
            if m <= PER * MAX_THREADS - 1:
                assert m < PER * threads_for(m) and threads_for(m) in (T, T + 32)
    p, rng = 257, random.Random(1)
    for m in (255, 256):                                 # 8·32 = m + 1 and the first size with 64 threads
        S = [rng.randrange(p) for _ in range(m)]
        xs = [pow(3, i, p) for i in rng.sample(range(256), 5)]
        compare(p, S, xs, m)
        with pytest.raises(AssertionError):
            mirror(p, S, xs, 256, 32)


def test_mirror_equals_the_plain_locator_on_random_cells():
    """Seeded random (n, k, ε, e): e random errors, up to two beyond the radius, and random junk."""
    done = 0
    for p in (97, 193, 257):
        g = generator(p)
        rng = np.random.default_rng(p)
        divisors = [d for d in range(2, p) if (p - 1) % d == 0]
        for _ in range(1000):
            n = int(rng.choice(divisors))
            code = rc.Code(p, g, n, int(rng.integers(1, n + 1)))
            m = code.m
            eps = int(rng.integers(0, m + 1))
            e = min(int(rng.integers(0, (m - eps) // 2 + 3)), n - eps)
            pos = rng.permutation(n)
            errata = {int(i): int(rng.integers(0, p)) for i in pos[:eps]}
            errata.update({int(i): int(rng.integers(1, p)) for i in pos[eps:eps + e]})
            base = rng.integers(0, p, n, dtype=np.uint64)
            if rng.integers(0, 4):
                base[code.k:] = 0
            compare_spec(code, rc.Spec("random", base, errata, {int(i): 1 for i in pos[:eps]}, rc.Expect(None)))
            done += 1
    assert done == 3000


def test_the_clip_at_m_is_never_taken():
    """nh = min(s + hb, m): hi and hb equal the lengths L of Ψ and of B (induction over the steps: both start at ε, and a
    step sets hi = max(hi, s + hb) = max(L, r + 1 + ε - L), the new L), so s + hb = r + 1 + ε - L ≤ m - (L - ε) ≤ m and
    the clip never changes nh.  The mirror asserts s + hb ≤ m at every update; here it runs over every syndrome
    sequence over F_5 of every length m ≤ 6 with every number of erasures, besides all the other rows of this file."""
    p = 5
    for m in range(1, 7):
        for eps in range(0, min(m, 4) + 1):
            for S in itertools.product(range(p), repeat=m):
                compare(p, list(S), list(range(1, eps + 1)), m)


# ---- what the corpus reaches -------------------------------------------------------------------------------------------
SMALL = [(97, 32, 16), (97, 48, 21), (97, 96, 33), (193, 64, 32), (257, 256, 31)]
BRANCHES = ["zero discrepancy before the last nonzero syndrome", "update without growth at s >= 3",
            "the length jumps by more than one", "s + hb < hi"]


def test_the_corpus_reaches_every_branch_of_the_bookkeeping():
    for p, n, m in SMALL:
        events, _ = corpus_events(p, n, m)
        assert sorted(events) == sorted(BRANCHES), (p, n, m, sorted(set(BRANCHES) - events))


@functools.lru_cache(maxsize=None)
def model_words(p, n, m):
    """The corpus for this code through the whole model: [(spec, row, erased, (message, status), the check that refused it)]"""
    code = rc.Code(p, generator(p), n, n - m)
    specs = rc.everything(code, np.random.default_rng([p, n, m, 1]))
    rows, erased, k, _ = rc.build(code, specs, rc.forward_py(code))
    out = []
    for spec, row, er in zip(specs, rows, erased):
        got, why = refused_by(code, [int(v) for v in row], list(er))
        out.append((spec, [int(v) for v in row], list(er), got, why))
    return code, out


@pytest.mark.parametrize("p,n,m", SMALL, ids=[f"p{p}-n{n}-m{m}" for p, n, m in SMALL])
def test_the_model_gives_every_row_its_expectation(p, n, m):
    code, words = model_words(p, n, m)
    for spec, row, er, (msg, st), why in words:
        want = spec.expect
        assert rc.syndromes(code, spec) == _syndromes_of(code, row), spec.name
        if want.status is not None:
            assert st == want.status, (spec.name, st, why)
        if want.msg is not None:
            assert msg == [int(v) for v in want.msg], spec.name
        check_bounded(p, code.g, row, er, code.k, (msg, st))
        assert (why is None) == (st >= 0)


def test_every_check_is_the_one_that_refuses_some_row():
    """Each of the decoder's checks is the one a corpus row is refused by, having passed all the checks before it;
    the rows refused by the last one, the re-encoding check, passed every other check there is."""
    seen = {}
    for p, n, m in SMALL:
        code, words = model_words(p, n, m)
        for spec, row, er, got, why in words:
            seen.setdefault(why, []).append(spec.name)
            if spec.name.startswith("delta") and spec.name.endswith("eps0"):
                t = int(spec.name.split("-")[1][1:])
                assert why == ("reencode" if 2 * (t + 1) <= m else "degree"), (spec.name, why)
                if why == "reencode":                    # Ψ ended as a nonzero constant
                    psi, deg, fail = compare_spec(code, spec)
                    assert deg == 0 and psi[0] and not fail
            if spec.name.startswith("recur_double"):
                assert why == "derivative", (spec.name, why)
            if spec.name.startswith("recur_offdomain"):
                assert why == "roots", (spec.name, why)
            if spec.name.startswith("erasures"):
                assert why == "erasures"
    assert set(seen) == {None, "erasures", "degree", "derivative", "roots", "reencode"}, sorted(map(str, seen))
    # the degree check alone: Berlekamp–Massey found the true locator 1 - c·z^e of e > r errors on a coset
    assert any(name.startswith("beyond_coset") for name in seen["degree"])


@pytest.mark.parametrize("p,n,k", TINY, ids=[f"p{p}-n{n}-k{k}" for p, n, k in TINY])
def test_constructed_rows_that_decode_match_brute_force(p, n, k):
    g = generator(p)
    code = rc.Code(p, g, n, k)
    decoded = 0
    for seed in range(6):
        rng = np.random.default_rng([p, n, k, seed])
        specs = rc.deltas(code, rng) + rc.recurrences(code, rng) + rc.beyond_on_a_coset(code, rng)
        if not specs:
            continue
        rows, erased, _, _ = rc.build(code, specs, rc.forward_py(code))
        for spec, row, er in zip(specs, rows, erased):
            row, er = [int(v) for v in row], list(er)
            msg, st = decode(p, g, row, er, k)
            if spec.expect.status is not None:
                assert st == spec.expect.status, spec.name
            best = nearest(p, g, row, er, k)
            radius = (n - k - sum(1 for e in er if e)) // 2
            if msg is None:
                assert all(d > radius for d in best.values()), spec.name
            else:
                decoded += 1
                assert best[tuple(msg)] == st and all(d > radius for mm, d in best.items() if mm != tuple(msg)), spec.name
    assert decoded or n - k < 2
