"""ronk_ntt_any_u64[_host]: transforms of any n | p - 1, forward and inverse.

Values are compared with routes that share no code with Bluestein's path: ronk_dft_u64 (one CTA per point), the
oracle's literal dft, Horner at sampled points, and ronk_ntt_u64 for powers of two.  Each call's launch record is
checked against `path`, a restatement of ntt_any.cu's path rule, on contexts whose RONK_ANYNTT_MIN forces Bluestein
(1) or keeps it off (2^30) and on the default crossover."""
import os

import numpy as np
import pytest

import oracle
from gpu_util import GL, MONT_PRIMES, ctx, dev, host

pytestmark = pytest.mark.gpu

EINVAL, EUNSUPPORTED = 1, 5
LITERAL_MAX = 1 << 17
OFF = 1 << 30
PRIMES = {**{k: (p, g) for k, (p, g, _) in MONT_PRIMES.items()}, "goldilocks": (GL, 7), "f101": (101, 2), "f17": (17, 14),
          "f127": (127, 3)}
GENERATORS = [k for k in PRIMES if k != "gl_g5"]   # 7^5 is no generator of F_p*: its "inverse" is no inverse
KOALABEAR, P32 = MONT_PRIMES["koalabear"][0], MONT_PRIMES["p32"][0]
SENTINEL = -1    # 0xFFFF…: no residue of any test prime

_ctxs = {}


def _context(min_n):
    """A context on the suite's stream whose RONK_ANYNTT_MIN is min_n (None: the measured crossover)."""
    import torch
    from ronkathon_b200 import Context
    if min_n not in _ctxs:
        ctx()
        old = os.environ.pop("RONK_ANYNTT_MIN", None)
        if min_n is not None:
            os.environ["RONK_ANYNTT_MIN"] = str(min_n)
        try:
            _ctxs[min_n] = Context(0, torch.cuda.current_stream().cuda_stream)
        finally:
            os.environ.pop("RONK_ANYNTT_MIN", None)
            if old is not None:
                os.environ["RONK_ANYNTT_MIN"] = old
    return _ctxs[min_n]


@pytest.fixture(scope="module", autouse=True)
def _close_contexts():
    yield
    for c in _ctxs.values():
        c.close()
    _ctxs.clear()


def crossover():
    """The crossover compiled into ntt_any.cu (kAnyNttMin), read from the source so that the rule below tracks it."""
    import re
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "ronkathon_b200", "csrc",
                            "ntt_any.cu")).read()
    return int(re.search(r"kAnyNttMin = (\d+);", src).group(1))


def conv_log(n):
    return (2 * n - 2).bit_length()


def path(p, n, min_n=None):
    """ntt_any.cu's path rule: 'pow2', 'bluestein', 'literal' or None (RONK_EUNSUPPORTED)."""
    min_n = crossover() if min_n is None else min_n
    if n & (n - 1) == 0:
        return "pow2" if n <= 1 << 26 else None
    if conv_log(n) <= 26 and (p - 1) % (1 << conv_log(n)) == 0 and n >= min_n:
        return "bluestein"
    return "literal" if n <= LITERAL_MAX else None


def odd_divisors(p, cap):
    m = p - 1
    while m % 2 == 0:
        m //= 2
    return [d for d in range(3, cap, 2) if m % d == 0]


def run(c, p, g, a, n, batch=1, inverse=False):
    from ronkathon_b200 import ops
    d = dev(a)
    ops.ntt_any_(c, d, n, batch, inverse=inverse, p=p, g=g)
    c.sync()
    return host(d)


def dft_device(p, g, a):
    import torch
    n = len(a)
    out = torch.empty(n, dtype=torch.int64, device="cuda")
    ctx().call("ronk_dft_u64", p, g, dev(a).data_ptr(), n, out.data_ptr())
    return host(out)


def inv_dft(p, g, X):
    """n^-1 · dft with g^-1, Python ints."""
    n = len(X)
    ninv = pow(n, p - 2, p)
    return np.array([int(v) * ninv % p for v in oracle.dft(p, X, g=pow(g, p - 2, p))], dtype=np.uint64)


def horner_samples(p, g, a, got, count=12, seed=0):
    n = len(a)
    w = pow(g, (p - 1) // n, p)
    idx = sorted({0, 1, n - 1} | set(int(v) for v in oracle.splitmix(n, seed + 7, count)))
    for k in idx:
        assert int(got[k]) == oracle.poly_eval_horner(p, a, pow(w, k, p)), (hex(p), n, k)


def record(c, fn):
    """Warm fn once, then the profile names of one profiled call and the launches of one unprofiled call."""
    fn()
    c.sync()
    c.prof_fetch()
    c.prof_enable(True)
    try:
        fn()
        names = [nm for nm, _ in c.prof_fetch()]
    finally:
        c.prof_enable(False)
    before = c.launches
    fn()
    c.sync()
    return names, c.launches - before


# ---- values -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(PRIMES))
def test_small_n_every_prime(name):
    """Every n | p - 1 up to 1024 that is not a power of two (a sample of at most 14), on both forced paths and the
    default: forward bit-identical to ronk_dft_u64 and the oracle, inverse to n^-1 · dft(g^-1)."""
    p, g = PRIMES[name]
    ns = [n for n in range(3, 1025) if (p - 1) % n == 0 and n & (n - 1)]
    ns = ns[:10] + ns[-4:] if len(ns) > 14 else ns
    for n in ns:
        a = oracle.splitmix(p, 40 + n, n)
        a[0] = p - 1
        exp = oracle.dft(p, a, g=g)
        assert np.array_equal(dft_device(p, g, a), exp), (name, n)
        iexp = inv_dft(p, g, a)
        for min_n in (1, OFF, None):
            c = _context(min_n)
            assert np.array_equal(run(c, p, g, a, n), exp), (name, n, min_n)
            assert np.array_equal(run(c, p, g, a, n, inverse=True), iexp), (name, n, min_n)


LARGE = [("goldilocks", 3 << 21), ("goldilocks", 257 * 4096), ("goldilocks", 65537 * 16), ("babybear", 15 << 20),
         ("koalabear", 127 << 10), ("p32", 21 << 10), ("p57", 29 << 14), ("pbig", None), ("gl_g5", 5 << 18)]


@pytest.mark.parametrize("name,n", LARGE, ids=[f"{a}-{b}" for a, b in LARGE])
def test_large_n(name, n):
    """Large n on the default context: Horner at sampled k, and (with a generator) inverse∘forward = id in full."""
    p, g = PRIMES[name]
    if n is None:
        n = odd_divisors(p, 1 << 12)[0] << 12
    assert (p - 1) % n == 0
    assert path(p, n) == "bluestein"
    a = oracle.splitmix(p, 50, n)
    a[-1] = p - 1
    got = run(ctx(), p, g, a, n)
    horner_samples(p, g, a, got)
    if name in GENERATORS:
        assert np.array_equal(run(ctx(), p, g, got, n, inverse=True), a)


@pytest.mark.parametrize("name", ["goldilocks", "babybear"])
@pytest.mark.parametrize("log_n", [0, 1, 5, 10, 16, 20])
def test_power_of_two_is_ntt(name, log_n):
    from ronkathon_b200 import ops
    p, g = PRIMES[name]
    n = 1 << log_n
    a = oracle.splitmix(p, 60 + log_n, 3 * n)
    for inverse in (False, True):
        want = dev(a)
        ops.ntt_(ctx(), want, log_n, 3, inverse=inverse, p=p, g=g)
        assert np.array_equal(run(ctx(), p, g, a, n, 3, inverse), host(want)), (log_n, inverse)


# ---- the envelope ------------------------------------------------------------------------------------------------------
def expect_refused(c, p, g, n, code, words=None, batch=1):
    """The call returns `code` and leaves a sentinel-filled device buffer and host array untouched."""
    import torch
    from ronkathon_b200 import _lib
    words = batch * n if words is None else words
    d = torch.full((words,), SENTINEL, dtype=torch.int64, device="cuda")
    rc = _lib.lib().ronk_ntt_any_u64(c._h, p, g, _lib._ptr(d), n, batch, 0)
    assert rc == code, (hex(p), g, n, rc)
    c.sync()
    assert bool((d == SENTINEL).all())
    if words <= 1 << 20:
        h = np.full(words, 0xFFFFFFFFFFFFFFFF, dtype=np.uint64)
        rc = _lib.lib().ronk_ntt_any_u64_host(c._h, p, g, _lib._ptr(h), n, batch, 1)
        assert rc == code and bool((h == 0xFFFFFFFFFFFFFFFF).all())


def test_goldilocks_top_of_envelope():
    """n = 3·2^23 (N = 2^26) runs; n = 65537·2^9, just over 2^25 and off both other paths, is refused."""
    n = 3 << 23
    assert path(GL, n) == "bluestein" and conv_log(n) == 26
    a = oracle.splitmix(GL, 70, n)
    got = run(ctx(), GL, 7, a, n)
    horner_samples(GL, 7, a, got, count=4)
    assert np.array_equal(run(ctx(), GL, 7, got, n, inverse=True), a)
    del got
    n = 65537 << 9
    assert n > 1 << 25 and path(GL, n) is None
    expect_refused(ctx(), GL, 7, n, EUNSUPPORTED, words=1 << 10)


def test_koalabear_two_adicity_edge():
    p, g = PRIMES["koalabear"]
    n = 127 << 16
    assert path(p, n) == "bluestein" and conv_log(n) == 24
    a = oracle.splitmix(p, 71, n)
    got = run(ctx(), p, g, a, n)
    horner_samples(p, g, a, got, count=6)
    assert np.array_equal(run(ctx(), p, g, got, n, inverse=True), a)
    assert path(p, 127 << 17) is None
    expect_refused(ctx(), p, g, 127 << 17, EUNSUPPORTED, words=1 << 10)


def test_p32_paths_and_literal_cap():
    """p32 (p - 1 = 2^16·3·7·3121): 21·2^10 takes Bluestein (N = 2^16), 3·2^14 the literal kernels (N = 2^17 ∤ p - 1),
    7·2^14 ≤ 2^17 is the literal path's largest size here, 3·2^16 above the cap is refused."""
    p, g = PRIMES["p32"]
    for n, want in ((21 << 10, "bluestein"), (3 << 14, "literal"), (7 << 14, "literal")):
        assert path(p, n) == want, n
        a = oracle.splitmix(p, 72, n)
        got = run(ctx(), p, g, a, n)
        horner_samples(p, g, a, got, count=4)
        assert np.array_equal(run(ctx(), p, g, got, n, inverse=True), a), n
    assert path(p, 3 << 16) is None
    expect_refused(ctx(), p, g, 3 << 16, EUNSUPPORTED, words=1 << 10)


def test_n_one():
    for name in ("goldilocks", "f101", "babybear"):
        p, g = PRIMES[name]
        a = oracle.splitmix(p, 73, 5)
        for inverse in (False, True):
            assert np.array_equal(run(ctx(), p, g, a, 1, 5, inverse), a)


def test_errors_leave_buffers_untouched():
    import torch
    from ronkathon_b200 import _lib
    c = ctx()
    for p, g, n, code in ((GL, 7, 0, EINVAL), (GL, 7, 7, EINVAL), (GL, 0, 3, EINVAL), (GL, GL, 3, EINVAL),
                          (101, 2, 3, EINVAL), (2, 1, 1, EUNSUPPORTED), (P32, 5, 3 << 16, EUNSUPPORTED)):
        expect_refused(c, p, g, n, code, words=max(n, 1) if n < 1 << 12 else 1 << 10)
    assert _lib.lib().ronk_ntt_any_u64(c._h, GL, 7, None, 3, 1, 0) == EINVAL
    assert _lib.lib().ronk_ntt_any_u64_host(c._h, GL, 7, None, 3, 1, 0) == EINVAL
    d = torch.full((3,), SENTINEL, dtype=torch.int64, device="cuda")
    assert _lib.lib().ronk_ntt_any_u64(c._h, GL, 7, _lib._ptr(d), 3, 0, 0) == 0   # batch 0: nothing to do
    c.sync()
    assert bool((d == SENTINEL).all())


# ---- paths -------------------------------------------------------------------------------------------------------------
def _transform_names(c, p, g, log_n, batch, inverse, mul):
    from ronkathon_b200 import ops
    x = dev(oracle.splitmix(p, 80, batch << log_n))
    if mul:
        mm = dev(np.tile(oracle.splitmix(p, 81, 1 << log_n), batch))
        return record(c, lambda: ops.ntt_mul_(c, x, mm, log_n, batch, p=p, g=g))[0]
    return record(c, lambda: ops.ntt_(c, x, log_n, batch, inverse=inverse, p=p, g=g))[0]


def expected_names(c, p, g, n, batch, inverse, min_n):
    kind = path(p, n, min_n)
    if kind == "pow2":
        return _transform_names(c, p, g, n.bit_length() - 1, batch, inverse, False) if n > 1 else []
    if kind == "literal":
        return ["pow_table"] + ["poly_eval"] * batch + (["anyntt_chirp_out"] if inverse else [])
    lg = conv_log(n)
    return (["anyntt_chirp_in"] + _transform_names(c, p, g, lg, batch, False, True)
            + _transform_names(c, p, g, lg, batch, True, False) + ["anyntt_chirp_out"])


PATH_SIZES = [("goldilocks", 3), ("goldilocks", 15), ("goldilocks", 255), ("goldilocks", 257 * 4), ("goldilocks", 3 << 12),
              ("goldilocks", 1024), ("babybear", 5 * 64), ("babybear", 15 << 10), ("p32", 21 << 8)]


@pytest.mark.parametrize("name,n", PATH_SIZES, ids=[f"{a}-{b}" for a, b in PATH_SIZES])
def test_launch_record_follows_the_path_rule(name, n):
    """Both forced settings and the default: the record matches the restated rule, and the two paths give the same
    words."""
    from ronkathon_b200 import ops
    p, g = PRIMES[name]
    a = oracle.splitmix(p, 90, 2 * n)
    results = []
    for min_n in (1, OFF, None):
        c = _context(min_n)
        for inverse in (False, True):
            d = dev(a)
            names, launches = record(c, lambda: ops.ntt_any_(c, d, n, 2, inverse=inverse, p=p, g=g))
            exp = expected_names(c, p, g, n, 2, inverse, min_n)
            assert names == exp, (min_n, inverse)
            assert launches == len(exp)
            results.append(run(c, p, g, a, n, 2, inverse))
    for i in range(2, len(results)):
        assert np.array_equal(results[i], results[i % 2]), i


PINNED = {
    # (min_n, p, g, n, inverse) → profile names after a warm call
    "bluestein_gl_3x2^14": ((1, GL, 7, 3 << 14, False),
                            ["anyntt_chirp_in", "ntt3_split", "ntt3_pass2", "ntt3_pass3", "intt3_split", "intt3_pass2",
                             "intt3_pass3", "anyntt_chirp_out"]),
    "literal_gl_960_inverse": ((OFF, GL, 7, 960, True), ["pow_table", "poly_eval", "anyntt_chirp_out"]),
    "literal_gl_960": ((OFF, GL, 7, 960, False), ["pow_table", "poly_eval"]),
    "pow2_gl_2^10": ((1, GL, 7, 1024, False), ["ntt_single"]),
}


@pytest.mark.parametrize("case", list(PINNED))
def test_launch_record_pinned(case):
    from ronkathon_b200 import ops
    (min_n, p, g, n, inverse), want = PINNED[case]
    c = _context(min_n)
    d = dev(oracle.splitmix(p, 91, n))
    names, launches = record(c, lambda: ops.ntt_any_(c, d, n, 1, inverse=inverse, p=p, g=g))
    assert names == want and launches == len(want)


# ---- contract ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,n", [("goldilocks", 3 << 12), ("babybear", 5 * 64), ("f101", 25)])
def test_batch_equals_separate_calls_and_host_equals_device(name, n):
    p, g = PRIMES[name]
    a = oracle.splitmix(p, 92, 5 * n)
    for inverse in (False, True):
        got = run(ctx(), p, g, a, n, 5, inverse)
        for b in range(5):
            sl = slice(b * n, (b + 1) * n)
            assert np.array_equal(got[sl], run(ctx(), p, g, a[sl].copy(), n, 1, inverse)), (b, inverse)
        h = a.copy()
        ctx().call("ronk_ntt_any_u64_host", p, g, h.ctypes.data, n, 5, int(inverse))
        assert np.array_equal(h, got), inverse


def test_spectrum_cache_is_keyed_by_n():
    """A second n on the same context, then the first again in both directions: bit-exact to a fresh context.
    3·2^12 and 5·2^11 share N = 2^14, so a key on N alone would hand the second the first's spectrum."""
    from ronkathon_b200 import Context
    import torch
    c = _context(1)
    n1, n2 = 3 << 12, 5 << 11
    a1, a2 = oracle.splitmix(GL, 93, n1), oracle.splitmix(GL, 94, n2)
    first = [run(c, GL, 7, a1, n1, 1, inv) for inv in (False, True)]
    second = run(c, GL, 7, a2, n2)
    again = [run(c, GL, 7, a1, n1, 1, inv) for inv in (False, True)]
    os.environ["RONK_ANYNTT_MIN"] = "1"
    try:
        fresh = Context(0, torch.cuda.current_stream().cuda_stream)
    finally:
        del os.environ["RONK_ANYNTT_MIN"]
    try:
        assert np.array_equal(second, run(fresh, GL, 7, a2, n2))
    finally:
        fresh.close()
    assert all(np.array_equal(x, y) for x, y in zip(first, again))
    assert np.array_equal(first[0], dft_device(GL, 7, a1))


def test_small_calls_after_a_2_26_point_call():
    """Scratch left by an n = 3·2^23 call (N = 2^26) holds junk; small calls there match a fresh context."""
    from ronkathon_b200 import Context
    import torch
    c = Context(0, torch.cuda.current_stream().cuda_stream)
    try:
        big = oracle.splitmix(GL, 95, 3 << 23)
        run(c, GL, 7, big, 3 << 23)
        del big
        for p, g, n in ((GL, 7, 3 << 12), (GL, 7, 255), (PRIMES["babybear"][0], 31, 5 * 64), (101, 2, 25)):
            a = oracle.splitmix(p, 96, 3 * n)
            for inverse in (False, True):
                fresh = Context(0, torch.cuda.current_stream().cuda_stream)
                try:
                    assert np.array_equal(run(c, p, g, a, n, 3, inverse), run(fresh, p, g, a, n, 3, inverse)), (n, inverse)
                finally:
                    fresh.close()
    finally:
        c.close()


def test_behind_a_gated_stream():
    """The gate of test_gpu_streams.py: a warm context on a non-blocking stream s; on s a bounded spin, the real input
    written over a wrong one, the call, a clone.  s must still be busy when the call returns, and the clone must equal
    the result on the suite's context."""
    import torch
    from ronkathon_b200 import Context
    n, batch = 3 << 12, 2
    real = dev(oracle.splitmix(GL, 97, batch * n))
    want = real.clone()
    from ronkathon_b200 import ops
    ops.ntt_any_(ctx(), want, n, batch)
    ctx().sync()
    s = torch.cuda.Stream()
    os.environ["RONK_ANYNTT_MIN"] = "1"
    try:
        c = Context(0, s.cuda_stream)
    finally:
        del os.environ["RONK_ANYNTT_MIN"]
    try:
        buf = real.flip(0).contiguous()
        with torch.cuda.stream(s):
            c.call("ronk_ntt_any_u64", GL, 7, buf.clone().data_ptr(), n, batch, 0)   # warm: spectrum and plans
        s.synchronize()
        real.clone().copy_(real)
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            torch.cuda._sleep(100_000_000)
            buf.copy_(real)
            c.call("ronk_ntt_any_u64", GL, 7, buf.data_ptr(), n, batch, 0)
            assert not s.query(), "s finished before the call returned"
            got = buf.clone()
        s.synchronize()
        assert torch.equal(got, want)
    finally:
        c.close()


def test_polynomial_idft_round_trip():
    from ronkathon_b200.field import PlutoBaseField
    from ronkathon_b200.polynomial import Lagrange, Monomial, Polynomial
    for n in (5, 10, 25, 100):
        coeffs = [int(v) for v in oracle.splitmix(101, n, n)]
        poly = Polynomial(coeffs, PlutoBaseField)
        X = poly.dft()
        back = X.idft()
        assert back.basis is Monomial and X.basis is Lagrange
        assert [int(v) for v in back.coefficients] == coeffs
