"""ronk_poly_divrem_batch_u64 (ops.poly_divrem_batch, kzg.open_batch): batches of divisions by one shared divisor or one
divisor per row.

Every row must be word for word what the single-row device entry gives for it (its errors included) and what the oracle
gives, on the default context and on contexts made with RONK_DIVREM_BATCH_PATH=1 (literal) and =2 (Newton wherever it
fits).  Batch 1 must record the single-row launch sequence, and on each path batch 2 and batch 64 record the same names."""
import os

import numpy as np
import pytest

import oracle
from gpu_util import GL, MONT_PRIMES, ctx, dev, host, s64

pytestmark = pytest.mark.gpu

PRIMES = {"gl": (GL, 7), **{n: (p, g) for n, (p, g, s) in MONT_PRIMES.items() if s >= 16}}
LITERAL = {"p101": (101, 2), "p17": (17, 3), "p127": (127, 3), "gl_g0": (GL, 0)}   # the literal kernel at every size
BATCHES = [1, 2, 3, 7, 64]
# (da, db): da < db, da = db, db = 1, db = 2, short quotients with long divisors (L < db - 1: b·q taken mod x^nr - 1, with
# nr = 512 ≥ da at (300, 290), b folded at (300, 257) where db = nr + 1 = 257, a folded at (513, 258) where da > nr = 512),
# and two longer ones
SHAPES = [(5, 9), (40, 40), (300, 1), (300, 2), (300, 290), (300, 257), (513, 258), (256, 129),
          ((1 << 12) + 1, (1 << 11) + 1)]
EINVAL, EUNSUPPORTED = 1, 5
SENTINEL = s64(0xDEADBEEFDEADBEEF)
_forced = {}


def _ctx(kind):
    """The suite's context, or one on the suite's stream with RONK_DIVREM_BATCH_PATH = 1 (literal) or 2 (Newton)."""
    if kind == "default":
        return ctx()
    if kind not in _forced:
        import torch
        from ronkathon_b200 import Context
        ctx()
        os.environ["RONK_DIVREM_BATCH_PATH"] = {"literal": "1", "newton": "2"}[kind]
        try:
            _forced[kind] = Context(0, torch.cuda.current_stream().cuda_stream)
        finally:
            del os.environ["RONK_DIVREM_BATCH_PATH"]
    return _forced[kind]


def _p(x):
    from ronkathon_b200 import _lib
    return _lib._ptr(x)


def _rc(c, name, *args):
    from ronkathon_b200 import _lib
    c.sync()
    before = c.launches
    rc = getattr(_lib.lib(), name)(c._h, *args)
    c.sync()
    return rc, c.launches - before


def _names(c, fn):
    c.sync()
    c.prof_fetch()
    c.prof_enable(True)
    try:
        fn()
        c.sync()
    finally:
        c.prof_enable(False)
    return [n for n, _ in c.prof_fetch()]


def _single(c, p, g, a, b):
    """The single-row entry's (q, r), or its error code."""
    import torch
    from ronkathon_b200 import RonkError
    A = dev(a)
    q, r = torch.empty_like(A), torch.empty_like(A)
    try:
        c.call("ronk_poly_divrem_u64", p, g, _p(A), len(a), _p(dev(b)) if len(b) else None, len(b), _p(q), _p(r))
    except RonkError as e:
        return e.code
    return host(q), host(r)


def _batch(c, p, g, A, B):
    from ronkathon_b200 import RonkError, ops
    try:
        q, r = ops.poly_divrem_batch(c, dev(A), dev(B), p=p, g=g)
    except RonkError as e:
        return e.code
    return host(q), host(r)


def _check(c, p, g, A, B, oracle_rows=None):
    """The batch equals the single-row entry on every row, and the oracle on the rows listed (all by default)."""
    shared = B.ndim == 1
    got = _batch(c, p, g, A, B)
    rows = [_single(c, p, g, A[y], B if shared else B[y]) for y in range(len(A))]
    if any(isinstance(x, int) for x in rows):
        assert got == EINVAL and all(x in (EINVAL,) or not isinstance(x, int) for x in rows), (got, rows)
        return got
    assert not isinstance(got, int), f"the batch refused ({got}) what every single row took"
    for y, (q, r) in enumerate(rows):
        assert np.array_equal(got[0][y], q) and np.array_equal(got[1][y], r), f"row {y} differs from the single-row entry"
    for y in (range(len(A)) if oracle_rows is None else oracle_rows):
        oq, orr = oracle.poly_divrem(p, A[y], B if shared else B[y])
        assert np.array_equal(got[0][y], oq) and np.array_equal(got[1][y], orr), f"row {y} differs from the oracle"
    return got


def _divisors(p, db, n, seed):
    B = oracle.splitmix(p, seed, n * db).reshape(n, db)
    if db:
        B[:, -1] = B[:, -1] % (p - 1) + 1   # nonzero top words
    return B


def _dividends(p, da, n, seed):
    A = oracle.splitmix(p, seed, n * da).reshape(n, da)
    if n >= 3 and da >= 2:
        A[1][da // 2:] = 0   # zero top words
        A[2][:] = 0          # all zero
    return A


# ---- every row is the single-row entry's and the oracle's ------------------------------------------------------------

@pytest.mark.parametrize("kind", ["default", "literal", "newton"])
@pytest.mark.parametrize("batch", BATCHES)
@pytest.mark.parametrize("name", list(PRIMES))
def test_rows_match_single(name, batch, kind):
    p, g = PRIMES[name]
    c = _ctx(kind)
    for da, db in SHAPES:
        if kind == "literal" and da > 1000 and name != "gl":
            continue
        A = _dividends(p, da, batch, 10 + da + batch)
        B = _divisors(p, db, batch, 20 + db + batch)
        orows = range(batch) if da * max(da - db, 1) * batch < 1 << 22 else (0, batch - 1)
        _check(c, p, g, A, B[0], orows)   # shared
        _check(c, p, g, A, B, orows)      # per row


@pytest.mark.parametrize("batch", [1, 2, 7, 64])
@pytest.mark.parametrize("name", list(LITERAL))
def test_literal_primes(name, batch):
    p, g = LITERAL[name]
    for kind in ("default", "newton"):
        c = _ctx(kind)
        for da, db in [(5, 9), (40, 40), (300, 1), (300, 2), (300, 290), (256, 129)]:
            A, B = _dividends(p, da, batch, 30 + da), _divisors(p, db, batch, 40 + db)
            _check(c, p, g, A, B[0])
            _check(c, p, g, A, B)


@pytest.mark.parametrize("kind", ["default", "literal", "newton"])
@pytest.mark.parametrize("name", ["gl", "babybear"])
def test_2_16_rows(name, kind):
    """(2^16, 2^15 + 1): oracle on the last row only."""
    p, g = PRIMES[name]
    if kind == "literal" and name != "gl":
        pytest.skip("one prime on the quadratic path")
    c = _ctx(kind)
    da, db = 1 << 16, (1 << 15) + 1
    A, B = _dividends(p, da, 3, 50), _divisors(p, db, 3, 51)
    _check(c, p, g, A, B[0], (0,))
    _check(c, p, g, A, B, (2,))


def test_2_20_goldilocks():
    """(2^20, 2^19 + 1) × 4 on the default context, shared and per row, against the single-row entry; the identity
    a = q·b + r on one row, by products on the device."""
    from ronkathon_b200 import ops
    c = ctx()
    da, db = 1 << 20, (1 << 19) + 1
    A, B = _dividends(GL, da, 4, 60), _divisors(GL, db, 4, 61)
    for Bx in (B[0], B):
        got = _check(c, GL, 7, A, Bx, ())
        q, r = got
        b0 = Bx if Bx.ndim == 1 else Bx[0]
        qb = host(ops.poly_mul(c, dev(q[0][:da - db + 1]), dev(b0)))
        with np.errstate(over="ignore"):
            s = [(int(x) + int(y)) % GL for x, y in zip(qb, np.concatenate([r[0], np.zeros(len(qb) - da, np.uint64)]))]
        assert s[:da] == [int(x) for x in A[0]]


def test_grid_y_cap():
    """More than 65 535 rows of small rows: every path steps its rows by grid.y, the literal kernel (one CTA per row) over
    about 66 rows per CTA, with a zero-top divisor among the rows."""
    batch = 70000
    for kind in ("default", "literal", "newton"):
        c = _ctx(kind)
        for da, db in [(12, 5), (12, 2), (12, 15)]:
            A, B = _dividends(GL, da, batch, 70 + da), _divisors(GL, db, batch, 71 + db)
            for Bx in (B[0], B):
                got = _batch(c, GL, 7, A, Bx)
                assert not isinstance(got, int), (kind, da, db, got)
                for y in (0, 1, 2, 1055, 1056, 1057, 65535, 65536, batch - 1):
                    want = oracle.poly_divrem(GL, A[y], Bx if Bx.ndim == 1 else Bx[y])
                    assert np.array_equal(got[0][y], want[0]) and np.array_equal(got[1][y], want[1]), (kind, da, db, y)
    # one zero-top divisor sends all 70 000 rows to the literal kernel on every context
    da, db, at = 40, 9, 40000
    A, B = _dividends(GL, da, batch, 72), _divisors(GL, db, batch, 73)
    B[at][-1] = 0
    A[at][db - 1:] = 0   # one reduction step, then the remainder stays partly reduced (no panic)
    for kind in ("default", "literal", "newton"):
        got = _batch(_ctx(kind), GL, 7, A, B)
        assert not isinstance(got, int), (kind, got)
        for y in (0, 1, 2, 1056, at - 1, at, at + 1, 65536, batch - 1):
            want = oracle.poly_divrem(GL, A[y], B[y])
            assert np.array_equal(got[0][y], want[0]) and np.array_equal(got[1][y], want[1]), (kind, y)


# ---- quirky divisors --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["default", "newton"])
@pytest.mark.parametrize("at", [0, 3, 6])
def test_zero_top_word_in_one_row(at, kind):
    """One divisor with a zero top word sends every row to the literal kernel; every row still has the single-row words.
    Row `at`'s dividend is zero from x^(db-1) up, so the reference takes one step and leaves a partly reduced remainder
    instead of panicking; at = 6 also has a divisor of degree below db / 2."""
    c = _ctx(kind)
    for da, db in [(300, 2), (300, 129), (4097, 2049)]:
        A, B = _dividends(GL, da, 7, 80), _divisors(GL, db, 7, 81)
        B[at][-1] = 0
        if at == 6:
            B[at][db // 2:] = 0
        A[at][db - 1:] = 0
        got = _check(c, GL, 7, A, B, (at,))
        assert not isinstance(got, int), f"({da}, {db}) refused: {got}"
        if db > 2:
            assert np.any(got[0][at] != 0), "row at took no reduction step"
        # the shared divisor with a zero top word, every dividend zero from x^(db-1) up
        As = A.copy()
        As[:, db - 1:] = 0
        got = _check(c, GL, 7, As, B[at])
        assert not isinstance(got, int), f"({da}, {db}) shared refused: {got}"


@pytest.mark.parametrize("at", [0, 4, 6])
def test_panicking_rows(at):
    """An all-zero divisor against a nonzero dividend, and the index-out-of-range case, at any row: RONK_EINVAL, as the
    single-row entry gives on that row."""
    for kind in ("default", "newton"):
        c = _ctx(kind)
        A, B = _dividends(GL, 40, 7, 90), _divisors(GL, 8, 7, 91)
        A[at] = oracle.splitmix(GL, 92, 40)
        Z = B.copy()
        Z[at][:] = 0
        assert _check(c, GL, 7, A, Z) == EINVAL
        O = B.copy()
        O[at][:] = 0
        O[at][0], O[at][1] = 5, 0   # b = [5, 0, …, 0]: deg 0 with db = 8 reads past the dividend's end
        A2 = A.copy()
        A2[at][:] = 0
        A2[at][10], A2[at][9] = 9, 1   # step 1 clears x^10; step 2: diff 9, diff + db = 17 > plen = 10
        assert _single(c, GL, 7, A2[at], O[at]) == EINVAL
        assert _check(c, GL, 7, A2, O) == EINVAL
    c = ctx()
    assert _batch(c, GL, 7, A, Z[at]) == EINVAL   # the shared divisor


# ---- launch records ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["default", "literal", "newton"])
@pytest.mark.parametrize("da,db", [(300, 2), (300, 129), (40, 50), ((1 << 12) + 1, (1 << 11) + 1), (1 << 16, (1 << 15) + 1)])
def test_launch_records(da, db, kind):
    from ronkathon_b200 import ops
    c = _ctx(kind)
    A = {b: dev(_dividends(GL, da, b, 100)) for b in (1, 2, 64)}
    B = {b: dev(_divisors(GL, db, b, 101)) for b in (1, 2, 64)}
    for shared in (True, False):
        bat = (lambda b: ops.poly_divrem_batch(c, A[b], B[b][0] if shared else B[b]))
        for b in (1, 2, 64):
            bat(b)   # warm: plans and scratch
        one, two, many = (_names(c, lambda b=b: bat(b)) for b in (1, 2, 64))
        assert one == _names(c, lambda: ops.poly_divrem(c, A[1][0], B[1][0]))
        if kind == "default":   # the default rule takes the batch into account
            continue
        if da < 1 << 15:
            assert two == many, (two, many)
        else:   # the 2^16-point transforms: one cluster launch up to batch 2, two launches above
            assert [n for n in two if "ntt" not in n] == [n for n in many if "ntt" not in n]


@pytest.mark.parametrize("da,db,batch,newton", [
    (64, 17, 256, False), (64, 17, 4096, True),      # one wave of literal rows against four
    (256, 129, 16, False), (1024, 513, 2, True), (1024, 17, 2, True),
])
def test_path_rule_takes_the_batch(da, db, batch, newton):
    """The default context's path on each side of the measured rule, read from the launch record."""
    from ronkathon_b200 import ops
    c = ctx()
    A, B = dev(_dividends(GL, da, batch, 102)), dev(_divisors(GL, db, batch, 103))
    ops.poly_divrem_batch(c, A, B)
    names = _names(c, lambda: ops.poly_divrem_batch(c, A, B))
    assert ("poly_divrem_rows" not in names) == newton, names[:4]


# ---- refusals ---------------------------------------------------------------------------------------------------------

def test_refusals_write_nothing():
    import torch
    c = ctx()
    A, B = dev(_dividends(GL, 100, 3, 110)), dev(_divisors(GL, 10, 3, 111))
    q = torch.full((300,), SENTINEL, dtype=torch.int64, device="cuda")
    r = torch.full((300,), SENTINEL, dtype=torch.int64, device="cuda")
    name = "ronk_poly_divrem_batch_u64"
    cases = [
        ((GL, 7, None, 100, _p(B), 10, 0, 3, _p(q), _p(r)), EINVAL),
        ((GL, 7, _p(A), 100, None, 10, 0, 3, _p(q), _p(r)), EINVAL),
        ((GL, 7, _p(A), 100, _p(B), 10, 0, 3, None, _p(r)), EINVAL),
        ((GL, 7, _p(A), 100, _p(B), 10, 0, 3, _p(q), None), EINVAL),
        ((4, 7, _p(A), 100, _p(B), 10, 0, 3, _p(q), _p(r)), EINVAL),           # not a prime
        ((GL, GL, _p(A), 100, _p(B), 10, 0, 3, _p(q), _p(r)), EINVAL),         # g ≥ p
        ((GL, 7, _p(A), 100, _p(B), 10, 0, 3, _p(A), _p(r)), EINVAL),          # q over a
        ((GL, 7, _p(A), 100, _p(B), 10, 0, 3, _p(q), _p(B)), EINVAL),          # r over b
        ((GL, 7, _p(A), 100, _p(B), 10, 0, 3, _p(q), _p(q)), EINVAL),          # r over q
        ((GL, 7, _p(A), 100, _p(B), 10, 0, 0, _p(q), _p(r)), 0),               # batch 0
        ((GL, 7, _p(A), 0, _p(B), 10, 0, 3, _p(q), _p(r)), 0),                 # da 0
        ((GL, 7, None, 0, None, 10, 0, 3, None, None), 0),
    ]
    for args, want in cases:
        rc, launches = _rc(c, name, *args)
        assert (rc, launches) == (want, 0), (args, rc, launches)
        assert bool((q == SENTINEL).all()) and bool((r == SENTINEL).all()), args
    # a bad modulus comes before the envelope, and the envelope before any pointer is read
    rc, _ = _rc(c, name, 4, 7, _p(A), 0x7FFFFFF1, _p(B), 10, 0, 3, _p(q), _p(r))
    assert rc == EINVAL


def test_envelope_refusals_on_host_twin():
    """RONK_EUNSUPPORTED before anything is staged: small host arrays behind sizes that claim more."""
    c = ctx()
    a, b = np.zeros(8, np.uint64), np.ones(8, np.uint64)
    q, r = np.full(8, 7, np.uint64), np.full(8, 7, np.uint64)
    name = "ronk_poly_divrem_batch_u64_host"
    for args in [
        (GL, 7, _p(a), 0x7FFFFFF1, _p(b), 2, 0, 1, _p(q), _p(r)),             # da above the single-row bound
        (GL, 7, _p(a), 8, _p(b), 0x7FFFFFF1, 0, 1, _p(q), _p(r)),             # db above it
        (GL, 7, _p(a), 1 << 20, _p(b), 2, 1, (1 << 20) + 1, _p(q), _p(r)),    # batch·da above 2^40
        (GL, 7, _p(a), 8, _p(b), 1 << 20, 0, (1 << 20) + 1, _p(q), _p(r)),    # batch·db above 2^40
        (GL, 7, _p(a), 1 << 20, _p(b), (1 << 19) + 1, 1, (1 << 12) + 1, _p(q), _p(r)),  # 2^12 + 1 rows of 2^20 points
    ]:
        rc, launches = _rc(c, name, *args)
        assert (rc, launches) == (EUNSUPPORTED, 0), args
    assert np.all(q == 7) and np.all(r == 7)


def test_host_twin():
    c = ctx()
    from ronkathon_b200 import ops
    for p, g, da, db in ((GL, 7, 5000, 2501), (GL, 7, 300, 2), (101, 2, 50, 7), (GL, 7, 4, 9)):
        A, B = _dividends(p, da, 5, 120), _divisors(p, db, 5, 121)
        for shared in (True, False):
            Bx = B[0] if shared else B
            wq, wr = (host(t) for t in ops.poly_divrem_batch(c, dev(A), dev(Bx), p=p, g=g))
            q, r = np.empty_like(A), np.empty_like(A)
            c.call("ronk_poly_divrem_batch_u64_host", p, g, _p(A), da, _p(np.ascontiguousarray(Bx)), db, int(shared), 5, _p(q),
                   _p(r))
            assert np.array_equal(q, wq) and np.array_equal(r, wr)


def test_gated_non_blocking_stream():
    """A division on a fresh context's non-blocking stream behind a spin: it waits for the stream's earlier work, and its
    words are the default stream's."""
    import torch
    from ronkathon_b200 import Context, ops
    c0 = ctx()
    A, B = _dividends(GL, 1 << 13, 8, 130), _divisors(GL, (1 << 12) + 1, 8, 131)
    want = [host(t) for t in ops.poly_divrem_batch(c0, dev(A), dev(B))]
    s = torch.cuda.Stream()
    c = Context(0, s.cuda_stream)
    try:
        Ad, Bd = dev(A), dev(B)
        with torch.cuda.stream(s):
            ops.poly_divrem_batch(c, Ad, Bd)   # warm: plans and scratch
        s.synchronize()
        Ag, Bg = torch.zeros_like(Ad), torch.zeros_like(Bd)
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            torch.cuda._sleep(100_000_000)
            Ag.copy_(Ad)
            Bg.copy_(Bd)
            q, r = ops.poly_divrem_batch(c, Ag, Bg)
        s.synchronize()
        assert np.array_equal(ops.to_host(q), want[0]) and np.array_equal(ops.to_host(r), want[1])
    finally:
        c.close()


# ---- kzg::open over many polynomials ----------------------------------------------------------------------------------

def test_kzg_open_batch():
    from ronkathon_b200 import kzg
    ctx()
    g1, _ = kzg.setup()
    assert kzg.open_batch([[11, 11, 11, 1]], 4, g1)[0].raw == bytes([26, 0, 45, 0])   # kzg/tests.rs:327-337
    polys = [[int(v) % 17 for v in oracle.splitmix(17, 140 + i, 4 + (i % 3))] for i in range(9)]
    for z in (0, 4, 16):
        assert kzg.open_batch(polys, z, g1) == [kzg.open_(f, z, g1) for f in polys]
