"""ronk_poly_multieval_batch_u64 / ronk_poly_interpolate_batch_u64 (ops.poly_multieval_batch, poly_interpolate_batch,
codes.shamir_split, shamir_combine): batches of rows over one shared point set, one subproduct tree per call.

Every row must be word for word what the single-row device entry gives for it (its errors included), on the default
context and on one made with RONK_TREE_MIN=1, which takes the tree wherever its transforms fit.  Batch 1 must record the
single-row launch sequence, and the launch sequence from batch 2 on must not depend on the batch."""
import os
import random

import numpy as np
import pytest

import oracle
from gpu_util import GL, MONT_PRIMES, ctx, dev, host, s64

pytestmark = pytest.mark.gpu

PRIMES = {"gl": (GL, 7), **{n: (p, g) for n, (p, g, s) in MONT_PRIMES.items() if s >= 16}}
LITERAL = {"p101": (101, 2), "p17": (17, 3), "p127": (127, 3), "gl_g0": (GL, 0)}   # off the tree at every size
SIZES = [1, 64, 65, (1 << 12) - 1, (1 << 12) + 1, (1 << 15) + 3]
BATCHES = [1, 2, 3, 7, 64]
EINVAL, EUNSUPPORTED = 1, 5
SENTINEL = s64(0xDEADBEEFDEADBEEF)
_tree = None


def _ctx(kind):
    """The suite's context, or one on the suite's stream that takes the tree at every size it fits."""
    global _tree
    if kind == "default":
        return ctx()
    if _tree is None:
        import torch
        from ronkathon_b200 import Context
        ctx()
        os.environ["RONK_TREE_MIN"] = "1"
        try:
            _tree = Context(0, torch.cuda.current_stream().cuda_stream)
        finally:
            del os.environ["RONK_TREE_MIN"]
    return _tree


def _p(x):
    from ronkathon_b200 import _lib
    return _lib._ptr(x)


def _rc(c, name, *args):
    """The return code of one C call, and the launches it made."""
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


def _points(p, m, seed, distinct):
    """m points with 0 and p - 1 among them (m ≥ 3): distinct, or with a repeated point (m ≥ 4)."""
    if distinct and p < 1 << 20:
        xs = np.array(random.Random(seed).sample(range(1, p - 1), max(m - 2, 0) if m >= 3 else m), dtype=np.uint64)
        if m >= 3:
            xs = np.insert(xs, 0, 0)
            xs = np.insert(xs, m // 2, p - 1)
    elif distinct:
        xs = np.unique(oracle.splitmix(p, seed, m + 64) % (p - 1) + 1)[:m].copy()
        random.Random(seed).shuffle(xs)
        if m >= 3:
            xs[0], xs[m // 2] = 0, p - 1
    else:
        xs = oracle.splitmix(p, seed, m)
        if m >= 4:
            xs[2] = xs[1]
        if m >= 3:
            xs[0], xs[m // 2] = 0, p - 1
    assert len(xs) == m and (not distinct or len(np.unique(xs)) == m)
    return np.ascontiguousarray(xs, dtype=np.uint64)


def _single(c, name, *args):
    """Row-wise reference: the single-row entry's words, or its error code."""
    from ronkathon_b200 import RonkError
    try:
        return c.call(name, *args) or 0
    except RonkError as e:
        return e.code


def _multieval_rows(c, p, g, F, xs):
    """(batch-call result or error, per-row single-row results or errors)."""
    import torch
    from ronkathon_b200 import RonkError, ops
    X = dev(xs)
    rows = []
    for f in F:
        out = torch.empty(len(xs), dtype=torch.int64, device="cuda")
        rc = _single(c, "ronk_poly_multieval_u64", p, g, _p(dev(f)), len(f), _p(X), len(xs), _p(out))
        rows.append(rc if rc else host(out))
    try:
        got = host(ops.poly_multieval_batch(c, dev(F), X, p=p, g=g)).reshape(len(F), len(xs))
    except RonkError as e:
        got = e.code
    return got, rows


def _interpolate_rows(c, p, g, xs, Y):
    import torch
    from ronkathon_b200 import RonkError, ops
    X = dev(xs)
    rows = []
    for y in Y:
        out = torch.empty(len(xs), dtype=torch.int64, device="cuda")
        rc = _single(c, "ronk_poly_interpolate_u64", p, g, _p(X), _p(dev(y)), len(xs), _p(out))
        rows.append(rc if rc else host(out))
    try:
        got = host(ops.poly_interpolate_batch(c, X, dev(Y), p=p, g=g)).reshape(len(Y), len(xs))
    except RonkError as e:
        got = e.code
    return got, rows


def _same(got, rows):
    if isinstance(got, int):
        assert all(isinstance(r, int) and r == got for r in rows), (got, rows)
        return
    for b, r in enumerate(rows):
        assert not isinstance(r, int), f"row {b}: the single-row entry refused ({r}) what the batch took"
        assert np.array_equal(got[b], r), f"row {b} differs from the single-row entry"


# ---- every row is the single-row entry's ------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["default", "tree"])
@pytest.mark.parametrize("batch", BATCHES)
@pytest.mark.parametrize("m", SIZES)
@pytest.mark.parametrize("name", list(PRIMES))
def test_multieval_rows_match_single(name, m, batch, kind):
    """Points 0, p - 1 and a repeated point; d below and above m."""
    p, g = PRIMES[name]
    c = _ctx(kind)
    xs = _points(p, m, 11 + m, distinct=False)
    for d in sorted({max(1, m // 2), 2 * m + 3}):
        if kind == "default" and name != "gl" and batch * d * m > 1 << 31:   # the largest literal runs on one prime only
            continue
        F = oracle.splitmix(p, 100 + d + batch, batch * d).reshape(batch, d)
        got, rows = _multieval_rows(c, p, g, F, xs)
        _same(got, rows)
        if not isinstance(got, int):
            for i in (0, m // 2, m - 1):
                assert int(got[-1][i]) == oracle.poly_eval_horner(p, F[-1], int(xs[i]))


@pytest.mark.parametrize("kind", ["default", "tree"])
@pytest.mark.parametrize("batch", BATCHES)
@pytest.mark.parametrize("k", SIZES)
@pytest.mark.parametrize("name", list(PRIMES))
def test_interpolate_rows_match_single(name, k, batch, kind):
    p, g = PRIMES[name]
    c = _ctx(kind)
    xs = _points(p, k, 21 + k, distinct=True)
    Y = oracle.splitmix(p, 200 + k + batch, batch * k).reshape(batch, k)
    got, rows = _interpolate_rows(c, p, g, xs, Y)
    _same(got, rows)
    if not isinstance(got, int):
        for i in (0, k - 1):
            assert oracle.poly_eval_horner(p, got[-1], int(xs[i])) == int(Y[-1][i])


@pytest.mark.parametrize("batch", [1, 2, 7, 64])
@pytest.mark.parametrize("name", list(LITERAL))
def test_literal_paths(name, batch):
    """Tiny primes and g = 0: one poly_eval launch, one interp_master / interp_nodes / interp_sum sequence for all rows."""
    p, g = LITERAL[name]
    for kind in ("default", "tree"):
        c = _ctx(kind)
        for m in sorted({1, min(16, p - 1), min(100, p - 1)}):
            xs = _points(p, m, 31 + m, distinct=False)
            for d in (1, m + 5):
                _same(*_multieval_rows(c, p, g, oracle.splitmix(p, 40 + d, batch * d).reshape(batch, d), xs))
            xs = _points(p, m, 41 + m, distinct=True)
            Y = oracle.splitmix(p, 50 + m, batch * m).reshape(batch, m)
            got, rows = _interpolate_rows(c, p, g, xs, Y)
            _same(got, rows)
            assert [oracle.poly_eval_horner(p, got[-1], int(x)) for x in xs] == [int(y) for y in Y[-1]]


# ---- round trips at scale ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("batch,log_m", [(16, 20), (256, 12)])
def test_round_trip(batch, log_m):
    from ronkathon_b200 import ops
    c = ctx()
    m = 1 << log_m
    xs = _points(GL, m, 7, distinct=True)
    F = dev(oracle.splitmix(GL, 8, batch * m).reshape(batch, m))
    X = dev(xs)
    V = ops.poly_multieval_batch(c, F, X)
    back = ops.poly_interpolate_batch(c, X, V)
    c.sync()
    assert bool((back == F).all()), "interpolate(multieval(F)) != F"
    v, f = host(V).reshape(batch, m), host(F).reshape(batch, m)
    for b, i in ((0, 0), (batch - 1, m - 1), (batch // 2, 12345 % m)):
        assert int(v[b][i]) == oracle.poly_eval_horner(GL, f[b], int(xs[i]))


# ---- launch records ---------------------------------------------------------------------------------------------------

LAUNCH_SHAPES = [(65, 65), (4097, 4097), (4097, 100), (100, 4097), ((1 << 15) + 3, (1 << 15) + 3)]


@pytest.mark.parametrize("kind", ["default", "tree"])
@pytest.mark.parametrize("m,d", LAUNCH_SHAPES)
def test_launch_records(m, d, kind):
    """Batch 1 records the single-row entry's names.  On one path (the tree context) batch 2 and batch 64 record the same
    names and count, save that ronk_ntt_u64 picks the kernels of 2^16-point transforms by batch."""
    from ronkathon_b200 import ops
    c = _ctx(kind)
    xs = dev(_points(GL, m, 3, distinct=True))
    F = {b: dev(oracle.splitmix(GL, 4, b * d).reshape(b, d)) for b in (1, 2, 64)}
    Y = {b: dev(oracle.splitmix(GL, 5, b * m).reshape(b, m)) for b in (1, 2, 64)}
    pairs = [(lambda b: ops.poly_multieval_batch(c, F[b], xs), lambda: ops.poly_multieval(c, F[1][0], xs)),
             (lambda b: ops.poly_interpolate_batch(c, xs, Y[b]), lambda: ops.poly_interpolate(c, xs, Y[1][0]))]
    for batched, single in pairs:
        for b in (1, 2, 64):
            batched(b)   # warm: plans and scratch
        single()
        one, two, many = (_names(c, lambda b=b: batched(b)) for b in (1, 2, 64))
        assert one == _names(c, single)
        if kind == "default":   # the default path rule takes the batch into account: 2 and 64 rows may differ in path
            continue
        if max(m, 2 * d) < 1 << 16:
            assert two == many
        else:   # the 2^16-point transforms: one cluster launch up to batch 2, two launches above
            assert [n for n in two if "ntt" not in n] == [n for n in many if "ntt" not in n]


@pytest.mark.parametrize("what,batch,n,tree", [
    ("multieval", 1, 16384, False), ("multieval", 1, 32768, True),    # the single-row crossover
    ("multieval", 2, 16384, False), ("multieval", 4, 16384, True),    # batch·n² from 2^30
    ("multieval", 16, 4096, False), ("multieval", 16, 8192, True),
    ("multieval", 256, 512, False), ("multieval", 256, 1024, True),   # batch·n from 2^18
    ("interpolate", 1, 1024, False), ("interpolate", 1, 2048, True),
    ("interpolate", 64, 1024, False), ("interpolate", 256, 1024, True),   # batch·k² from 2^28
])
def test_path_rule_takes_the_batch(what, batch, n, tree):
    """The default context's path on each side of the batched crossovers, read from the launch record."""
    from ronkathon_b200 import ops
    c = ctx()
    xs = dev(_points(GL, n, 6, distinct=True))
    rows = dev(oracle.splitmix(GL, 7, batch * n).reshape(batch, n))
    fn = (lambda: ops.poly_multieval_batch(c, rows, xs)) if what == "multieval" else (lambda: ops.poly_interpolate_batch(c, xs, rows))
    fn()
    names = _names(c, fn)
    assert ("tree_leaves" in names) == tree, names[:4]


# ---- refusals, poisoned outputs and guard words -----------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["default", "tree"])
@pytest.mark.parametrize("k", [5, 65, 3000, 4097])
def test_repeated_node_leaves_out_untouched(k, kind):
    import torch
    c = _ctx(kind)
    xs = _points(GL, k, 9, distinct=True)
    xs[k - 1] = xs[1]
    Y = dev(oracle.splitmix(GL, 10, 3 * k).reshape(3, k))
    out = torch.full((3 * k + 8,), SENTINEL, dtype=torch.int64, device="cuda")
    rc, _ = _rc(c, "ronk_poly_interpolate_batch_u64", GL, 7, _p(dev(xs)), _p(Y), k, 3, _p(out))
    assert rc == EINVAL
    assert bool((out == SENTINEL).all()), "a refused interpolation wrote out"


@pytest.mark.parametrize("kind", ["default", "tree"])
@pytest.mark.parametrize("name", ["gl", "babybear", "p101"])
def test_guard_words(name, kind):
    import torch
    p, g = {**PRIMES, **LITERAL}[name]
    c = _ctx(kind)
    for m in (63, 65, 4097):
        if m >= p:
            continue
        xs = dev(_points(p, m, 12, distinct=True))
        F = dev(oracle.splitmix(p, 13, 3 * m).reshape(3, m))
        out = torch.full((3 * m + 64,), SENTINEL, dtype=torch.int64, device="cuda")
        c.call("ronk_poly_multieval_batch_u64", p, g, _p(F), m, 3, _p(xs), m, _p(out))
        c.sync()
        assert bool((out[3 * m:] == SENTINEL).all()), "multieval wrote past out[batch·m)"
        back = torch.full((3 * m + 64,), SENTINEL, dtype=torch.int64, device="cuda")
        c.call("ronk_poly_interpolate_batch_u64", p, g, _p(xs), _p(out), m, 3, _p(back))
        assert bool((back[3 * m:] == SENTINEL).all()), "interpolate wrote past out[batch·k)"
        assert bool((back[:3 * m] == F.view(-1)).all())


def test_refusals_before_any_launch():
    import torch
    c = ctx()
    xs, F = dev(_points(GL, 100, 14, distinct=True)), dev(oracle.splitmix(GL, 15, 300))
    out = torch.empty(300, dtype=torch.int64, device="cuda")
    far = [1 << 40, 1 << 44, 1 << 47]   # addresses never read: the checks refuse first
    cases = [
        ("ronk_poly_multieval_batch_u64", (GL, 7, None, 100, 3, _p(xs), 100, _p(out)), EINVAL),
        ("ronk_poly_multieval_batch_u64", (GL, 7, _p(F), 100, 3, None, 100, _p(out)), EINVAL),
        ("ronk_poly_multieval_batch_u64", (GL, GL, _p(F), 100, 3, _p(xs), 100, _p(out)), EINVAL),
        ("ronk_poly_multieval_batch_u64", (GL, 7, _p(F), 100, 3, _p(xs), 100, _p(F)), EINVAL),       # out over coeffs
        ("ronk_poly_multieval_batch_u64", (GL, 7, _p(F), 100, 3, _p(xs), 100, _p(xs)), EINVAL),      # out over xs
        ("ronk_poly_multieval_batch_u64", (GL, 7, _p(F), 100, 0, _p(xs), 100, _p(out)), 0),
        ("ronk_poly_multieval_batch_u64", (GL, 7, _p(F), 100, 3, _p(xs), 0, _p(out)), 0),
        ("ronk_poly_multieval_batch_u64", (GL, 7, far[0], 1, 3, far[1], (1 << 24) + 1, far[2]), EUNSUPPORTED),
        ("ronk_poly_multieval_batch_u64", (GL, 7, far[0], 1 << 16, 1 << 16, far[1], 1 << 16, far[2]), EUNSUPPORTED),
        ("ronk_poly_interpolate_batch_u64", (GL, 7, _p(xs), None, 100, 3, _p(out)), EINVAL),
        ("ronk_poly_interpolate_batch_u64", (GL, 7, _p(xs), _p(F), 100, 3, _p(F)), EINVAL),         # out over ys
        ("ronk_poly_interpolate_batch_u64", (GL, 7, _p(xs), _p(F), 100, 3, _p(xs)), EINVAL),        # out over xs
        ("ronk_poly_interpolate_batch_u64", (GL, 7, _p(xs), _p(F), 100, 0, _p(out)), 0),
        ("ronk_poly_interpolate_batch_u64", (GL, 7, far[0], far[1], (1 << 24) + 1, 1, far[2]), EUNSUPPORTED),
        ("ronk_poly_interpolate_batch_u64", (GL, 7, far[0], far[1], 1 << 20, 1 << 13, far[2]), EUNSUPPORTED),
        ("ronk_poly_interpolate_batch_u64", (GL, 0, far[0], far[1], 8192, 4096, far[2]), EUNSUPPORTED),  # partial sums
        ("ronk_poly_interpolate_batch_u64", (GL, 0, far[0], far[1], 8193, 1, far[2]), EUNSUPPORTED),
    ]
    for name, args, want in cases:
        rc, launches = _rc(c, name, *args)
        assert (rc, launches) == (want, 0), (name, args, rc, launches)


def test_host_twins():
    c = ctx()
    from ronkathon_b200 import ops
    for p, g, m in ((GL, 7, 5000), (GL, 7, 300), (101, 2, 50)):
        xs = _points(p, m, 16, distinct=True)
        F = oracle.splitmix(p, 17, 4 * m).reshape(4, m)
        want = host(ops.poly_multieval_batch(c, dev(F), dev(xs), p=p, g=g))
        got = np.empty((4, m), np.uint64)
        c.call("ronk_poly_multieval_batch_u64_host", p, g, _p(F), m, 4, _p(xs), m, _p(got))
        assert np.array_equal(got.reshape(-1), want.reshape(-1))
        back = np.empty((4, m), np.uint64)
        c.call("ronk_poly_interpolate_batch_u64_host", p, g, _p(xs), _p(got), m, 4, _p(back))
        assert np.array_equal(back, F)


def test_gated_non_blocking_stream():
    """multieval on a fresh context's non-blocking stream behind a spin: it returns before the stream runs, and its words
    are the default stream's."""
    import torch
    from ronkathon_b200 import Context, ops
    c0 = ctx()
    xs, F = _points(GL, 1 << 16, 18, distinct=True), oracle.splitmix(GL, 19, 3 << 16).reshape(3, 1 << 16)
    want = host(ops.poly_multieval_batch(c0, dev(F), dev(xs)))
    s = torch.cuda.Stream()
    c = Context(0, s.cuda_stream)
    try:
        X, Fd = dev(xs), dev(F)
        with torch.cuda.stream(s):
            ops.poly_multieval_batch(c, Fd, X)   # warm: plans and scratch
        s.synchronize()
        Xg, Fg = torch.zeros_like(X), torch.zeros_like(Fd)
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            torch.cuda._sleep(100_000_000)
            Xg.copy_(X)
            Fg.copy_(Fd)
            out = ops.poly_multieval_batch(c, Fg, Xg)
            assert not s.query(), "the stream finished before the call returned"
        s.synchronize()
        assert np.array_equal(ops.to_host(out), want)
    finally:
        c.close()


# ---- Shamir over batches of secrets -----------------------------------------------------------------------------------

def test_shamir_reference_cases():
    """shamir/mod.rs's tests on PlutoBaseField: (12, 3 of 5) from the first 3 shares, (98, 4 of 7) from all 7, and 42
    split 3 of 6 rebuilt from the subsets [0,2,4], [1,3,5], [0,1,2]."""
    from ronkathon_b200 import codes
    from ronkathon_b200.field import PlutoBaseField as F
    ctx()
    xs, ys = codes.shamir_split([F(12)], 3, 5, F)
    assert codes.shamir_combine(xs[:3], ys[:, :3], F) == [F(12)]
    xs, ys = codes.shamir_split([F(98)], 4, 7, F)
    assert codes.shamir_combine(xs, ys, F) == [F(98)]
    xs, ys = codes.shamir_split([F(42)], 3, 6, F)
    for idx in ([0, 2, 4], [1, 3, 5], [0, 1, 2]):
        assert codes.shamir_combine(xs[idx], ys[:, idx], F) == [F(42)]
    # the shares are the polynomial's values at 1..n, and the caller's coefficients are used as given
    xs, ys = codes.shamir_split([5, 6], 3, 4, F, coefficients=[[1, 2], [3, 4]])
    assert xs.tolist() == [1, 2, 3, 4]
    assert ys.tolist() == [[(5 + x + 2 * x * x) % 101 for x in range(1, 5)], [(6 + 3 * x + 4 * x * x) % 101 for x in range(1, 5)]]


def test_shamir_many_goldilocks_secrets():
    from ronkathon_b200 import codes
    from ronkathon_b200.field import GoldilocksField as F
    ctx()
    secrets = [int(v) for v in oracle.splitmix(GL, 60, 10000)]
    xs, ys = codes.shamir_split(secrets, 5, 9, F)
    assert ys.shape == (10000, 9)
    rng = random.Random(61)
    groups = {}
    for i in range(10000):
        groups.setdefault(tuple(sorted(rng.sample(range(9), 5))), []).append(i)
    for idx, rows in groups.items():
        got = codes.shamir_combine(xs[list(idx)], ys[rows][:, list(idx)], F)
        assert [v.value for v in got] == [secrets[r] for r in rows]
    # more shares than the threshold: the Lagrange sum at 0 over all of them
    assert [v.value for v in codes.shamir_combine(xs, ys[:50], F)] == secrets[:50]


def test_shamir_repeated_share_panics():
    from ronkathon_b200 import RonkPanic, codes
    from ronkathon_b200.field import PlutoBaseField as F
    ctx()
    xs, ys = codes.shamir_split([F(7)], 3, 5, F)
    with pytest.raises(RonkPanic):
        codes.shamir_combine([xs[0], xs[1], xs[1]], ys[:, [0, 1, 1]], F)
