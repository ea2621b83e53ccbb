"""ronk_rs_decode_at_u64[_host]: errors-and-erasures Reed–Solomon decoding at any n distinct points, and
codes.shamir_recover above it.

At x_i = ω_n^i in order every row of the structured corpus (tests/rs_corpus.py) must give ronk_rs_decode_u64's words,
beyond the radius too: both are complete bounded-distance decoders.  At random points and permuted roots of unity, rows
at the full radius must give their message and error count, and rows past it -1 with a zero message or a message
within the radius, checked by re-evaluation.  Every size runs on the suite's context and on one made with
RONK_TREE_MIN=1, which takes the subproduct tree wherever its transforms fit."""
import os
import random

import numpy as np
import pytest

import rs_corpus as rc
from gpu_util import GL, MONT_PRIMES, ctx, dev, host
from test_rs_decode_at_model import decode_at as model_decode_at

pytestmark = pytest.mark.gpu

EINVAL, EUNSUPPORTED = 1, 5
PRIMES = {**{k: (p, g) for k, (p, g, _) in MONT_PRIMES.items()}, "goldilocks": (GL, 7)}
_tree = None


def _ctx(kind):
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
    from ronkathon_b200 import _lib as L
    return L._ptr(x)


def _lib():
    from ronkathon_b200 import _lib as L
    return L.lib()


def decode_at(c, p, g, xs, rows, k, erased=None):
    """rows: batch × n host array → (batch × k messages, statuses), through ops.rs_decode_at"""
    import torch
    from ronkathon_b200 import ops
    rows = np.atleast_2d(np.asarray(rows, dtype=np.uint64))
    er = None if erased is None else torch.from_numpy(np.ascontiguousarray(erased, dtype=np.uint8).ravel()).cuda()
    msg, st = ops.rs_decode_at(c, dev(np.asarray(xs, dtype=np.uint64)), dev(rows.ravel()), k, er, rows.shape[0], p=p, g=g)
    return host(msg).reshape(rows.shape[0], k), st.cpu().numpy()


def decode_omega(c, p, g, rows, k, erased):
    import torch
    from ronkathon_b200 import ops
    er = torch.from_numpy(np.ascontiguousarray(erased, dtype=np.uint8).ravel()).cuda()
    msg, st = ops.rs_decode(c, dev(rows.ravel()), k, er, rows.shape[0], p=p, g=g)
    return host(msg).reshape(rows.shape[0], k), st.cpu().numpy()


def evaluate(c, p, g, msgs, xs):
    from ronkathon_b200 import ops
    return host(ops.poly_multieval_batch(c, dev(msgs), dev(np.asarray(xs, dtype=np.uint64)), p=p, g=g)).reshape(len(msgs), -1)


def check_bounded(c, p, g, xs, rows, erased, k, msgs, st):
    """Every row: -1 with a zero message, or a message whose evaluations differ from the row in exactly `status`
    non-erased positions, 2·status + ε ≤ n - k."""
    n = len(xs)
    er = np.asarray(erased, bool)
    dist = ((evaluate(c, p, g, msgs, xs) != rows) & ~er).sum(1)
    for r in range(len(rows)):
        if st[r] == -1:
            assert not msgs[r].any(), r
        else:
            assert 2 * st[r] + er[r].sum() <= n - k and dist[r] == st[r], (r, st[r], dist[r])


def roots_of_unity(p, g, n):
    w = pow(g, (p - 1) // n, p)
    return np.array([pow(w, i, p) for i in range(n)], dtype=np.uint64)


def _odd_factor(p):
    q = p - 1
    while q % 2 == 0:
        q //= 2
    return next(d for d in range(3, 1000, 2) if q % d == 0)


# ---- at ω_n^i: ronk_rs_decode_u64's words on the structured corpus -----------------------------------------------------

def _cells():
    out = []
    for name, (p, g) in PRIMES.items():
        if name == "p2adic3":
            out += [(name, 8, 4), (name, 8, 5)]
            continue
        out += [(name, 256, 33), (name, 256, 200), (name, _odd_factor(p) << 4, 40)]
    out += [("goldilocks", 4096, 1025), ("babybear", 3 << 10, 1500)]
    return out


CELLS = _cells()


@pytest.mark.parametrize("name,n,m", CELLS, ids=[f"{a}-n{b}-m{c}" for a, b, c in CELLS])
def test_corpus_at_roots_of_unity_equals_the_omega_decoder(name, n, m):
    p, g = PRIMES[name]
    assert (p - 1) % n == 0
    c = ctx()
    code = rc.Code(p, g, n, n - m)
    specs = rc.everything(code, np.random.default_rng([n, m, len(name)]))
    rows, erased, k, _ = rc.build(code, specs, _forward_device(c, code))
    want_msg, want_st = decode_omega(c, p, g, rows, k, erased)
    msg, st = decode_at(c, p, g, roots_of_unity(p, g, n), rows, k, erased)
    assert np.array_equal(st, want_st), np.nonzero(st != want_st)
    assert np.array_equal(msg, want_msg)
    assert (st == -1).any() and (st > 0).any()


def _forward_device(c, code):
    from ronkathon_b200 import ops
    return lambda Y: host(ops.rs_encode(c, dev(np.ascontiguousarray(Y).ravel()), code.n, len(Y), p=code.p, g=code.g)).reshape(len(Y), code.n)


# ---- random points: at the radius, past it, and the point 0 ------------------------------------------------------------

def _points(p, n, rng, zero_at=None):
    xs = rng.sample(range(1, min(p, 1 << 62)), n)
    if zero_at is not None:
        xs[zero_at] = 0
    return np.array(xs, dtype=np.uint64)


def _rows(p, xs, k, batch, rng, past=False, c=None, g=None):
    """batch rows with different errata patterns: ε erasures and e = (m - ε)/2 errors (one more when past); row 0 puts
    an error on position 0 and row 1 erases it.  Returns (msgs, rows, erased, errors)."""
    n = len(xs)
    m = n - k
    msgs = np.array([[rng.randrange(p) for _ in range(k)] for _ in range(batch)], dtype=np.uint64)
    rows = evaluate(c, p, g, msgs, xs)
    erased = np.zeros((batch, n), np.uint8)
    errors = np.zeros(batch, np.int64)
    for b in range(batch):
        eps = rng.randrange(0, m + 1) if b > 1 else (0 if b == 0 else min(1, m))
        er = rng.sample(range(1, n), eps) if b != 1 else ([0] if eps else [])
        e = min((m - eps) // 2 + (1 if past else 0), n - eps)
        live = [i for i in range(n) if i not in er]
        bad = ([0] + rng.sample(live[1:], e - 1) if e else []) if b == 0 else rng.sample(live, e)
        for i in er:
            erased[b, i] = 1 + rng.randrange(255)
            rows[b, i] = rng.randrange(p)
        for i in bad:
            rows[b, i] = (int(rows[b, i]) + 1 + rng.randrange(p - 1)) % p
        errors[b] = e
    return msgs, rows, erased, errors


FIELDS = ("goldilocks", "babybear", "pbig", "gl_g5")
SIZES = [(64, 32, 24), (300, 101, 12), (2048, 1000, 4)]      # n, m, batch
RANDOM = [(f, kind, n, m, b) for f in FIELDS for kind in ("default", "tree") for n, m, b in SIZES]


@pytest.mark.parametrize("name,kind,n,m,batch", RANDOM, ids=[f"{a}-{b}-n{c}-m{d}" for a, b, c, d, _ in RANDOM])
def test_random_points_at_and_past_the_radius(name, kind, n, m, batch):
    p, g = PRIMES[name]
    c = _ctx(kind)
    rng = random.Random(f"{name}{kind}{n}{m}")
    k = n - m
    xs = _points(p, n, rng, zero_at=0)
    msgs, rows, erased, errors = _rows(p, xs, k, batch, rng, c=c, g=g)
    got, st = decode_at(c, p, g, xs, rows, k, erased)
    assert np.array_equal(st, errors) and np.array_equal(got, msgs)
    _, rows, erased, _ = _rows(p, xs, k, batch, rng, past=True, c=c, g=g)
    got, st = decode_at(c, p, g, xs, rows, k, erased)
    check_bounded(c, p, g, xs, rows, erased, k, got, st)


@pytest.mark.parametrize("kind", ["default", "tree"])
def test_permuted_roots_of_unity(kind):
    p, g = GL, 7
    c = _ctx(kind)
    rng = random.Random(kind)
    n, k = 512, 300
    xs = roots_of_unity(p, g, n)[np.random.default_rng(5).permutation(n)]
    msgs, rows, erased, errors = _rows(p, xs, k, 16, rng, c=c, g=g)
    got, st = decode_at(c, p, g, xs, rows, k, erased)
    assert np.array_equal(st, errors) and np.array_equal(got, msgs)


def test_matches_the_model_word_for_word():
    """Small rows at every distance on a Montgomery prime, 0 among the points: the Python model's words."""
    p, g = PRIMES["babybear"]
    c = ctx()
    rng = random.Random(3)
    n, k = 24, 9
    xs = _points(p, n, rng, zero_at=5)
    rows = np.array([[rng.randrange(p) for _ in range(n)] for _ in range(6)], dtype=np.uint64)
    msgs, near, erased, _ = _rows(p, xs, k, 10, rng, past=True, c=c, g=g)
    rows = np.concatenate([rows, near])
    erased = np.concatenate([np.zeros((6, n), np.uint8), erased])
    got, st = decode_at(c, p, g, xs, rows, k, erased)
    for r in range(len(rows)):
        want, want_st = model_decode_at(p, [int(x) for x in xs], [int(v) for v in rows[r]], list(erased[r]), k)
        assert st[r] == want_st and got[r].tolist() == (want if want is not None else [0] * k), r


def test_more_than_8192_points_on_the_tree():
    p, g = GL, 7
    c = ctx()
    rng = random.Random(9)
    n, k = 16384, 16384 - 64
    xs = _points(p, n, rng)
    msgs, rows, erased, errors = _rows(p, xs, k, 2, rng, c=c, g=g)
    got, st = decode_at(c, p, g, xs, rows, k, erased)
    assert np.array_equal(st, errors) and np.array_equal(got, msgs)
    m_ = np.zeros(2 * k, np.uint64)
    s_ = np.zeros(2, np.int32)
    rc_ = _lib().ronk_rs_decode_at_u64_host(c._h, p, 0, _p(xs), _p(rows), None, n, k, 2, _p(m_), _p(s_))
    assert rc_ == EUNSUPPORTED          # g = 0: the literal interpolation stops at 8192 points


# ---- edges, errors and the host twin -----------------------------------------------------------------------------------

def _call(c, entry, p, g, xs, rows, erased, n, k, batch, msg, st):
    return getattr(_lib(), entry)(c._h, p, g, _p(xs), _p(rows), _p(erased) if erased is not None else None, n, k, batch,
                                   _p(msg), _p(st))


def test_edges():
    p, g = GL, 7
    c = ctx()
    rng = random.Random(11)
    # m = 0: the interpolant, status 0; an erasure is refused
    xs = _points(p, 40, rng, zero_at=3)
    msgs = np.array([[rng.randrange(p) for _ in range(40)] for _ in range(3)], dtype=np.uint64)
    rows = evaluate(c, p, g, msgs, xs)
    er = np.zeros((3, 40), np.uint8)
    er[2, 7] = 1
    got, st = decode_at(c, p, g, xs, rows, 40, er)
    assert st.tolist() == [0, 0, -1] and np.array_equal(got[:2], msgs[:2]) and not got[2].any()
    # m = 8191 at the cap, erased = NULL
    n, k = 8192, 1
    xs = _points(p, n, rng)
    msgs = np.array([[rng.randrange(p)] for _ in range(2)], dtype=np.uint64)
    rows = evaluate(c, p, g, msgs, xs)
    for b in range(2):
        for i in rng.sample(range(n), 4095):
            rows[b, i] = (int(rows[b, i]) + 1) % p
    got, st = decode_at(c, p, g, xs, rows, k)
    assert st.tolist() == [4095, 4095] and np.array_equal(got, msgs)
    m_, s_ = np.zeros(4, np.uint64), np.zeros(2, np.int32)
    assert _call(c, "ronk_rs_decode_at_u64_host", p, g, np.arange(1, 8194, dtype=np.uint64), np.zeros(2 * 8193, np.uint64),
                 None, 8193, 1, 2, m_, s_) == EUNSUPPORTED                   # m = 8192
    # batch 0 writes nothing
    assert _call(c, "ronk_rs_decode_at_u64_host", p, g, xs, rows, None, n, k, 0, m_, s_) == 0


def test_refused_calls_write_nothing():
    import torch
    p, g = GL, 7
    c = ctx()
    rng = random.Random(12)
    n, k, b = 64, 20, 3
    xs = _points(p, n, rng)
    _, rows, erased, _ = _rows(p, xs, k, b, rng, c=c, g=g)
    bad_xs = xs.copy()
    bad_xs[9] = bad_xs[40]
    for host_twin in (False, True):
        if host_twin:
            X, R, E = bad_xs, rows, erased
            msg, st = np.full(b * k, 0x5A5A, np.uint64), np.full(b, 0x5A5A, np.int32)
            entry = "ronk_rs_decode_at_u64_host"
        else:
            X, R, E = dev(bad_xs), dev(rows.ravel()), torch.from_numpy(erased.ravel()).cuda()
            msg, st = dev(np.full(b * k, 0x5A5A, np.uint64)), torch.full((b,), 0x5A5A, dtype=torch.int32, device="cuda")
            entry = "ronk_rs_decode_at_u64"
        assert _call(c, entry, p, g, X, R, E, n, k, b, msg, st) == EINVAL          # a repeated point
        c.sync()
        mh = msg if host_twin else msg.cpu().numpy()
        sh = st if host_twin else st.cpu().numpy()
        assert (np.asarray(mh).view(np.uint64) == 0x5A5A).all() and (sh == 0x5A5A).all()
    # errors in the documented order, on host pointers
    m_, s_ = np.zeros(b * k, np.uint64), np.zeros(b, np.int32)
    assert _call(c, "ronk_rs_decode_at_u64_host", p, g, None, rows, None, n, k, b, m_, s_) == EINVAL
    assert _call(c, "ronk_rs_decode_at_u64_host", p, p, xs, rows, None, n, k, b, m_, s_) == EINVAL      # g >= p
    assert _call(c, "ronk_rs_decode_at_u64_host", p, g, xs, rows, None, 0, k, b, m_, s_) == EINVAL
    assert _call(c, "ronk_rs_decode_at_u64_host", p, g, xs, rows, None, n, 0, b, m_, s_) == EINVAL
    assert _call(c, "ronk_rs_decode_at_u64_host", p, g, xs, rows, None, n, n + 1, b, m_, s_) == EINVAL
    big = xs.copy()
    big[3] = p
    assert _call(c, "ronk_rs_decode_at_u64_host", p, g, big, rows, None, n, k, b, m_, s_) == EINVAL      # x >= p
    # overlaps: msg over received, status over msg
    R = dev(rows.ravel())
    X = dev(xs)
    assert _lib().ronk_rs_decode_at_u64(c._h, p, g, _p(X), _p(R), None, n, k, b, _p(R), _p(R[b * k:])) == EINVAL
    S = dev(np.zeros(b * k, np.uint64))
    assert _lib().ronk_rs_decode_at_u64(c._h, p, g, _p(X), _p(R), None, n, k, b, _p(S), _p(S)) == EINVAL
    assert _lib().ronk_rs_decode_at_u64(c._h, p, g, _p(X), _p(R), None, n, k, b, _p(X), _p(S)) == EINVAL


def test_host_twin_equals_device_and_erased_values_are_never_read():
    p, g = PRIMES["pbig"]
    c = ctx()
    rng = random.Random(13)
    n, k, b = 200, 80, 8
    xs = _points(p, n, rng, zero_at=0)
    _, rows, erased, _ = _rows(p, xs, k, b, rng, c=c, g=g)
    got, st = decode_at(c, p, g, xs, rows, k, erased)
    m_, s_ = np.zeros(b * k, np.uint64), np.zeros(b, np.int32)
    assert _call(c, "ronk_rs_decode_at_u64_host", p, g, xs, rows, erased, n, k, b, m_, s_) == 0
    assert np.array_equal(m_.reshape(b, k), got) and np.array_equal(s_, st)
    for poison in (0, p - 1, p, (1 << 64) - 1):                       # non-canonical values too
        r2 = rows.copy()
        r2[erased != 0] = poison
        g2, s2 = decode_at(c, p, g, xs, r2, k, erased)
        assert np.array_equal(g2, got) and np.array_equal(s2, st)


def _names(c, fn):
    c.sync()
    c.prof_fetch()
    c.prof_enable(True)
    try:
        fn()
        c.sync()
    finally:
        c.prof_enable(False)
    return [nm for nm, _ in c.prof_fetch()]


@pytest.mark.parametrize("kind,n,m,g0", [("default", 64, 20, False), ("default", 96, 30, True), ("tree", 1024, 300, False)])
def test_launch_sequence_does_not_depend_on_the_batch(kind, n, m, g0):
    p, g = GL, 7
    c = _ctx(kind)
    rng = random.Random(14)
    xs = _points(p, n, rng, zero_at=1)
    seqs = []
    for b in (2, 7):
        _, rows, erased, _ = _rows(p, xs, n - m, b, rng, c=c, g=g)
        seqs.append(_names(c, lambda: decode_at(c, p, 0 if g0 else g, xs, rows, n - m, erased)))
    assert seqs[0] == seqs[1]
    assert {"rs_mask", "rs_locator_at", "rs_forney", "rs_finish"} <= set(seqs[0])


def test_gated_non_blocking_stream():
    import torch
    from ronkathon_b200 import Context, ops
    p, g = GL, 7
    c0 = ctx()
    rng = random.Random(15)
    n, k, b = 256, 100, 16
    xs = _points(p, n, rng)
    msgs, rows, erased, errors = _rows(p, xs, k, b, rng, c=c0, g=g)
    s = torch.cuda.Stream()
    c = Context(0, s.cuda_stream)
    try:
        X, R, E = dev(xs), dev(rows.ravel()), torch.from_numpy(erased.ravel()).cuda()
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            torch.cuda._sleep(50_000_000)
            Xg, Rg = X.clone(), R.clone()
            msg, st = ops.rs_decode_at(c, Xg, Rg, k, E, b, p=p, g=g)
        s.synchronize()
        assert np.array_equal(ops.to_host(msg).reshape(b, k), msgs) and np.array_equal(st.cpu().numpy(), errors)
    finally:
        c.close()


# ---- Shamir recovery ---------------------------------------------------------------------------------------------------

def test_shamir_recover():
    """256 secrets, 64 shares, threshold 20: up to 22 wrong shares and some missing ones per row (2e + ε ≤ 44) come back
    exactly with their error counts; a row one wrong share past the radius is None."""
    from ronkathon_b200 import codes
    from ronkathon_b200.field import GoldilocksField as F
    ctx()
    rng = random.Random(16)
    n, t, batch = 64, 20, 256
    secrets = [rng.randrange(GL) for _ in range(batch)]
    xs, ys = codes.shamir_split(secrets, t, n, F)
    missing = np.zeros((batch, n), bool)
    want = []
    for b in range(batch):
        eps = rng.randrange(0, 11) if b % 3 else 0
        gone = rng.sample(range(n), eps)
        missing[b, gone] = True
        e = (44 - eps) // 2 if b % 2 else rng.randrange((44 - eps) // 2 + 1)
        for i in rng.sample([i for i in range(n) if i not in gone], e):
            ys[b, i] = (int(ys[b, i]) + 1 + rng.randrange(GL - 1)) % GL
        for i in gone:
            ys[b, i] = rng.randrange(GL)
        want.append(e)
    got, errs = codes.shamir_recover(xs, ys, t, F, missing=missing)
    assert [int(v.value) for v in got] == secrets and errs == want
    row = ys[:1].copy()
    for i in range(23):                                          # 23 wrong shares: past (64 - 20) / 2
        row[0, i] = (int(row[0, i]) + 1) % GL
    got, errs = codes.shamir_recover(xs, row, t, F)
    assert got == [None] and errs == [-1]
