"""Lagrange-basis rows on a coset evaluated at many points (ronk_poly_lagrange_eval_u64) and opened at one point
(ronk_poly_lagrange_open_u64) on the device, bit-exact:

* every test prime, Goldilocks with g = 7, F_101 and F_17, at n = 1, 2, 3, 255, 256, 257, powers of two and 3·2^k wherever
  they divide p - 1, batch 1, 3 and 1024, m = 1, 2, 17 and 300, shift 1 and seeded shifts, points 0, 1, p - 1, s and the
  nodes j = 0, 1 and n - 1, against the Python-integer model (tests/lagrange_model.py);
* shift 1 against the single-point ronk_poly_lagrange_eval_u64_host, word for word, up to 2^14;
* Goldilocks at 2^20 and 2^24 and BabyBear at 2^20 against an independent device route: the inverse coset transform,
  then ronk_poly_eval_u64;
* openings: values, the quotient against the model, the quotient's top coefficient, q(r)·(r - z) = f(r) - f(z), and
  kzg.open_lagrange against kzg.open_ for every z in F_17;
* refused calls that write nothing, guard words, launch records, the host twins and a gated non-blocking stream."""
import ctypes as C
import random

import numpy as np
import pytest

import lagrange_model as lm
import oracle
from gpu_util import GL, MONT_PRIMES, ctx, dev, host

pytestmark = pytest.mark.gpu

POISON = -1
FRONT = 16
FIELDS = {"gl": (GL, 7), "f101": (101, 2), "f17": (17, 3), **{k: v[:2] for k, v in MONT_PRIMES.items()}}

_ctx = None


@pytest.fixture(scope="module", autouse=True)
def _module_context():
    """The module runs on a context of its own, destroyed at the end with torch's cached memory returned: the 2^24-point
    rows and their partial sums should not stay on the suite's shared context."""
    global _ctx
    import torch
    from ronkathon_b200 import Context
    ctx()
    _ctx = Context(0, torch.cuda.current_stream().cuda_stream)
    try:
        yield
    finally:
        _ctx.close()
        _ctx = None
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


def _c():
    return _ctx


def order_ok(p, g, n):
    w = pow(g, (p - 1) // n, p)
    return all(pow(w, n // q, p) != 1 for q in range(2, n + 1) if n % q == 0 and all(q % r for r in range(2, q)))


def sizes(name):
    p, g = FIELDS[name]
    cand = [1, 2, 3, 4, 255, 256, 257, 1 << 12, 48, 3 << 10]
    return [n for n in cand if (p - 1) % n == 0 and order_ok(p, g, n)]


GRID = [(name, n) for name in FIELDS for n in sizes(name)]


def shifts(p, seed):
    return [1, random.Random(seed).randrange(2, p)]


def edge_points(p, g, n, s, seed, count):
    xs = lm.nodes(p, g, n, s)
    pts = [0, 1, p - 1, s, xs[0], xs[min(1, n - 1)], xs[-1]]
    rng = random.Random(seed)
    while len(pts) < count:
        pts.append(rng.randrange(p))
    return pts[:count]


def model_eval(p, g, rows, xs, s):
    """out[b][i] = L_b(xs[i]) by the model, one weight vector per point."""
    n = len(rows[0])
    nd = lm.nodes(p, g, n, s)
    sn = pow(s, n, p)
    inv_nsn = pow(n * sn % p, -1, p)
    out = [[0] * len(xs) for _ in rows]
    for i, x in enumerate(xs):
        zx = (pow(x, n, p) - sn) % p
        if zx == 0:
            continue
        c = [xj * pow((x - xj) % p, -1, p) % p for xj in nd]
        for b, r in enumerate(rows):
            out[b][i] = zx * inv_nsn % p * (sum(int(y) * cj for y, cj in zip(r, c)) % p) % p
    return out


def eval_dev(rows, xs, n, s, p, g):
    from ronkathon_b200 import ops
    return ops.lagrange_eval(_c(), rows, xs, n, shift=s, p=p, g=g)


def open_dev(rows, z, n, s, p, g):
    from ronkathon_b200 import ops
    return ops.lagrange_open(_c(), rows, z, n, shift=s, p=p, g=g)


def rows_of(p, batch, n, seed):
    return oracle.splitmix(p, seed, batch * n).reshape(batch, n)


# ---- evaluation against the model ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,n", GRID, ids=[f"{a}-{b}" for a, b in GRID])
def test_eval_words(name, n):
    p, g = FIELDS[name]
    m = 17 if n <= 257 else 2
    for batch in (1, 3):
        for s in shifts(p, n):
            rows = rows_of(p, batch, n, n + batch)
            xs = edge_points(p, g, n, s, n * 7 + batch, m)
            got = host(eval_dev(dev(rows), dev(np.array(xs, dtype=np.uint64)), n, s, p, g)).reshape(batch, m)
            assert got.tolist() == model_eval(p, g, rows.tolist(), xs, s), (batch, s)


@pytest.mark.parametrize("name", ["gl", "babybear", "pbig", "f101", "f17"])
@pytest.mark.parametrize("m", [1, 2, 17, 300])
def test_eval_many_rows_and_points(name, m):
    """batch 1024 × n = 4 at m = 1, 2, 17 and 300: past one warp of rows per CTA and past one group of 8 points."""
    p, g = FIELDS[name]
    n, batch = 4, 1024
    s = shifts(p, m)[1]
    rows = rows_of(p, batch, n, m)
    xs = edge_points(p, g, n, s, m, m)
    got = host(eval_dev(dev(rows), dev(np.array(xs, dtype=np.uint64)), n, s, p, g)).reshape(batch, m)
    assert got.tolist() == model_eval(p, g, rows.tolist(), xs, s)


@pytest.mark.parametrize("name", ["gl", "babybear", "p57", "f101", "f17"])
def test_eval_shift_one_equals_the_single_point_host_entry(name):
    """With s = 1 every word is the one ronk_poly_lagrange_eval_u64_host (the O(n²) literal kernel) gives."""
    p, g = FIELDS[name]
    for n in [n for n in (1, 2, 3, 4, 5, 255, 256, 257, 1024, 1 << 14) if (p - 1) % n == 0 and order_ok(p, g, n)]:
        rows = rows_of(p, 2, n, n)
        xs = edge_points(p, g, n, 1, n, 6 if n < 4096 else 3)
        got = host(eval_dev(dev(rows), dev(np.array(xs, dtype=np.uint64)), n, 1, p, g)).reshape(2, -1)
        for b in range(2):
            for i, x in enumerate(xs):
                res = C.c_uint64()
                _c().call("ronk_poly_lagrange_eval_u64_host", p, g, rows[b].ctypes.data_as(C.c_void_p), n, x, C.byref(res))
                assert int(got[b][i]) == res.value, (n, b, x)


LARGE = [("gl", 20, 4), ("gl", 24, 4), ("babybear", 20, 4), ("pbig", 16, 3), ("gl", 12, 5)]


def transform_route(rows_t, log_n, batch, s, xs_t, p, g):
    """Independent device route: coefficients by the inverse coset transform, then ronk_poly_eval_u64 per row."""
    from ronkathon_b200 import ops
    coeffs = rows_t.clone().view(-1)
    ops.ntt_coset_(_c(), coeffs, log_n, s, batch=batch, inverse=True, p=p, g=g)
    coeffs = coeffs.view(batch, -1)
    return [host(ops.poly_eval(_c(), coeffs[b].contiguous(), xs_t, p=p)) for b in range(batch)], coeffs


@pytest.mark.parametrize("name,log_n,batch", LARGE, ids=[f"{a}-2^{b}x{c}" for a, b, c in LARGE])
def test_eval_large_against_the_transform_route(name, log_n, batch):
    from ronkathon_b200 import ops
    p, g = FIELDS[name]
    n = 1 << log_n
    rows = ops.splitmix_fill(_c(), batch * n, log_n, p).view(batch, n)
    for s in shifts(p, log_n):
        w = pow(g, (p - 1) // n, p)
        nd = [s, s * w % p]
        rng = random.Random(log_n * 3 + s % 1000)
        xs = [0, 1, p - 1] + [rng.randrange(p) for _ in range(5)]
        xs = [x for x in xs if pow(x, n, p) != pow(s, n, p)]   # off the nodes, where the route gives f(x)
        xs_t = dev(np.array(xs + [nd[0], nd[1]], dtype=np.uint64))
        got = host(eval_dev(rows, xs_t, n, s, p, g)).reshape(batch, -1)
        want, _ = transform_route(rows, log_n, batch, s, dev(np.array(xs, dtype=np.uint64)), p, g)
        for b in range(batch):
            assert got[b][:len(xs)].tolist() == want[b].tolist(), (b, s)
            assert got[b][len(xs):].tolist() == [0, 0]   # the nodes x_0, x_1


# ---- opening ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,n", GRID, ids=[f"{a}-{b}" for a, b in GRID])
def test_open_words(name, n):
    p, g = FIELDS[name]
    if n > 257:
        pytest.skip("the model's quotient is checked up to 257 nodes; larger n in test_open_large")
    for batch in (1, 3):
        for s in shifts(p, n + 1):
            rows = rows_of(p, batch, n, n + 100 + batch)
            nd = lm.nodes(p, g, n, s)
            zs = sorted({0, 1, p - 1, random.Random(n).randrange(p), nd[0], nd[min(1, n - 1)], nd[-1]})
            for z in zs:
                v, q = open_dev(dev(rows), z, n, s, p, g)
                v, q = host(v), host(q).reshape(batch, n)
                for b in range(batch):
                    wv, wq = lm.quotient(p, g, rows[b].tolist(), z, s)
                    assert int(v[b]) == wv and q[b].tolist() == wq, (batch, s, z, b)


@pytest.mark.parametrize("name", ["gl", "babybear", "f17"])
def test_open_many_rows(name):
    p, g = FIELDS[name]
    n, batch = 8 if name != "f17" else 4, 1024
    rows = rows_of(p, batch, n, 77)
    s = shifts(p, 5)[1]
    for z in (lm.nodes(p, g, n, s)[n - 1], 12345 % p):
        v, q = open_dev(dev(rows), z, n, s, p, g)
        v, q = host(v), host(q).reshape(batch, n)
        for b in range(0, batch, 37):
            wv, wq = lm.quotient(p, g, rows[b].tolist(), z, s)
            assert int(v[b]) == wv and q[b].tolist() == wq, (z, b)


OPEN_LARGE = [("gl", 12, 3), ("gl", 16, 2), ("gl", 20, 4), ("gl", 24, 2), ("babybear", 20, 4), ("pbig", 14, 2),
              ("koalabear", 13, 1)]


@pytest.mark.parametrize("name,log_n,batch", OPEN_LARGE, ids=[f"{a}-2^{b}x{c}" for a, b, c in OPEN_LARGE])
def test_open_large(name, log_n, batch):
    """Off and on the nodes: values against the evaluation (off) or the row's word (on); the quotient's inverse
    transform ends in a zero; and at a random r, q(r)·(r - z) = f(r) - f(z)."""
    import torch
    from ronkathon_b200 import ops
    p, g = FIELDS[name]
    n = 1 << log_n
    rows = ops.splitmix_fill(_c(), batch * n, log_n + 50, p).view(batch, n)
    s = shifts(p, log_n)[1]
    k = n - 1 - 5 % n
    xk = s * pow(pow(g, (p - 1) // n, p), k, p) % p
    r = next(x for x in range(random.Random(log_n + 7).randrange(2, p // 2), p) if pow(x, n, p) != pow(s, n, p))
    z_off = next(z for z in range(12345, p) if pow(z, n, p) != pow(s, n, p))
    for z, on in ((z_off, False), (xk, True)):
        v, q = open_dev(rows, z, n, s, p, g)
        hv = host(v)
        if on:
            assert hv.tolist() == host(rows[:, k].contiguous()).tolist()
        else:
            assert hv.tolist() == host(eval_dev(rows, dev(np.array([z], dtype=np.uint64)), n, s, p, g)).reshape(-1).tolist()
        coeffs = q.clone().view(-1)
        ops.ntt_coset_(_c(), coeffs, log_n, s, batch=batch, inverse=True, p=p, g=g)
        assert (coeffs.view(batch, n)[:, -1] == 0).all(), "the quotient has degree ≤ n - 2"
        fr = host(eval_dev(rows, dev(np.array([r], dtype=np.uint64)), n, s, p, g)).reshape(-1)
        qr = host(eval_dev(q, dev(np.array([r], dtype=np.uint64)), n, s, p, g)).reshape(-1)
        for b in range(batch):
            assert int(qr[b]) * ((r - z) % p) % p == (int(fr[b]) - int(hv[b])) % p, (on, b)
        del coeffs
    torch.cuda.synchronize()


def srs(n):
    from ronkathon_b200.curve import G1_GENERATOR
    from ronkathon_b200.field import PlutoScalarField
    return [G1_GENERATOR * PlutoScalarField(2).pow(i) for i in range(n)]


@pytest.mark.parametrize("n", [4, 8, 16])
def test_kzg_open_lagrange_equals_open(n):
    from ronkathon_b200 import kzg
    from ronkathon_b200.field import PlutoScalarField
    from ronkathon_b200.polynomial import Lagrange, Polynomial
    g1 = srs(n)
    rng = random.Random(n)
    coeffs = [rng.randrange(17) for _ in range(n)]
    evals = Polynomial(coeffs, PlutoScalarField).fft()
    assert evals.basis is Lagrange
    for z in range(17):
        assert kzg.open_lagrange(evals, z, g1) == kzg.open_(coeffs, z, g1), z


def test_reference_kzg_opening_kat():
    """kzg/tests.rs:157-181 through the Lagrange route: z = 4 = ω_4^3 is a node."""
    from ronkathon_b200 import kzg
    from ronkathon_b200.curve import AffinePoint
    from ronkathon_b200.field import PlutoScalarField
    from ronkathon_b200.polynomial import Polynomial
    g1, _ = kzg.setup()
    evals = Polynomial([11, 11, 11, 1], PlutoScalarField).fft()
    assert kzg.open_lagrange(evals, PlutoScalarField(4), g1) == AffinePoint(bytes([26, 0, 45, 0]))


def test_polynomial_evaluate_many_in_the_lagrange_basis():
    from ronkathon_b200.field import PlutoBaseField
    from ronkathon_b200.polynomial import Lagrange, Polynomial
    poly = Polynomial([5, 17, 3, 99, 0, 42, 1, 7, 64, 2], PlutoBaseField, Lagrange)   # n = 10 divides 100
    xs = list(range(101))
    assert [v.value for v in poly.evaluate_many(xs)] == [poly.evaluate(x).value for x in xs]


# ---- refused calls, guard words, launch records, host twins, streams -----------------------------------------------------
def arena(words):
    import torch
    return torch.full((FRONT + words + FRONT,), POISON, dtype=torch.int64, device="cuda")


def test_refused_calls_write_nothing():
    import torch
    from ronkathon_b200 import _lib
    lib, h = _lib.lib(), _c()._h
    n = 256
    rows = dev(rows_of(GL, 2, n, 1))
    xs = dev(np.array([3, 5, 7], dtype=np.uint64))
    out = arena(4 * n)
    snap_r, snap_x, snap_o = rows.clone(), xs.clone(), out.clone()
    R, X, O = rows.data_ptr(), xs.data_ptr(), out.data_ptr() + 8 * FRONT
    EI, EU = _lib.EINVAL, _lib.EUNSUPPORTED
    ev, op = lib.ronk_poly_lagrange_eval_u64, lib.ronk_poly_lagrange_open_u64
    g49 = 49   # a square: ω = 49^((p-1)/n) has order n/2 for even n
    cases = [
        (ev, (h, GL, 7, None, n, 2, 1, X, 3, O), EI),                 # null evals
        (ev, (h, GL, 7, R, n, 2, 1, None, 3, O), EI),                 # null xs
        (ev, (h, GL, 7, R, n, 2, 1, X, 3, None), EI),                 # null out
        (ev, (h, 2, 1, R, 1, 2, 1, X, 3, O), EU),                     # p = 2
        (ev, (h, 100, 3, R, 1, 2, 1, X, 3, O), EI),                   # not a prime
        (ev, (h, GL, 0, R, n, 2, 1, X, 3, O), EI),                    # g = 0
        (ev, (h, GL, GL, R, n, 2, 1, X, 3, O), EI),                   # g = p
        (ev, (h, GL, 7, R, 0, 2, 1, X, 3, O), EI),                    # n = 0
        (ev, (h, GL, 7, R, 7, 2, 1, X, 3, O), EI),                    # 7 does not divide p - 1
        (ev, (h, 101, 2, R, 3, 2, 1, X, 3, O), EI),                   # 3 does not divide 100
        (ev, (h, GL, g49, R, n, 2, 1, X, 3, O), EI),                  # ω of order n/2: two nodes coincide
        (ev, (h, 101, 4, R, 4, 2, 1, X, 3, O), EI),                   # 4 = 2^2 in F_101: ω_4 of order 2
        (ev, (h, GL, 7, R, n, 2, 0, X, 3, O), EI),                    # shift 0
        (ev, (h, GL, 7, R, n, 2, GL, X, 3, O), EI),                   # shift p
        (ev, (h, GL, 7, R, 1 << 20, 4097, 1, X, 3, O), EU),           # batch·n > 2^32
        (ev, (h, GL, 7, R, n, 1 << 20, 1, X, 1 << 13, O), EU),        # batch·m > 2^32 (batch·n = 2^28)
        (ev, (h, GL, 7, R, n, 2, 1, X, 3, R + 8), EI),                # out overlaps evals
        (ev, (h, GL, 7, R, n, 2, 1, X, 3, X + 16), EI),               # out overlaps xs
        (op, (h, GL, 7, None, n, 2, 1, 5, O, O + 64), EI),            # null evals
        (op, (h, GL, 7, R, n, 2, 1, 5, None, O + 64), EI),            # null values
        (op, (h, GL, 7, R, n, 2, 1, 5, O, None), EI),                 # null quotient
        (op, (h, 2, 1, R, 1, 2, 1, 0, O, O + 64), EU),                # p = 2
        (op, (h, GL, 0, R, n, 2, 1, 5, O, O + 64), EI),               # g = 0
        (op, (h, GL, 7, R, 0, 2, 1, 5, O, O + 64), EI),               # n = 0
        (op, (h, GL, 7, R, 7, 2, 1, 5, O, O + 64), EI),               # 7 does not divide p - 1
        (op, (h, GL, g49, R, n, 2, 1, 5, O, O + 64), EI),             # ω of order n/2
        (op, (h, GL, 7, R, n, 2, 0, 5, O, O + 64), EI),               # shift 0
        (op, (h, GL, 7, R, n, 2, GL + 3, 5, O, O + 64), EI),          # shift > p
        (op, (h, GL, 7, R, n, 2, 1, GL, O, O + 64), EI),              # z = p
        (op, (h, GL, 7, R, 1 << 24, 257, 1, 5, O, O + 64), EU),       # batch·n > 2^32
        (op, (h, GL, 7, R, n, 2, 1, 5, R + 8, O), EI),                # values overlap evals
        (op, (h, GL, 7, R, n, 2, 1, 5, O, R + 16), EI),               # quotient overlaps evals
        (op, (h, GL, 7, R, n, 2, 1, 5, O + 8 * 100, O), EI),          # values overlap quotient
    ]
    for fn, args, code in cases:
        assert fn(*args) == code, (fn.__name__, args[1:])
        _c().sync()
        assert torch.equal(rows, snap_r) and torch.equal(xs, snap_x) and torch.equal(out, snap_o), (fn.__name__, args[1:])
    # batch 0 or m 0 does nothing
    assert ev(h, GL, 7, R, n, 0, 1, X, 3, O) == 0 and ev(h, GL, 7, R, n, 2, 1, X, 0, O) == 0
    assert op(h, GL, 7, R, n, 0, 1, 5, O, O + 64) == 0
    _c().sync()
    assert torch.equal(out, snap_o)


GUARDS = [("gl", 256, 3, 5), ("gl", 5120, 2, 9), ("babybear", 4096, 3, 3), ("f101", 100, 7, 2), ("pbig", 3, 9, 11)]


@pytest.mark.parametrize("name,n,batch,m", GUARDS, ids=[f"{a}-{b}x{c}-m{d}" for a, b, c, d in GUARDS])
def test_guard_words(name, n, batch, m):
    """Outputs inside poisoned arenas at an odd word offset: nothing outside them moves, inputs are left as they were."""
    import torch
    from ronkathon_b200 import _lib
    p, g = FIELDS[name]
    if (p - 1) % n:
        n = 4
    rows = dev(rows_of(p, batch, n, 3))
    xs = dev(np.array(edge_points(p, g, n, 1, 4, m), dtype=np.uint64))
    snap_r = rows.clone()
    out = arena(batch * m + 1)
    oview = out[FRONT + 1:FRONT + 1 + batch * m]
    _c().call("ronk_poly_lagrange_eval_u64", p, g, rows.data_ptr(), n, batch, 1, xs.data_ptr(), m, oview.data_ptr())
    _c().sync()
    assert (out[:FRONT + 1] == POISON).all() and (out[FRONT + 1 + batch * m:] == POISON).all()
    assert torch.equal(oview, eval_dev(rows, xs, n, 1, p, g).view(-1))
    nd = lm.nodes(p, g, n, 1)
    for z in (nd[-1], 2 if n > 2 else p - 2):
        vbuf, qbuf = arena(batch + 1), arena(batch * n + 1)
        vview, qview = vbuf[FRONT + 1:FRONT + 1 + batch], qbuf[FRONT + 1:FRONT + 1 + batch * n]
        _c().call("ronk_poly_lagrange_open_u64", p, g, rows.data_ptr(), n, batch, 1, z, vview.data_ptr(), qview.data_ptr())
        _c().sync()
        for buf, ln in ((vbuf, batch), (qbuf, batch * n)):
            assert (buf[:FRONT + 1] == POISON).all() and (buf[FRONT + 1 + ln:] == POISON).all(), z
        v, q = open_dev(rows, z, n, 1, p, g)
        assert torch.equal(vview, v) and torch.equal(qview, q.view(-1))
    assert torch.equal(rows, snap_r)
    assert _lib.OK == 0


def launch_names(c, fn):
    c.sync()
    c.prof_enable(True)
    try:
        fn()
        return [n for n, _ in c.prof_fetch()]
    finally:
        c.prof_enable(False)


EVAL_REC = ["lagrange_table", "lagrange_partial", "lagrange_finish"]
OFF_REC = ["lagrange_table", "lagrange_partial", "lagrange_finish", "lagrange_quotient"]
ON_REC = ["lagrange_table", "lagrange_locate", "lagrange_quotient", "lagrange_partial", "lagrange_finish"]


@pytest.mark.parametrize("name,n", [("gl", 1 << 20), ("gl", 3), ("babybear", 4096), ("f17", 16)])
def test_launch_records(name, n):
    """The sequence depends on (p, g, n, shift) and, for open, on whether z is a node; not on batch or m."""
    p, g = FIELDS[name]
    s = 3 % p
    nd = lm.nodes(p, g, n, s)
    for batch, m in ((1, 1), (3, 300)):
        rows = dev(rows_of(p, batch, n, 5))
        xs = dev(np.array(edge_points(p, g, n, s, 6, m), dtype=np.uint64))
        c0 = _c().launches
        assert launch_names(_c(), lambda: eval_dev(rows, xs, n, s, p, g)) == EVAL_REC
        z_off = next(z for z in range(p) if pow(z, n, p) != pow(s, n, p))
        assert launch_names(_c(), lambda: open_dev(rows, z_off, n, s, p, g)) == OFF_REC
        assert launch_names(_c(), lambda: open_dev(rows, nd[n // 2], n, s, p, g)) == ON_REC
        assert _c().launches - c0 == len(EVAL_REC) + len(OFF_REC) + len(ON_REC)


@pytest.mark.parametrize("name,n,batch", [("gl", 1024, 3), ("babybear", 48, 2), ("f101", 20, 5)])
def test_host_twins_equal_device(name, n, batch):
    from ronkathon_b200 import _lib
    p, g = FIELDS[name]
    s = shifts(p, n)[1]
    rows = rows_of(p, batch, n, 8)
    xs = np.array(edge_points(p, g, n, s, 9, 11), dtype=np.uint64)
    out = np.zeros(batch * len(xs), dtype=np.uint64)
    _c().call("ronk_poly_lagrange_eval_batch_u64_host", p, g, rows.ctypes.data_as(C.c_void_p), n, batch, s,
              xs.ctypes.data_as(C.c_void_p), len(xs), out.ctypes.data_as(C.c_void_p))
    assert np.array_equal(out, host(eval_dev(dev(rows), dev(xs), n, s, p, g)).reshape(-1))
    for z in (lm.nodes(p, g, n, s)[1], 7 % p):
        v, q = np.zeros(batch, dtype=np.uint64), np.zeros(batch * n, dtype=np.uint64)
        _c().call("ronk_poly_lagrange_open_u64_host", p, g, rows.ctypes.data_as(C.c_void_p), n, batch, s, z,
                  v.ctypes.data_as(C.c_void_p), q.ctypes.data_as(C.c_void_p))
        dv, dq = open_dev(dev(rows), z, n, s, p, g)
        assert np.array_equal(v, host(dv)) and np.array_equal(q, host(dq).reshape(-1))
    bad = xs.copy()
    bad[3] = p   # a non-canonical point is refused before anything is staged
    keep = out.copy()
    assert _lib.lib().ronk_poly_lagrange_eval_batch_u64_host(_c()._h, p, g, rows.ctypes.data_as(C.c_void_p), n, batch, s,
                                                              bad.ctypes.data_as(C.c_void_p), len(bad),
                                                              out.ctypes.data_as(C.c_void_p)) == _lib.EINVAL
    assert np.array_equal(out, keep)


@pytest.mark.parametrize("n,batch", [(1 << 12, 5), (1 << 22, 2)])
def test_gated_non_blocking_stream(n, batch):
    """A fresh context on a non-blocking stream held behind a sleep: the calls return before the stream has run, read
    the inputs copied in behind the gate and give the default context's words."""
    import torch
    from ronkathon_b200 import ops
    from ronkathon_b200._lib import Context
    p, g = GL, 7
    rows = ops.splitmix_fill(_c(), batch * n, 21, p).view(batch, n)
    xs = dev(np.array([5, 0, 7, 123456789], dtype=np.uint64))
    z_on = 7 * pow(pow(g, (p - 1) // n, p), 3, p) % p
    want_e = eval_dev(rows, xs, n, 7, p, g)
    want_off = open_dev(rows, 11, n, 7, p, g)
    want_on = open_dev(rows, z_on, n, 7, p, g)
    _c().sync()
    s = torch.cuda.Stream()
    c = Context(0, s.cuda_stream)
    try:
        rin = rows.flip(1).contiguous()
        with torch.cuda.stream(s):   # once on wrong inputs: first uses out of the gate
            ops.lagrange_eval(c, rin, xs, n, shift=7)
            ops.lagrange_open(c, rin, 11, n, shift=7)
            ops.lagrange_open(c, rin, z_on, n, shift=7)
        s.synchronize()
        with torch.cuda.stream(s):
            torch.cuda._sleep(100_000_000)
            rin.copy_(rows)
            e = ops.lagrange_eval(c, rin, xs, n, shift=7)
            off = ops.lagrange_open(c, rin, 11, n, shift=7)
            on = ops.lagrange_open(c, rin, z_on, n, shift=7)
            assert not s.query(), "the stream finished before the calls returned"
        s.synchronize()
        assert torch.equal(e, want_e)
        for got, want in ((off, want_off), (on, want_on)):
            assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    finally:
        c.close()


def test_ops_shapes():
    from ronkathon_b200 import ops
    p, g = 17, 3
    row = dev(np.array([1, 2, 3, 4], dtype=np.uint64))
    out = ops.lagrange_eval(_c(), row, dev(np.array([5, 6], dtype=np.uint64)), 4, p=p, g=g)
    assert tuple(out.shape) == (2,)
    v, q = ops.lagrange_open(_c(), row, 5, 4, p=p, g=g)
    assert v.dim() == 0 and tuple(q.shape) == (4,)
    wv, wq = lm.quotient(p, g, [1, 2, 3, 4], 5)
    assert int(host(v.reshape(1))[0]) == wv and host(q).tolist() == wq
