"""ronk_poly_from_roots_u64 / ronk_poly_multieval_u64 / ronk_poly_interpolate_u64 (ops.poly_from_roots, poly_multieval,
poly_interpolate): the subproduct tree of csrc/poly_tree.cu and its fallbacks.

Multipoint evaluation must equal ronk_poly_eval_u64 word for word, interpolation must equal
ronk_poly_interpolate_u64_host where that runs, and every size must be reachable on the tree path: a second context
created with RONK_TREE_MIN=1 takes the tree wherever its transforms fit, below the measured crossovers too."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle
from gpu_util import GL, MONT_PRIMES, ctx, dev, host

pytestmark = pytest.mark.gpu

TREE_PRIMES = {"gl": (GL, 7), **{n: (p, g) for n, (p, g, s) in MONT_PRIMES.items() if s >= 16}}
B = 6  # levels the shared-memory kernels build
_tree = None


def tree_ctx():
    """A context on the suite's stream that takes the tree path at every size it fits."""
    global _tree
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


def _generator(p):
    from ronkathon_b200 import _lib
    g = C.c_uint64()
    assert _lib.lib().ronk_field_generator(p, C.byref(g)) == 0
    return g.value


def _points(p, m, seed, repeat=True):
    xs = oracle.splitmix(p, seed, m)
    if m >= 3:
        xs[0], xs[m // 2] = 0, p - 1
    if repeat and m >= 4:
        xs[2] = xs[1]
    return xs


def _names(c, fn):
    c.sync()
    c.prof_fetch()
    c.prof_enable(True)
    try:
        out = fn()
        c.sync()
    finally:
        c.prof_enable(False)
    return out, [n for n, _ in c.prof_fetch()]


def _direct(p, f, xs):
    from ronkathon_b200 import ops
    return host(ops.poly_eval(ctx(), dev(f), dev(xs), p=p))


def _host_interp(p, xs, ys):
    from ronkathon_b200 import _lib
    out = np.empty(len(xs), np.uint64)
    ctx().call("ronk_poly_interpolate_u64_host", p, _lib._ptr(xs), _lib._ptr(ys), len(xs), _lib._ptr(out))
    return out


@pytest.mark.parametrize("name", list(TREE_PRIMES))
def test_multieval_matches_poly_eval(name):
    """Points 0 and p - 1 and a repeated point; d from 0 to 3m, m across the bottom-kernel and transform edges."""
    from ronkathon_b200 import ops
    p, g = TREE_PRIMES[name]
    for m in (1, 2, 3, (1 << B) - 1, (1 << B) + 1, 1000, 4095, 4097, 1 << 16):
        xs = _points(p, m, 100 + m)
        ds = (0, 1, m) if m == 1 << 16 else (0, 1, max(m - 1, 1), m, m + 1, 3 * m)
        for d in sorted(set(ds)):
            f = oracle.splitmix(p, 200 + d, d)
            exp = _direct(p, f, xs)
            for c in (tree_ctx(), ctx()):
                got = host(ops.poly_multieval(c, dev(f), dev(xs), p=p, g=g))
                assert np.array_equal(got, exp), (name, m, d, c is ctx())


def test_multieval_path_names():
    """Above the crossover the default context runs the tree (no poly_eval launch), below it the direct kernel."""
    from ronkathon_b200 import ops
    for m, tree in ((4, False), ((1 << 15) - 1, False), (1 << 15, True)):
        f, xs = dev(oracle.splitmix(GL, 1, m)), dev(oracle.splitmix(GL, 2, m))
        _, names = _names(ctx(), lambda: ops.poly_multieval(ctx(), f, xs))
        assert ("poly_eval" not in names and "tree_eval_leaves" in names) if tree else names == ["poly_eval"], (m, names)


@pytest.mark.parametrize("p", [101, 17, 127, "gl_g0"])
def test_fallback(p):
    """Primes without the roots of unity the tree needs, and g = 0: the existing kernels run, with the same words."""
    from ronkathon_b200 import ops
    p, g = (GL, 0) if p == "gl_g0" else (p, _generator(p))
    for c in (tree_ctx(), ctx()):
        m = 1000
        f, xs = oracle.splitmix(p, 3, m), _points(p, m, 4)
        got, names = _names(c, lambda: host(ops.poly_multieval(c, dev(f), dev(xs), p=p, g=g)))
        assert names == ["poly_eval"] and np.array_equal(got, _direct(p, f, xs))
        k = min(p - 1, 600)
        if p == GL:
            xs = _points(p, k, 5, repeat=False)
        else:
            xs = np.random.default_rng(5).permutation(p)[:k].astype(np.uint64)
            if 0 not in xs:
                xs[0] = 0
        ys = oracle.splitmix(p, 6, k)
        got, names = _names(c, lambda: host(ops.poly_interpolate(c, dev(xs), dev(ys), p=p, g=g)))
        assert names == ["interp_master", "interp_nodes", "interp_sum"], names
        assert np.array_equal(got, _host_interp(p, xs, ys))
        if k > 1 << B:
            r, names = _names(c, lambda: host(ops.poly_from_roots(c, dev(xs[:200]), p=p, g=g)))
            assert names == ["interp_master"], names
            assert np.array_equal(r, _from_roots_oracle(p, xs[:200]))


def _from_roots_oracle(p, xs):
    acc = np.array([1], np.uint64)
    for x in xs:
        acc = oracle.poly_mul(p, acc, np.array([(p - int(x)) % p, 1], np.uint64))
    return acc


@pytest.mark.parametrize("name", list(TREE_PRIMES))
def test_from_roots(name):
    from ronkathon_b200 import ops
    p, g = TREE_PRIMES[name]
    for k in (0, 1, 2, 3, 63, 64, 65, 100, 300):
        xs = _points(p, k, 300 + k)
        for c in (tree_ctx(), ctx()):
            got = host(ops.poly_from_roots(c, dev(xs), p=p, g=g))
            assert np.array_equal(got, _from_roots_oracle(p, xs)), (name, k)
    for k in ((1 << 12) + 1, 1 << 16) + ((1 << 20,) if name in ("gl", "babybear") else ()):
        xs = _points(p, k, 400 + k)
        got = host(ops.poly_from_roots(ctx(), dev(xs), p=p, g=g))
        assert len(got) == k + 1 and got[k] == 1
        for z in oracle.splitmix(p, 500 + k, 2):
            exp = 1
            for x in xs.tolist():
                exp = exp * (int(z) - x) % p
            assert oracle.poly_eval_horner(p, got, int(z)) == exp, (name, k)


@pytest.mark.parametrize("name", list(TREE_PRIMES))
def test_interpolate_matches_host_variant(name):
    from ronkathon_b200 import ops
    p, g = TREE_PRIMES[name]
    for k in (1, 2, 3, 64, 65, 1000) + ((8192,) if name in ("gl", "babybear", "pbig") else ()):
        xs = _points(p, k, 600 + k, repeat=False)
        assert len(set(xs.tolist())) == k
        ys = oracle.splitmix(p, 700 + k, k)
        exp = _host_interp(p, xs, ys)
        for c in (tree_ctx(), ctx()):
            got = host(ops.poly_interpolate(c, dev(xs), dev(ys), p=p, g=g))
            assert np.array_equal(got, exp), (name, k, c is ctx())


@pytest.mark.parametrize("k,name", [((1 << 16) + 3, "gl"), ((1 << 16) + 3, "pbig"), (1 << 20, "gl")])
def test_interpolate_reproduces_values(k, name):
    from ronkathon_b200 import ops
    p, g = TREE_PRIMES[name]
    xs, ys = dev(_points(p, k, 800, repeat=False)), ops.splitmix_fill(ctx(), k, 801, p)
    coeffs = ops.poly_interpolate(ctx(), xs, ys, p=p, g=g)
    assert np.array_equal(host(ops.poly_multieval(ctx(), coeffs, xs, p=p, g=g)), host(ys))


@pytest.mark.parametrize("j", [1, 4, 10, 16])
def test_interpolate_roots_of_unity_is_inverse_transform(j):
    from ronkathon_b200 import ops
    n = 1 << j
    w = pow(7, (GL - 1) // n, GL)
    xs = np.array([pow(w, i, GL) for i in range(n)], np.uint64)
    ys = dev(oracle.splitmix(GL, 900 + j, n))
    got = host(ops.poly_interpolate(tree_ctx(), dev(xs), ys))
    exp = host(ops.ntt_(ctx(), ys.clone(), j, inverse=True))
    assert np.array_equal(got, exp)


@pytest.mark.parametrize("k", [1000, 70000])
def test_repeated_x_panics(k):
    """A repeated x inside one bottom subtree and across the root's halves; out keeps its words."""
    import torch
    from ronkathon_b200 import RonkPanic, _lib
    for i, j in ((3, 5), (0, k - 1)):
        xs = _points(GL, k, 1000 + k, repeat=False)
        xs[j] = xs[i]
        X, Y = dev(xs), dev(oracle.splitmix(GL, 1001, k))
        out = torch.full((k,), 12345, dtype=torch.int64, device="cuda")
        with pytest.raises(RonkPanic, match="repeated x"):
            tree_ctx().call("ronk_poly_interpolate_u64", GL, 7, _lib._ptr(X), _lib._ptr(Y), k, _lib._ptr(out))
        assert bool((out == 12345).all())


def test_literal_cap_and_tree_above_it():
    from ronkathon_b200 import RonkError, ops
    from ronkathon_b200._lib import EUNSUPPORTED
    k = 8193
    xs, ys = dev(_points(GL, k, 1100, repeat=False)), dev(oracle.splitmix(GL, 1101, k))
    with pytest.raises(RonkError) as e:
        ops.poly_interpolate(ctx(), xs, ys, g=0)
    assert e.value.code == EUNSUPPORTED
    coeffs = ops.poly_interpolate(ctx(), xs, ys)
    assert np.array_equal(host(ops.poly_multieval(ctx(), coeffs, xs)), host(ys))


def test_identity_at_size():
    """interpolate(xs, multieval(f, xs)) == f at 2^22 Goldilocks points."""
    import torch
    from ronkathon_b200 import ops
    n = 1 << 22
    f, xs = ops.splitmix_fill(ctx(), n, 1200, GL), ops.splitmix_fill(ctx(), n, 1201, GL)
    ys = ops.poly_multieval(ctx(), f, xs)
    assert torch.equal(ops.poly_interpolate(ctx(), xs, ys), f)


def test_argument_checks_and_launch_record():
    import torch
    from ronkathon_b200 import RonkError, RonkPanic, _lib, ops
    from ronkathon_b200._lib import EUNSUPPORTED
    c = tree_ctx()
    k = 300
    xs, ys = dev(_points(GL, k, 1300, repeat=False)), dev(oracle.splitmix(GL, 1301, k))
    out = torch.full((k + 1,), 7, dtype=torch.int64, device="cuda")
    P = _lib._ptr
    bad = [
        ("ronk_poly_from_roots_u64", GL, 7, None, k, P(out)),
        ("ronk_poly_from_roots_u64", GL, 7, P(xs), k, None),
        ("ronk_poly_from_roots_u64", GL, 7, P(out), k, P(out)),                      # out overlaps xs
        ("ronk_poly_from_roots_u64", GL, GL, P(xs), k, P(out)),                      # g out of range
        ("ronk_poly_multieval_u64", GL, 7, None, k, P(xs), k, P(out)),
        ("ronk_poly_multieval_u64", GL, 7, P(ys), k, None, k, P(out)),
        ("ronk_poly_multieval_u64", GL, 7, P(ys), k, P(xs), k, P(ys)),               # out = coeffs
        ("ronk_poly_multieval_u64", GL, 7, P(ys), k, P(out), k, P(out)),             # out = xs
        ("ronk_poly_interpolate_u64", GL, 7, None, P(ys), k, P(out)),
        ("ronk_poly_interpolate_u64", GL, 7, P(xs), None, k, P(out)),
        ("ronk_poly_interpolate_u64", GL, 7, P(xs), P(ys), k, P(xs)),
        ("ronk_poly_interpolate_u64", GL, 7, P(xs), P(out), k, P(out)),
    ]
    for args in bad:
        with pytest.raises(RonkPanic):
            c.call(*args)
    for args in (("ronk_poly_from_roots_u64", GL, 7, P(xs), (1 << 24) + 1, P(out)),
                 ("ronk_poly_multieval_u64", GL, 7, P(ys), k, P(xs), (1 << 24) + 1, P(out)),
                 ("ronk_poly_interpolate_u64", GL, 7, P(xs), P(ys), (1 << 24) + 1, P(out))):
        with pytest.raises(RonkError) as e:
            c.call(*args)
        assert e.value.code == EUNSUPPORTED
    assert bool((out == 7).all()) and np.array_equal(host(xs), _points(GL, k, 1300, repeat=False))
    for fn in (lambda: ops.poly_from_roots(c, xs), lambda: ops.poly_multieval(c, ys, xs),
               lambda: ops.poly_interpolate(c, xs, ys)):
        before = c.launches
        _, names = _names(c, fn)
        assert c.launches - before == len(names) and "tree_leaves" in names, names
