"""The edges of the subproduct-tree envelope (csrc/poly_tree.cu through ronk_poly_from_roots_u64 / multieval_u64 /
interpolate_u64): every test prime on both sides of the size at which its two-adicity stops the tree, the multieval
crossover on min(d, m), lopsided and 2^24-point shapes, degenerate point sets, and a context whose workspaces hold junk
from earlier, larger calls.

Which path runs is pinned for every call: tree_expected() restates poly.cu's path rule, and the launch record names the
path taken.  Values are compared with routes that share no code with the tree: ronk_poly_eval_u64 (one CTA per point),
ronk_poly_interpolate_u64_host, the oracle, the forward transform, and products taken with the field kernels alone.
Above 2^16 points the direct kernel runs on a strided subset of the points plus the special ones."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle
from gpu_util import BABYBEAR, GL, MONT_PRIMES, ctx, dev, host, s64

pytestmark = pytest.mark.gpu

KOALA = MONT_PRIMES["koalabear"][0]
P32 = MONT_PRIMES["p32"][0]
SENTINEL = 0x5EED5EED5EED5EED
FALLBACK = {"from_roots": ["interp_master"], "multieval": ["poly_eval"],
            "interpolate": ["interp_master", "interp_nodes", "interp_sum"]}
CROSSOVER = {"from_roots": 128, "multieval": 1 << 15, "interpolate": 2048}  # poly.cu's k*TreeMin
LITERAL_MAX = 8192   # largest interpolation / from_roots off the tree
MAX_POINTS = 1 << 24


def tree_expected(p, k, d, op="multieval", forced=True):
    """The path poly.cu takes for k points (and d coefficients, multieval) with g != 0: "tree", "fallback" or
    "unsupported".  The tree needs every transform of its plan to divide p - 1 and be at most 2^26 points: the levels
    above the 64-leaf shared-memory blocks take 2^j-point transforms up to 2^⌈log2 k⌉, evaluation's root 2^⌈log2(2d-1)⌉
    (interpolation evaluates M', d = k).  forced: a RONK_TREE_MIN=1 context; else the measured crossovers."""
    if k > MAX_POINTS:
        return "unsupported"
    K = (k - 1).bit_length()

    def fits(d):
        lmax = K if K > 6 else 0
        if d:
            lmax = max(lmax, 1, (2 * d - 2).bit_length())
        return lmax <= 26 and (p - 1) % (1 << lmax) == 0

    low = 1 if forced else CROSSOVER[op]
    if op == "from_roots":
        tree = k <= 64 or (fits(0) and k >= low)
    elif op == "multieval":
        tree = d > 0 and fits(d) and min(d, k) >= low
    else:
        tree = fits(k) and (k >= low or k > LITERAL_MAX)
    if tree:
        return "tree"
    return "unsupported" if op != "multieval" and k > LITERAL_MAX else "fallback"


@pytest.fixture(scope="module")
def contexts():
    """make(forced) → a new context on the suite's stream, closed when the module ends (their workspaces reach several
    GB).  forced: RONK_TREE_MIN=1, the tree at every size it fits."""
    import torch
    from ronkathon_b200 import Context
    made = []

    def make(forced):
        ctx()
        if forced:
            os.environ["RONK_TREE_MIN"] = "1"
        try:
            c = Context(0, torch.cuda.current_stream().cuda_stream)
        finally:
            os.environ.pop("RONK_TREE_MIN", None)
        made.append(c)
        return c

    yield make
    ctx().sync()
    for c in made:
        c.close()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def tree(contexts):
    return contexts(True)


@pytest.fixture(scope="module")
def dflt(contexts):
    return contexts(False)


def _generator(p):
    from ronkathon_b200 import _lib
    g = C.c_uint64()
    assert _lib.lib().ronk_field_generator(p, C.byref(g)) == 0
    return g.value


def _call(c, op, p, g, a, b=None):
    """ronk_poly_<op>_u64 on c with a sentinel-filled out: from_roots(xs=a), multieval(coeffs=a, xs=b),
    interpolate(xs=a, ys=b).  Returns (out, path, launch names); out is None and untouched when unsupported."""
    import torch
    from ronkathon_b200 import RonkError, _lib
    from ronkathon_b200._lib import EUNSUPPORTED
    P = _lib._ptr
    if op == "from_roots":
        n, args = a.numel() + 1, (P(a), a.numel())
    elif op == "multieval":
        n, args = b.numel(), (P(a), a.numel(), P(b), b.numel())
    else:
        n, args = a.numel(), (P(a), P(b), a.numel())
    out = torch.full((n,), SENTINEL, dtype=torch.int64, device="cuda")
    c.sync()
    c.prof_fetch()
    c.prof_enable(True)
    path = None
    try:
        c.call(f"ronk_poly_{op}_u64", p, g, *args, P(out))
    except RonkError as e:
        if e.code != EUNSUPPORTED:
            raise
        path = "unsupported"
    finally:
        c.sync()
        c.prof_enable(False)
    names = [name for name, _ in c.prof_fetch()]
    if path == "unsupported":
        assert names == [] and bool((out == SENTINEL).all()), names
        return None, path, names
    if names[:1] == ["tree_leaves"]:
        return out, "tree", names
    assert names == FALLBACK[op], names
    return out, "fallback", names


def _check(c, op, p, g, a, b=None, forced=True):
    """_call, with the path asserted against tree_expected; returns out."""
    k = b.numel() if op == "multieval" else a.numel()
    d = a.numel() if op == "multieval" else 0
    out, path, names = _call(c, op, p, g, a, b)
    assert path == tree_expected(p, k, d, op, forced), (op, p, k, d, forced, names[:4])
    return out


def _points(p, m, seed, repeat=True):
    """m seeded residues on the device: 0 at index 0, p - 1 at m // 2, x[2] = x[1]."""
    from ronkathon_b200 import ops
    xs = ops.splitmix_fill(ctx(), m, seed, p)
    if m >= 3:
        xs[0], xs[m // 2] = 0, s64(p - 1)
    if repeat and m >= 4:
        xs[2] = xs[1]
    return xs


def _distinct(p, n, seed):
    """n distinct residues in a seeded order (host array), with 0 at index 0 and p - 1 at n // 2 when n ≥ 3."""
    rng = np.random.default_rng(seed)
    if p < 1 << 20:
        v = rng.permutation(np.arange(1, p - 1, dtype=np.uint64))
    else:
        v = np.sort(oracle.splitmix(p, seed, n + (n >> 3) + 8))
        keep = np.concatenate([[True], v[1:] != v[:-1]]) & (v != 0) & (v != p - 1)
        v = rng.permutation(v[keep])
    assert len(v) >= n
    v = v[:n].copy()
    if n >= 3:
        v[0], v[n // 2] = 0, p - 1
    return v


def _subset(n):
    """About 4096 strided indices plus 0, 1, 2 (the repeated pair of _points), n // 2 and n - 1."""
    idx = np.concatenate([np.arange(0, n, -(-n // 4096)), [0, 1, 2, n // 2, n - 1]])
    return np.unique(idx[idx < n]).astype(np.int64)


def _direct(p, f, xs):
    """ronk_poly_eval_u64 on the shared context (one CTA per point, no transform)."""
    from ronkathon_b200 import ops
    return host(ops.poly_eval(ctx(), f, xs, p=p))


def _direct_subset(p, f, xs):
    """(indices, f at xs[indices] by the direct kernel)."""
    import torch
    idx = _subset(xs.numel())
    return idx, _direct(p, f, xs[torch.from_numpy(idx).cuda()].contiguous())


def _host_interp(p, xs, ys):
    from ronkathon_b200 import _lib
    out = np.empty(len(xs), np.uint64)
    ctx().call("ronk_poly_interpolate_u64_host", p, _lib._ptr(xs), _lib._ptr(ys), len(xs), _lib._ptr(out))
    return out


def _from_roots_oracle(p, xs):
    acc = np.array([1], np.uint64)
    for x in xs:
        acc = oracle.poly_mul(p, acc, np.array([(p - int(x)) % p, 1], np.uint64))
    return acc


def _prod_minus(p, z, xs):
    """Π (z - xs[i]) on the device by the field kernels alone: one sub, then pairwise mul halvings (padded with 1)."""
    import torch
    from ronkathon_b200 import ops
    n = xs.numel()
    v = ops.field_binop(ctx(), "sub", torch.full((n,), s64(z), dtype=torch.int64, device="cuda"), xs, p=p)
    pad = (1 << (n - 1).bit_length()) - n
    if pad:
        v = torch.cat([v, torch.ones(pad, dtype=torch.int64, device="cuda")])
    while v.numel() > 1:
        h = v.numel() // 2
        v = ops.field_binop(ctx(), "mul", v[:h].contiguous(), v[h:].contiguous(), p=p)
    return int(host(v)[0])


def _check_product(p, M, xs, seed):
    """M = Π (X - xs[i]) without a quadratic reference: monic of degree k, M(z) = Π (z - x_i) at two random z, and
    M(x_i) = 0 on the subset."""
    k = xs.numel()
    Mh = host(M)
    assert len(Mh) == k + 1 and Mh[k] == 1
    zs = oracle.splitmix(p, seed, 2)
    assert _direct(p, M, dev(zs)).tolist() == [_prod_minus(p, int(z), xs) for z in zs]
    _, at = _direct_subset(p, M, xs)
    assert not at.any()


def _check_interp_values(p, coeffs, xs, ys):
    """The interpolant takes ys at xs, on the subset, by the direct kernel."""
    idx, at = _direct_subset(p, coeffs, xs)
    assert np.array_equal(at, host(ys)[idx])


# ---- A. every test prime on both sides of its two-adicity edge -------------------------------------------------------
EDGE_PRIMES = {"p127": (127, 1), "p101": (101, 2), "p2adic3": ((1 << 64) - 279, 3), "p17": (17, 4),
               "p32": (P32, 16), "koalabear": (KOALA, 24)}


def _edge_prime(name):
    p, s = EDGE_PRIMES[name]
    g = MONT_PRIMES[name][1] if name in MONT_PRIMES else _generator(p)
    assert pow(g, (p - 1) // 2, p) == p - 1 and ((p - 1) & -(p - 1)).bit_length() - 1 == s
    return p, g, s


@pytest.mark.parametrize("name", list(EDGE_PRIMES))
def test_from_roots_small_on_tree_leaves(name, dflt):
    """k ≤ 64 is one shared-memory CTA for every prime, on the default context: repeated roots, 0 and p - 1."""
    p, g, _ = _edge_prime(name)
    for k in (1, 2, 3, 63, 64):
        xs = oracle.splitmix(p, 10 + k, k)
        if k >= 3:
            xs[0], xs[k // 2] = 0, p - 1
        if k >= 4:
            xs[2] = xs[1]
        out, path, names = _call(dflt, "from_roots", p, g, dev(xs))
        assert path == tree_expected(p, k, 0, "from_roots", forced=False) == "tree" and names == ["tree_leaves"]
        assert np.array_equal(host(out), _from_roots_oracle(p, xs)), (name, k)


@pytest.mark.parametrize("name", list(EDGE_PRIMES))
def test_multieval_at_fit_edge(name, tree):
    """d = 2^(s-1) is the largest degree whose root transforms divide p - 1; one more coefficient takes poly_eval.
    For small p, m > p repeats points."""
    p, g, s = _edge_prime(name)
    for m in (1, 5, 64):
        xs = dev(oracle.splitmix(p, 20 + m, m))
        for d in (1 << (s - 1), (1 << (s - 1)) + 1):
            f = dev(oracle.splitmix(p, 30 + d, d))
            got = _check(tree, "multieval", p, g, f, xs)
            assert np.array_equal(host(got), _direct(p, f, xs)), (name, m, d)


@pytest.mark.parametrize("name", list(EDGE_PRIMES))
def test_interpolate_at_fit_edge(name, tree):
    """k = 2^(s-1) runs the tree; k + 1 the literal kernels up to 8192 nodes, else RONK_EUNSUPPORTED."""
    p, g, s = _edge_prime(name)
    for k in (1 << (s - 1), (1 << (s - 1)) + 1):
        xs, ys = _distinct(p, k, 40 + k), oracle.splitmix(p, 50 + k, k)
        X, Y = dev(xs), dev(ys)
        got = _check(tree, "interpolate", p, g, X, Y)
        if got is None:
            continue
        if k <= LITERAL_MAX:
            assert np.array_equal(host(got), _host_interp(p, xs, ys)), (name, k)
        else:
            _check_interp_values(p, got, X, Y)


@pytest.mark.parametrize("forced", [True, False])
def test_p32_full_edges(forced, tree, dflt):
    """p32 (s = 16) at 2^15 / 2^16 points, where its two-adicity binds: multieval on min(d, m) ≥ 2^15 takes the tree on
    the default context too."""
    p, g = MONT_PRIMES["p32"][:2]
    c = tree if forced else dflt
    for m, d in ((1 << 16, 1 << 15), (1 << 16, (1 << 15) + 1), ((1 << 16) + 1, 5)):
        xs, f = _points(p, m, 60 + m), dev(oracle.splitmix(p, 61 + d, d))
        got = _check(c, "multieval", p, g, f, xs, forced=forced)
        assert np.array_equal(host(got), _direct(p, f, xs)), (m, d)
    for k in (1 << 15, (1 << 15) + 1):
        X, Y = dev(_distinct(p, k, 62 + k)), dev(oracle.splitmix(p, 63 + k, k))
        got = _check(c, "interpolate", p, g, X, Y, forced=forced)
        if got is not None:
            assert np.array_equal(_direct(p, got, X), host(Y))
    for k in (1 << 16, (1 << 16) + 1):
        xs = _points(p, k, 64 + k)
        got = _check(c, "from_roots", p, g, xs, forced=forced)
        if got is not None:
            _check_product(p, got, xs, 65)


# ---- B. the multieval crossover is on min(d, m) ---------------------------------------------------------------------
@pytest.mark.parametrize("d,m", [(5, 1 << 16), (1 << 15, 1 << 15), (1 << 20, (1 << 15) - 1), (1 << 15, 1 << 20)])
def test_multieval_crossover_on_min(d, m, dflt):
    from ronkathon_b200 import ops
    f, xs = ops.splitmix_fill(ctx(), d, 70 + d, GL), _points(GL, m, 71 + m)
    got = host(_check(dflt, "multieval", GL, 7, f, xs, forced=False))
    idx, exp = _direct_subset(GL, f, xs)
    assert np.array_equal(got[idx], exp)


# ---- C. lopsided shapes ---------------------------------------------------------------------------------------------
def test_many_points_tiny_polynomial(tree):
    """Shamir-share shapes on the forced tree: 2^20 points, d from 1 to 65."""
    m = 1 << 20
    xs = _points(GL, m, 80)
    for d in (1, 2, 3, 64, 65):
        f = dev(oracle.splitmix(GL, 81 + d, d))
        got = _check(tree, "multieval", GL, 7, f, xs)
        assert np.array_equal(host(got), _direct(GL, f, xs)), d


@pytest.mark.parametrize("p,g", [(GL, 7), MONT_PRIMES["babybear"][:2]], ids=["gl", "babybear"])
def test_huge_polynomial_few_points(p, g, tree):
    """d = 2^25, the largest d whose root (Newton inversion, 2^26-point products) fits; 2^25 + 1 takes poly_eval.
    Two Horner values from the oracle keep the direct kernel from being its own reference."""
    d = 1 << 25
    fh = oracle.splitmix(p, 90, d + 1)
    f, f1 = dev(fh[:d]), dev(fh)
    for m in (1, 2, 63, 64, 65, 4097):
        xs = _points(p, m, 91 + m)
        got = host(_check(tree, "multieval", p, g, f, xs))
        assert np.array_equal(got, _direct(p, f, xs)), m
        if m == 65:
            for i in (1, m // 2):
                assert int(got[i]) == oracle.poly_eval_horner(p, fh[:d], int(host(xs)[i])), i
    xs = _points(p, 65, 92)
    got = _check(tree, "multieval", p, g, f1, xs)
    assert np.array_equal(host(got), _direct(p, f1, xs))


# ---- D. the top of the envelope -------------------------------------------------------------------------------------
def test_goldilocks_2_24(dflt):
    """m = d = 2^24: values on the subset, with a repeated pair; then the interpolant at 2^24 distinct points is f."""
    from ronkathon_b200 import ops
    n = MAX_POINTS
    f = ops.splitmix_fill(ctx(), n, 100, GL)
    xs = dev(_distinct(GL, n, 101))
    rep = xs.clone()
    rep[2] = rep[1]
    got = host(_check(dflt, "multieval", GL, 7, f, rep, forced=False))
    idx, exp = _direct_subset(GL, f, rep)
    assert np.array_equal(got[idx], exp) and got[1] == got[2]
    ys = _check(dflt, "multieval", GL, 7, f, xs, forced=False)
    coeffs = _check(dflt, "interpolate", GL, 7, xs, ys, forced=False)
    assert bool((coeffs == f).all())


def test_babybear_2_24_points_2_25_coefficients(dflt):
    """The root runs 2^26-point Montgomery transforms."""
    p, g = MONT_PRIMES["babybear"][:2]
    f, xs = dev(oracle.splitmix(p, 110, 1 << 25)), _points(p, MAX_POINTS, 111)
    got = host(_check(dflt, "multieval", p, g, f, xs, forced=False))
    idx, exp = _direct_subset(p, f, xs)
    assert np.array_equal(got[idx], exp)


def test_koalabear_at_its_two_adicity(dflt):
    """s = 24 binds inside the envelope: m = 2^24 with d = 2^23, and the product of 2^24 linear factors (interpolation
    at 2^23 / 2^23 + 1 is test_interpolate_at_fit_edge)."""
    from ronkathon_b200 import ops
    p, g = MONT_PRIMES["koalabear"][:2]
    f, xs = ops.splitmix_fill(ctx(), 1 << 23, 120, p), _points(p, MAX_POINTS, 121)
    got = host(_check(dflt, "multieval", p, g, f, xs, forced=False))
    idx, exp = _direct_subset(p, f, xs)
    assert np.array_equal(got[idx], exp)
    M = _check(dflt, "from_roots", p, g, xs, forced=False)
    _check_product(p, M, xs, 122)
    assert _check(dflt, "from_roots", p, g, _points(p, MAX_POINTS + 1, 123), forced=False) is None


@pytest.mark.parametrize("p,g,k", [(GL, 7, (1 << 20) + 1), (GL, 7, (1 << 23) + 1),
                                   (*MONT_PRIMES["babybear"][:2], (1 << 20) + 1)], ids=["gl-2^20", "gl-2^23", "babybear-2^20"])
def test_just_past_a_power_of_two(p, g, k, dflt):
    """The root's right child is one point and 2^(K-1) - 1 constant-1 leaves, so every node on the right spine is
    partial (no wrap correction)."""
    from ronkathon_b200 import ops
    f, xs = ops.splitmix_fill(ctx(), k, 130, p), dev(_distinct(p, k, 131))
    got = host(_check(dflt, "multieval", p, g, f, xs, forced=False))
    idx, exp = _direct_subset(p, f, xs)
    assert np.array_equal(got[idx], exp)
    ys = ops.splitmix_fill(ctx(), k, 132, p)
    _check_interp_values(p, _check(dflt, "interpolate", p, g, xs, ys, forced=False), xs, ys)


# ---- E. the generator changes the kernels, not the words ------------------------------------------------------------
@pytest.mark.parametrize("p,g1,g2", [(GL, 7, pow(7, 5, GL)), (BABYBEAR, 31, pow(31, 3, BABYBEAR))], ids=["gl", "babybear"])
def test_generator_independence(p, g1, g2, dflt):
    """Goldilocks with g = 7 takes the Goldilocks policy, g = 7^5 the Montgomery one; babybear's g and g^3 give different
    roots of unity.  Values and interpolants at 2^20 + 3 points agree word for word."""
    from ronkathon_b200 import ops
    assert pow(g2, (p - 1) // 2, p) == p - 1
    n = (1 << 20) + 3
    f, xs, ys = ops.splitmix_fill(ctx(), n, 140, p), dev(_distinct(p, n, 141)), ops.splitmix_fill(ctx(), n, 142, p)
    vals = [host(_check(dflt, "multieval", p, g, f, xs, forced=False)) for g in (g1, g2)]
    assert np.array_equal(*vals)
    interps = [host(_check(dflt, "interpolate", p, g, xs, ys, forced=False)) for g in (g1, g2)]
    assert np.array_equal(*interps)


# ---- F. degenerate point sets and panics at size --------------------------------------------------------------------
@pytest.mark.parametrize("m", [1 << 16, 1 << 20])
def test_all_points_equal(m, dflt):
    """The whole tree is (X - x)^m."""
    import torch
    fh = oracle.splitmix(GL, 150 + m, m)
    f = dev(fh)
    for x in (0, GL - 1):
        xs = torch.full((m,), s64(x), dtype=torch.int64, device="cuda")
        got = host(_check(dflt, "multieval", GL, 7, f, xs, forced=False))
        assert bool((got == oracle.poly_eval_horner(GL, fh, x)).all()), x


def test_shuffled_roots_of_unity_give_the_transform(dflt):
    from ronkathon_b200 import ops
    n = 1 << 16
    w = pow(7, (GL - 1) // n, GL)
    pw = np.empty(n, np.uint64)
    acc = 1
    for i in range(n):
        pw[i] = acc
        acc = acc * w % GL
    perm = np.random.default_rng(160).permutation(n)
    f = ops.splitmix_fill(ctx(), n, 161, GL)
    got = host(_check(dflt, "multieval", GL, 7, f, dev(pw[perm]), forced=False))
    assert np.array_equal(got, host(ops.ntt_(ctx(), f.clone(), 16))[perm])


@pytest.mark.parametrize("p,g", [(GL, 7), MONT_PRIMES["koalabear"][:2]], ids=["gl", "koalabear"])
def test_repeated_x_at_size_panics(p, g, dflt):
    """A pair straddling the root's halves, and a pair inside the last 64-leaf block: RonkPanic, out untouched."""
    import torch
    from ronkathon_b200 import RonkPanic, _lib
    k = 1 << 20
    base = _distinct(p, k, 170)
    Y = dev(oracle.splitmix(p, 171, k))
    for i, j in ((5, k // 2 + 7), (k - 40, k - 2)):
        xs = base.copy()
        xs[j] = xs[i]
        X = dev(xs)
        out = torch.full((k,), SENTINEL, dtype=torch.int64, device="cuda")
        with pytest.raises(RonkPanic, match="repeated x"):
            dflt.call("ronk_poly_interpolate_u64", p, g, _lib._ptr(X), _lib._ptr(Y), k, _lib._ptr(out))
        assert bool((out == SENTINEL).all()), (i, j)


# ---- G. workspaces left dirty by larger calls -----------------------------------------------------------------------
def test_dirty_workspaces(contexts):
    """Small calls after a 2^24-point multieval and a 2^22-point interpolation (junk in every scratch block) give the
    words the same calls give on contexts that have run nothing before them."""
    from ronkathon_b200 import ops
    r100, r4097 = _points(GL, 100, 180), _points(GL, 4097, 181)
    f3000, x1000 = dev(oracle.splitmix(GL, 182, 3000)), _points(GL, 1000, 183)
    f5, x65536 = dev(oracle.splitmix(GL, 184, 5)), _points(GL, 1 << 16, 185)
    i65, i4097 = dev(_distinct(GL, 65, 186)), dev(_distinct(GL, 4097, 187))
    y65, y4097 = dev(oracle.splitmix(GL, 188, 65)), dev(oracle.splitmix(GL, 189, 4097))
    a, b = ops.splitmix_fill(ctx(), 1 << 16, 190, GL), ops.splitmix_fill(ctx(), (1 << 15) + 1, 191, GL)
    calls = [
        lambda c: ops.poly_from_roots(c, r100),
        lambda c: ops.poly_from_roots(c, r4097),
        lambda c: ops.poly_multieval(c, f3000, x1000),
        lambda c: ops.poly_multieval(c, f5, x65536),
        lambda c: ops.poly_interpolate(c, i65, y65),
        lambda c: ops.poly_interpolate(c, i4097, y4097),
        lambda c: ops.poly_divrem(c, a, b),
    ]

    def run(c, fn):
        out = fn(c)
        return np.concatenate([host(t) for t in out]) if isinstance(out, tuple) else host(out)

    clean = []
    for fn in calls:
        c = contexts(True)
        clean.append(run(c, fn))
        c.close()
    dirty = contexts(True)
    ops.poly_multieval(dirty, ops.splitmix_fill(ctx(), MAX_POINTS, 192, GL), ops.splitmix_fill(ctx(), MAX_POINTS, 193, GL))
    for rnd in range(2):
        for i, fn in enumerate(calls):
            assert np.array_equal(run(dirty, fn), clean[i]), (rnd, i)
        if rnd == 0:
            n = 1 << 22
            ops.poly_interpolate(dirty, ops.splitmix_fill(ctx(), n, 194, GL), ops.splitmix_fill(ctx(), n, 195, GL))
