"""CPU tier: a Python-integer model of the three subproduct-tree walks of csrc/poly_tree.cu (product tree up, scaled
remainder tree down, interpolation up), checked against the oracle.  It pins the index arithmetic the kernels use: the
node degrees on the right spine, the wrap correction of two full children, the root slice of rev(f)·rev(M)^-1 and the
middle-product offsets, with every D-point product taken cyclically as the transforms take it.

`lb` is the number of levels the shared-memory kernels build (min(B, K) with B = 6 on the device); small values put
more levels on the cyclic-product path."""
import numpy as np
import pytest

import oracle

GL = oracle.GOLDILOCKS
BABYBEAR = 2013265921


def _log2_ceil(v):
    return max(0, (v - 1).bit_length())


def node_deg(k, j, i):
    """Degree of node i at level j: the leaves past k are the constant 1."""
    return max(0, min(1 << j, k - (i << j)))


def cyclic(p, a, b, D):
    out = [0] * D
    for i, x in enumerate(a):
        if x:
            for j, y in enumerate(b):
                out[(i + j) % D] = (out[(i + j) % D] + x * y) % p
    return out


def schoolbook(p, a, b):
    out = [0] * (len(a) + len(b) - 1)
    for i, x in enumerate(a):
        for j, y in enumerate(b):
            out[i + j] = (out[i + j] + x * y) % p
    return out


def series_inverse(p, h, n):
    """h^-1 mod y^n, h[0] = 1."""
    g = [0] * n
    g[0] = 1
    for i in range(1, n):
        g[i] = -sum(h[a] * g[i - a] for a in range(1, min(i, len(h) - 1) + 1)) % p
    return g


def product_tree(p, xs, B):
    """levels[j][i] = node i of level j (2^j + 1 words), j in [lb, K]."""
    k = len(xs)
    K = _log2_ceil(k)
    lb, N = min(B, K), 1 << K
    leaf = [[(-x) % p, 1] if i < k else [1, 0] for i, x in enumerate(list(xs) + [0] * (N - k))]
    levels = {}
    nodes = leaf
    for j in range(lb):  # the shared-memory kernel: schoolbook products
        nodes = [schoolbook(p, nodes[2 * i], nodes[2 * i + 1]) for i in range(len(nodes) // 2)]
    levels[lb] = nodes
    for j in range(lb, K):  # one cyclic D-point product per parent, then the wrap correction
        D = 2 << j
        nxt = []
        for i in range(N >> (j + 1)):
            c = cyclic(p, levels[j][2 * i], levels[j][2 * i + 1], D)
            if node_deg(k, j + 1, i) == D:  # two full monic children: X^D wrapped onto X^0
                c[0] = (c[0] - 1) % p
                nxt.append(c + [1])
            else:
                nxt.append(c + [0])
        levels[j + 1] = nxt
    return levels, K, lb, N


def multieval(p, f, xs, B, tree=None):
    k, d = len(xs), len(f)
    if d == 0:
        return [0] * k
    levels, K, lb, N = tree or product_tree(p, xs, B)
    M = levels[K][0]
    # root: h = rev_d(f)·rev_k(M)^-1 mod y^d, ρ[u] = h[d-1-u] for u < min(d, k), zero above
    hr = [M[k - i] for i in range(min(k + 1, d))]
    G = series_inverse(p, hr, d)
    h = schoolbook(p, [f[d - 1 - i] for i in range(d)], G)[:d]
    R = [[h[d - 1 - u] if u < min(d, k) else 0 for u in range(N)]]
    for j in range(K - 1, lb - 1, -1):  # parents at level j + 1
        D = 2 << j
        nxt = []
        for i in range(N >> (j + 1)):
            dl, dr = node_deg(k, j, 2 * i), node_deg(k, j, 2 * i + 1)
            ml = cyclic(p, levels[j][2 * i], R[i], D)      # M_L·ρ
            mr = cyclic(p, levels[j][2 * i + 1], R[i], D)  # M_R·ρ
            nxt.append([mr[dr + u] if u < dl else 0 for u in range(D // 2)])
            nxt.append([ml[dl + u] if u < dr else 0 for u in range(D // 2)])
        R = nxt
    out = [0] * k
    for s, (Ms, rho) in enumerate(zip(levels[lb], R)):  # bottom: r = polynomial part of M·ρ·X^-δ, then Horner
        dl = node_deg(k, lb, s)
        r = [sum(Ms[e + dl - u] * rho[u] for u in range(e, dl)) % p for e in range(dl)]
        for i in range(dl):
            x, acc = xs[(s << lb) + i], 0
            for c in reversed(r):
                acc = (acc * x + c) % p
            out[(s << lb) + i] = acc
    return out


def interpolate(p, xs, ys, B):
    tree = product_tree(p, xs, B)
    levels, K, lb, N = tree
    k = len(xs)
    M = levels[K][0]
    w = multieval(p, [(i + 1) * M[i + 1] % p for i in range(k)], xs, B, tree)  # M'(x_i)
    c = [y * pow(v, -1, p) % p for y, v in zip(ys, w)]
    # bottom: r and M per level in shared memory
    r = [[c[i]] if i < k else [0] for i in range(N)]
    m = [[(-xs[i]) % p, 1] if i < k else [1, 0] for i in range(N)]
    for j in range(lb):
        r = [[(a + b) % p for a, b in zip(schoolbook(p, r[2 * i], m[2 * i + 1])[:2 << j],
                                           schoolbook(p, r[2 * i + 1], m[2 * i])[:2 << j])] for i in range(len(r) // 2)]
        m = [schoolbook(p, m[2 * i], m[2 * i + 1]) for i in range(len(m) // 2)]
    assert m == levels[lb]
    for j in range(lb, K):
        D = 2 << j
        r = [[(a + b) % p for a, b in zip(cyclic(p, r[2 * i], levels[j][2 * i + 1], D),
                                           cyclic(p, r[2 * i + 1], levels[j][2 * i], D))] for i in range(N >> (j + 1))]
    return r[0][:k]


def _points(p, k, seed):
    xs = [int(v) for v in oracle.splitmix(p, seed, k)]
    if k >= 3:
        xs[0], xs[k // 2] = 0, p - 1
    return xs


KS = [1, 2, 3, 63, 64, 65, 100]


@pytest.mark.parametrize("p", [GL, BABYBEAR])
@pytest.mark.parametrize("B", [0, 2, 6])
@pytest.mark.parametrize("k", KS)
def test_product_tree(p, B, k):
    xs = _points(p, k, 10 + k)
    levels, K, lb, N = product_tree(p, xs, B)
    exp = np.array([1], np.uint64)
    for x in xs:
        exp = oracle.poly_mul(p, exp, np.array([(-x) % p, 1], np.uint64))
    assert levels[K][0][:k + 1] == [int(v) for v in exp]
    assert all(v == 0 for v in levels[K][0][k + 1:])


@pytest.mark.parametrize("p", [GL, BABYBEAR])
@pytest.mark.parametrize("B", [0, 2, 6])
@pytest.mark.parametrize("k", KS)
def test_multieval(p, B, k):
    xs = _points(p, k, 20 + k)
    if k >= 4:
        xs[1] = xs[2]  # a repeated point
    for d in sorted({0, 1, max(k - 1, 0), k, k + 1, 3 * k}):
        f = [int(v) for v in oracle.splitmix(p, 30 + d, d)]
        assert multieval(p, f, xs, B) == [oracle.poly_eval_horner(p, f, x) for x in xs], (k, d)


@pytest.mark.parametrize("p", [GL, BABYBEAR])
@pytest.mark.parametrize("B", [0, 2, 6])
@pytest.mark.parametrize("k", KS)
def test_interpolate(p, B, k):
    xs = _points(p, k, 40 + k)
    assert len(set(xs)) == k
    ys = [int(v) for v in oracle.splitmix(p, 50 + k, k)]
    got = interpolate(p, xs, ys, B)
    assert [oracle.poly_eval_horner(p, got, x) for x in xs] == ys
    if k <= 12:
        assert got == [int(v) for v in oracle.rs_decode(p, np.array(xs, np.uint64), np.array(ys, np.uint64), k)]
