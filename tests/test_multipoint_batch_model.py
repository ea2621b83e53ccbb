"""CPU tier: the batched walks of csrc/poly_tree.cu and the batched literal interpolation of csrc/poly.cu, modelled in
Python integers on the kernels' flat buffers and checked row by row against the oracle.

It extends test_multipoint_model.py (its product tree is used as is) to the batched layout: row b of every row buffer at
b·N, a level's parents indexed over batch·P with the node index i & (P - 1), the node spectra shared by every row (one
cyclic product per parent against the node of its row-local index), the root's rows against the shared inverse padded
with a zero word, the leaves kernels over blockIdx.y with y·M'(x)^-1 fused in, and the literal interpolation's per-row
partial sums at partial[(b·nwarps + warp)·k + i]."""
import numpy as np
import pytest

import oracle
from test_multipoint_model import _log2_ceil, node_deg, product_tree, series_inverse

GL = oracle.GOLDILOCKS
PRIMES = {"gl": GL, "babybear": 2013265921, "koalabear": 2130706433}
SIZES = [1, 63, 64, 65, 200, 1000]
BATCHES = [1, 2, 3, 7]
B = 6


def _mul(p, a, b):
    return [int(v) for v in oracle.poly_mul(p, np.array(a, np.uint64), np.array(b, np.uint64))]


def cyclic(p, a, b, D):
    out = [0] * D
    for i, v in enumerate(_mul(p, a, b)):
        out[i % D] = (out[i % D] + v) % p
    return out


def eval_leaves(p, Ml, R, xs, k, lb, N, batch):
    """tree_eval_leaves_kernel over grid (N >> lb, rows): ρ_b at R[b·N + s·w …], out[b·k + base + i]."""
    w, out = 1 << lb, [0] * (batch * k)
    for b in range(batch):
        for s in range(N >> lb):
            dl, base = node_deg(k, lb, s), s << lb
            rho = R[b * N + s * w: b * N + (s + 1) * w]
            r = [sum(Ml[s][e + dl - u] * rho[u] for u in range(e, dl)) % p for e in range(dl)]
            for i in range(dl):
                acc = 0
                for c in reversed(r):
                    acc = (acc * xs[base + i] + c) % p
                out[b * k + base + i] = acc
    return out


def multieval_rows(p, C, d, batch, xs, tree=None):
    """tree_down over `batch` rows of C (batch × d, flat): the root's rows, then per level the shared node spectra met
    with every row, the extraction over batch·P parents, and the leaves over every row."""
    k = len(xs)
    levels, K, lb, N = tree or product_tree(p, xs, B)
    M = levels[K][0]
    hl = min(k + 1, d)
    G = series_inverse(p, [M[k - i] for i in range(hl)], d) + [0]          # the shared inverse, zero word d
    FR = [C[b * d + d - 1 - i] for b in range(batch) for i in range(d)]    # reverse_rows: stride d
    H = []
    for b in range(batch):                                                 # rows of 2d words against G
        H += (_mul(p, FR[b * d:(b + 1) * d], G) + [0] * (2 * d))[:2 * d]
    R = [H[b * 2 * d + d - 1 - u] if u < min(d, k) else 0 for b in range(batch) for u in range(N)]
    for j in range(K - 1, lb - 1, -1):
        D, w, P = 2 << j, 1 << j, N >> (j + 1)
        PA, PB = [0] * (batch * N), [0] * (batch * N)
        for i in range(batch * P):   # parent i of the flat buffer: node i & (P - 1) of its level
            il = i & (P - 1)
            PA[i * D:(i + 1) * D] = cyclic(p, levels[j][2 * il], R[i * D:(i + 1) * D], D)
            PB[i * D:(i + 1) * D] = cyclic(p, levels[j][2 * il + 1], R[i * D:(i + 1) * D], D)
        Rn = [0] * (batch * N)
        for x in range(batch * N):   # tree_extract_kernel: nchild = 2·batch·P, pmask = P - 1
            c, u = x >> j, x & (w - 1)
            i = c >> 1
            il = i & (P - 1)
            dl, dr = node_deg(k, j, 2 * il), node_deg(k, j, 2 * il + 1)
            Rn[x] = (PA[2 * i * w + dl + u] if u < dr else 0) if c & 1 else (PB[2 * i * w + dr + u] if u < dl else 0)
        R = Rn
    return eval_leaves(p, levels[lb], R, xs, k, lb, N, batch)


def interpolate_rows(p, xs, Y, batch):
    """tree_interpolate from batch 2: M'(x_i) as one row, inverted once; the leaves kernel over every row with
    y_{b,i}·M'(x_i)^-1 fused in; the up-sweep over batch·P parents against the shared node spectra."""
    tree = product_tree(p, xs, B)
    levels, K, lb, N = tree
    k = len(xs)
    M = levels[K][0]
    W = multieval_rows(p, [(i + 1) * M[i + 1] % p for i in range(k)], k, 1, xs, tree)
    scale = [pow(v, -1, p) for v in W]
    R = [0] * (batch * N)
    for b in range(batch):                 # tree_leaves_kernel<INTERP> at blockIdx.y = b
        for s in range(N >> lb):
            base = s << lb
            r = [[Y[b * k + base + i] * scale[base + i] % p] if base + i < k else [0] for i in range(1 << lb)]
            m = [[(-xs[base + i]) % p, 1] if base + i < k else [1, 0] for i in range(1 << lb)]
            for j in range(lb):
                r = [[(a + c) % p for a, c in zip(_mul(p, r[2 * i], m[2 * i + 1])[:2 << j],
                                                   _mul(p, r[2 * i + 1], m[2 * i])[:2 << j])] for i in range(len(r) // 2)]
                m = [_mul(p, m[2 * i], m[2 * i + 1]) for i in range(len(m) // 2)]
            assert m[0] == levels[lb][s]
            R[b * N + base: b * N + base + (1 << lb)] = (r[0] + [0] * (1 << lb))[:1 << lb]
    for j in range(lb, K):
        D, w, P = 2 << j, 1 << j, N >> (j + 1)
        Rn = [0] * (batch * N)
        for i in range(batch * P):   # spread over batch·P parents; tree_node_mac_kernel against node i & (P - 1)
            il = i & (P - 1)
            rl, rr = R[2 * i * w:(2 * i + 1) * w], R[(2 * i + 1) * w:(2 * i + 2) * w]
            Rn[i * D:(i + 1) * D] = [(a + c) % p for a, c in zip(cyclic(p, rl, levels[j][2 * il + 1], D),
                                                                 cyclic(p, rr, levels[j][2 * il], D))]
        R = Rn
    return [R[b * N + i] for b in range(batch) for i in range(k)]


def interp_literal_rows(p, xs, Y, batch):
    """interp_nodes_kernel / interp_sum_kernel over grid (⌈k/256⌉, rows): partial[(b·nwarps + warp)·k + i - 1] is the
    sum over warp's nodes j of c_{b,j}·q_j[i - 1], and out[b·k + i] sums the row's nwarps partials."""
    k = len(xs)
    Mm = [1]
    for x in xs:
        Mm = _mul(p, Mm, [(-x) % p, 1])
    nwarps = (k + 255) // 256 * 8
    partial = [0] * (batch * nwarps * k)
    for j in range(nwarps * 32):
        if j >= k:
            continue
        x, qv, dd, q = xs[j], 0, 0, [0] * k
        for i in range(k, 0, -1):
            qv = (Mm[i] + qv * x) % p
            q[i - 1] = qv
            dd = (dd * x + qv) % p
        dinv = pow(dd, -1, p)
        for b in range(batch):
            c = Y[b * k + j] * dinv % p
            for i in range(k):
                at = (b * nwarps + (j >> 5)) * k + i
                partial[at] = (partial[at] + c * q[i]) % p
    return [sum(partial[(b * nwarps + w) * k + i] for w in range(nwarps)) % p for b in range(batch) for i in range(k)]


def _points(p, k, seed, distinct):
    xs = [int(v) for v in oracle.splitmix(p, seed, k)]
    if k >= 3:
        xs[0], xs[k // 2] = 0, p - 1
    if not distinct and k >= 4:
        xs[2] = xs[1]
    assert not distinct or len(set(xs)) == k
    return xs


@pytest.mark.parametrize("batch", BATCHES)
@pytest.mark.parametrize("k", SIZES)
@pytest.mark.parametrize("name", list(PRIMES))
def test_multieval_rows(name, k, batch):
    p = PRIMES[name]
    xs = _points(p, k, 70 + k, distinct=False)
    tree = product_tree(p, xs, B)
    for d in sorted({1, max(1, k // 2), k + 3}):
        C = [int(v) for v in oracle.splitmix(p, 80 + d + batch, batch * d)]
        got = multieval_rows(p, C, d, batch, xs, tree)
        for b in range(batch):
            f = np.array(C[b * d:(b + 1) * d], np.uint64)
            assert got[b * k:(b + 1) * k] == [oracle.poly_eval_horner(p, f, x) for x in xs], (b, d)


@pytest.mark.parametrize("batch", BATCHES)
@pytest.mark.parametrize("k", SIZES)
@pytest.mark.parametrize("name", list(PRIMES))
def test_interpolate_rows(name, k, batch):
    p = PRIMES[name]
    xs = _points(p, k, 90 + k, distinct=True)
    Y = [int(v) for v in oracle.splitmix(p, 95 + batch, batch * k)]
    got = interpolate_rows(p, xs, Y, batch)
    for b in range(batch):
        f = np.array(got[b * k:(b + 1) * k], np.uint64)
        assert [oracle.poly_eval_horner(p, f, x) for x in xs] == Y[b * k:(b + 1) * k], b


@pytest.mark.parametrize("batch", BATCHES)
@pytest.mark.parametrize("k", [1, 3, 63, 300])
@pytest.mark.parametrize("p", [101, GL])
def test_literal_interpolation_rows(p, k, batch):
    if k >= p:
        pytest.skip("more nodes than field elements")
    xs = list(range(1, k + 1)) if p == 101 else _points(p, k, 97 + k, distinct=True)
    Y = [int(v) for v in oracle.splitmix(p, 98 + batch, batch * k)]
    got = interp_literal_rows(p, xs, Y, batch)
    for b in range(batch):
        want = oracle.rs_decode(p, np.array(xs, np.uint64), np.array(Y[b * k:(b + 1) * k], np.uint64), k) if k <= 12 else None
        row = got[b * k:(b + 1) * k]
        if want is not None:
            assert row == [int(v) for v in want]
        assert [oracle.poly_eval_horner(p, np.array(row, np.uint64), x) for x in xs] == Y[b * k:(b + 1) * k]


def test_log2_ceil_matches_the_tree_shape():
    assert [_log2_ceil(v) for v in (1, 2, 3, 64, 65, 1000)] == [0, 1, 2, 6, 7, 10]
