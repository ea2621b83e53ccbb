"""Shared helpers for the -m gpu tests: one Context on torch's current stream, seeded inputs, and exact
references in Python integers (importable without a GPU)."""
import numpy as np
import pytest

import oracle

GL = oracle.GOLDILOCKS
_ctx = None

# Test primes for the run-time-modulus (Montgomery, R = 2^64) policy, which every (p, g) except Goldilocks with g = 7
# takes: name → (p, g, 2-adicity).  Each g is a quadratic non-residue, so ω = g^((p-1)/n) has order exactly n for
# every n = 2^k up to the 2-adicity.
BABYBEAR = 2013265921          # 15·2^27 + 1
PBIG = 0xFFFFFFFF70000001      # above 2^63 and not Goldilocks: the subtractive REDC at every size
MONT_PRIMES = {
    "babybear": (BABYBEAR, 31, 27),                         # p < 2^31, every size to 2^26
    "koalabear": (2130706433, 3, 24),                       # 127·2^24 + 1
    "p32": (4295294977, 5, 16),                             # 0x100050001: residues straddle the 32-bit word boundary
    "p57": (4179340454199820289, 3, 57),                    # 29·2^57 + 1
    "pbig": (PBIG, 3, 28),
    "gl_g5": (GL, pow(7, 5, GL), 32),                       # Goldilocks through the Montgomery kernels: ω' = ω^5
    "p2adic3": ((1 << 64) - 279, 5, 3),                     # above 2^63, partial radix-16 constant table, n ≤ 8
}
for _name, (_p, _g, _s) in MONT_PRIMES.items():
    assert pow(_g, (_p - 1) // 2, _p) == _p - 1, _name
    assert ((_p - 1) & -(_p - 1)).bit_length() - 1 == _s, _name


def s64(v):
    """A uint64 residue as the int64 torch stores it."""
    return int(np.array([v], dtype=np.uint64).view(np.int64)[0])


def ctx():
    global _ctx
    import torch
    from ronkathon_b200 import Context, set_default_context
    if _ctx is None:
        assert torch.cuda.is_available(), "GPU tests need an H100"
        torch.cuda.set_device(0)
        _ctx = Context(0, torch.cuda.current_stream().cuda_stream)
        set_default_context(_ctx)
    return _ctx


def dev(a):
    from ronkathon_b200 import ops
    return ops.to_device(np.ascontiguousarray(a, dtype=np.uint64))


def host(t):
    from ronkathon_b200 import ops
    ctx().sync()
    return ops.to_host(t)


def summary(x):
    idx = np.arange(1, len(x) + 1, dtype=np.uint64)
    with np.errstate(over="ignore"):
        return {"first": int(x[0]), "second": int(x[1]), "last": int(x[-1]),
                "sum_mod_2_64": int(np.sum(x, dtype=np.uint64)),
                "weighted_sum_mod_2_64": int(np.sum(x * idx, dtype=np.uint64)),
                "xor": int(np.bitwise_xor.reduce(x))}


def msm_inputs(n, seed_pts=44, seed_sc=45):
    """SURVEY §8d: points k·G1 + l·G2 with (k,l) from splitmix(seed 44) mod 17, scalars seed 45."""
    G1, G2 = bytes([1, 0, 2, 0]), bytes([36, 0, 0, 31])
    table = {}
    for k in range(17):
        for l in range(17):
            table[(k, l)] = oracle.point_add(oracle.point_smul(G1, k), oracle.point_smul(G2, l))
    kl = oracle.splitmix(17, seed_pts, 2 * n).astype(np.int64)
    lut = np.zeros((17, 17, 4), dtype=np.uint8)
    for (k, l), v in table.items():
        lut[k, l] = np.frombuffer(v, dtype=np.uint8)
    pts = lut[kl[0::2], kl[1::2]]
    sc = oracle.splitmix(17, seed_sc, n).astype(np.uint8)
    return np.ascontiguousarray(pts), sc


def lagrange_closed_form(p, g, c, x):
    """L(x) = (x^n - 1)/n · Σ_j c_j ω^j / (x - ω^j) with Python ints — the barycentric form on the roots of unity,
    whose weights are ω^j/n.  At a node the reference's fold is multiplied by l(x) = 0, so the value is 0."""
    n = len(c)
    w = pow(g, (p - 1) // n, p)
    xn1 = (pow(x, n, p) - 1) % p
    if xn1 == 0:
        return 0
    acc, wj = 0, 1
    for cj in c:
        acc = (acc + int(cj) * wj * pow((x - wj) % p, -1, p)) % p
        wj = wj * w % p
    return xn1 * pow(n, -1, p) * acc % p
