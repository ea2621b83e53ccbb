"""CPU emulation of the coset transforms (tests/emu/coset_emu.cpp compiles the COSET load and store phases of the tile
kernel and the COSET rounds of the 256-point-tile passes for the host and runs them thread by thread, as ntt.cu
launches them) against a Python-integer model: X[k] = Σ_j a_j (s·ω^k)^j, and its inverse."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle
from gpu_util import BABYBEAR, PBIG

GL = oracle.GOLDILOCKS
P64 = C.POINTER(C.c_uint64)
_HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def emu():
    csrc = os.path.join(_HERE, "..", "ronkathon_b200", "csrc")
    src = os.path.join(_HERE, "emu", "coset_emu.cpp")
    so = os.path.join(_HERE, "emu", "libcoset_emu.so")
    deps = [src] + [os.path.join(csrc, h) for h in ("ntt_kernel.cuh", "ntt3_kernel.cuh", "field.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(x) for x in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", so, src])
    lib = C.CDLL(so)
    lib.emu_ntt_coset.argtypes = [C.c_uint64, C.c_uint64, P64, C.c_uint32, C.c_uint32, C.c_uint64, C.c_int]
    lib.emu_ntt3_coset.argtypes = [P64, C.c_uint32, C.c_uint32, C.c_uint64, C.c_int]
    return lib


def _ptr(a):
    return a.ctypes.data_as(P64)


def scaled(p, a, c):
    """a ⊙ c^j, j the index within each row (rows are the last axis)."""
    n = a.shape[-1]
    pw = np.empty(n, dtype=np.uint64)
    v = 1
    for j in range(n):
        pw[j] = v
        v = v * c % p
    return np.stack([oracle.vec_mul(p, r, pw) for r in a.reshape(-1, n)]).reshape(a.shape)


def coset_model(p, g, a, s, inverse=False):
    """Rows of a (batch × n): the forward coset transform NTT(a ⊙ s^j), or the inverse INTT(a) ⊙ s^-j."""
    n = a.shape[-1]
    if inverse:
        return scaled(p, np.stack([oracle.ntt_fast(p, r, inverse=True, g=g) for r in a]), pow(s, p - 2, p))
    return np.stack([oracle.ntt_fast(p, r, g=g) for r in scaled(p, a, s)])


def horner(p, row, x):
    acc = 0
    for c in reversed([int(v) for v in row]):
        acc = (acc * x + c) % p
    return acc


# (p, g, 2-adicity): Goldilocks on its shift policy and on the Montgomery one, two Montgomery primes
FIELDS = [(GL, 7, 32), (GL, pow(7, 5, GL), 32), (BABYBEAR, 31, 27), (PBIG, 3, 28)]


def shifts(p, g):
    return [g, p - 1, int(oracle.splitmix(p, 99, 1)[0]) or 2]


# the single-tile kernel (n ≤ 2^13) at its edges, and the generic pass pair from 2^14
@pytest.mark.parametrize("log_n", [1, 4, 5, 9, 12, 13, 14, 15])
@pytest.mark.parametrize("batch", [1, 3])
@pytest.mark.parametrize("p,g,adicity", FIELDS)
def test_tile_coset_matches_model(emu, p, g, adicity, log_n, batch):
    n = 1 << log_n
    a = oracle.splitmix(p, 7 * log_n + batch, batch * n).reshape(batch, n)
    a[0, 0], a[-1, -1] = p - 1, p - 1
    for s in shifts(p, g):
        fwd = a.copy()
        assert emu.emu_ntt_coset(p, g, _ptr(fwd), log_n, batch, s, 0) == 0
        want = coset_model(p, g, a, s)
        assert np.array_equal(fwd, want), (s, "forward")
        if log_n <= 5:   # the definition itself, point by point
            w = pow(g, (p - 1) >> log_n, p)
            for r in range(batch):
                assert [horner(p, a[r], s * pow(w, k, p) % p) for k in range(n)] == [int(v) for v in fwd[r]]
        inv = fwd.copy()
        assert emu.emu_ntt_coset(p, g, _ptr(inv), log_n, batch, s, 1) == 0
        assert np.array_equal(inv, a), (s, "inverse")


@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("batch", [1, 3])
def test_three_pass_coset_matches_model(emu, batch, inverse):
    """Goldilocks with g = 7 at 2^21, the smallest size of the 256-point-tile coset passes (pass 1 of 32 points)."""
    log_n, n = 21, 1 << 21
    a = oracle.splitmix(GL, 21 + batch, batch * n).reshape(batch, n)
    s = int(oracle.splitmix(GL, 5, 1)[0])
    got = a.copy()
    assert emu.emu_ntt3_coset(_ptr(got), log_n, batch, s, inverse) == 0
    assert np.array_equal(got, coset_model(GL, 7, a, s, inverse=bool(inverse)))


def test_refuses_what_it_does_not_cover(emu):
    a = np.zeros(16, dtype=np.uint64)
    assert emu.emu_ntt_coset(101, 2, _ptr(a), 3, 1, 5, 0) == 1     # 8 does not divide 100
    assert emu.emu_ntt3_coset(_ptr(a), 20, 1, 5, 0) == 1            # the tile passes cover 2^21 … 2^24
