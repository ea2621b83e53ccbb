"""CPU emulation of the fused batched product (tests/emu/polymul_emu.cpp compiles polymul_kernel.cuh's device phases for
the host and runs polymul_fused_kernel's data flow tile by tile, thread by thread) against the oracle's schoolbook
product, and a bank-conflict audit of the kernel's own shared-memory access patterns."""
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
    src = os.path.join(_HERE, "emu", "polymul_emu.cpp")
    so = os.path.join(_HERE, "emu", "libpolymul_emu.so")
    deps = [src] + [os.path.join(csrc, h) for h in ("polymul_kernel.cuh", "ntt_kernel.cuh", "field.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(x) for x in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", so, src])
    lib = C.CDLL(so)
    lib.emu_poly_mul_fused.argtypes = [C.c_uint64, C.c_uint64, P64, C.c_uint32, P64, C.c_uint32, C.c_int, C.c_uint64, P64]
    lib.emu_polymul_worst_conflict.argtypes = [C.c_uint32, C.c_uint32, C.c_int]
    return lib


def _ptr(a):
    return a.ctypes.data_as(P64)


# (p, g): Goldilocks on its shift policy and on the Montgomery one, and two Montgomery primes
FIELDS = [(GL, 7), (GL, pow(7, 5, GL)), (BABYBEAR, 31), (PBIG, 3)]
TILE = 1 << 11


@pytest.mark.parametrize("shared", [0, 1])
@pytest.mark.parametrize("da,db,batch", [
    (1, 2, 3), (3, 5, 7), (9, 9, 300), (17, 16, 130),   # several products per tile, odd da and db, a partial last tile
    (1, 64, 65), (64, 1, 31), (100, 157, 9), (7, 1000, 5), (513, 512, 5), (1024, 1025, 3),
])
@pytest.mark.parametrize("p,g", FIELDS)
def test_fused_data_flow_matches_oracle(emu, p, g, da, db, batch, shared):
    a = oracle.splitmix(p, da + 3 * db, batch * da)
    b = oracle.splitmix(p, db + 5 * da, db if shared else batch * db)
    a[0], b[-1] = p - 1, p - 1
    L = da + db - 1
    c = np.full(batch * L + 5, 0xDEADBEEF, dtype=np.uint64)
    assert emu.emu_poly_mul_fused(p, g, _ptr(a), da, _ptr(b), db, shared, batch, _ptr(c)) == 0
    assert np.all(c[batch * L:] == 0xDEADBEEF), "wrote past c[batch·L)"
    got = c[:batch * L].reshape(batch, L)
    rows = range(batch) if batch * da * db <= 1 << 20 else (0, 1, batch // 2, batch - 2, batch - 1)
    for r in rows:
        brow = b if shared else b[r * db:(r + 1) * db]
        assert np.array_equal(got[r], oracle.poly_mul(p, a[r * da:(r + 1) * da], brow)), r


def test_fused_refuses_what_it_does_not_cover(emu):
    a = np.ones(2048, dtype=np.uint64)
    c = np.zeros(4096, dtype=np.uint64)
    assert emu.emu_poly_mul_fused(GL, 7, _ptr(a), 1024, _ptr(a), 1026, 0, 1, _ptr(c)) == 1   # N = 2^12 > the cap
    assert emu.emu_poly_mul_fused(101, 2, _ptr(a), 3, _ptr(a), 3, 0, 1, _ptr(c)) == 1        # 8 does not divide 100
    assert emu.emu_poly_mul_fused(GL, 0, _ptr(a), 3, _ptr(a), 3, 0, 1, _ptr(c)) == 1         # g = 0


@pytest.mark.parametrize("log_n", range(1, 12))
def test_bit_reversal_permutation_is_conflict_free(emu, log_n):
    assert emu.emu_polymul_worst_conflict(log_n, 0, 1) == 1


@pytest.mark.parametrize("log_n", range(1, 12))
def test_row_strided_scatter_and_store_conflicts_are_bounded(emu, log_n):
    """The load's scatter (rows of every d ≤ N words) and the store's gather (rows of L words, N/2 < L ≤ N) walk
    contiguous runs of rows.  Inside a row the lanes hit distinct banks; a half-warp that straddles row boundaries
    lands up to 4 (scatter) or 3 (store) lanes on one bank.  Both phases are bound by their HBM traffic; the bound is
    what the swizzle gives today, so a layout change that makes it worse shows here."""
    n = 1 << log_n
    assert max(emu.emu_polymul_worst_conflict(log_n, d, 0) for d in range(1, n + 1)) <= 4
    assert max(emu.emu_polymul_worst_conflict(log_n, L, 2) for L in range(n // 2 + 1, n + 1)) <= 3
    if log_n in (1, 11):    # one row of N words, or single-word rows two apart: conflict-free
        assert emu.emu_polymul_worst_conflict(log_n, n, 0) == 1 and emu.emu_polymul_worst_conflict(log_n, n, 2) == 1
