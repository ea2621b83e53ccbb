"""The context's scratch stack: every per-call device buffer (staged `_host` arguments, operands, the subproduct tree,
Newton's buffers, transform workspaces, commit partials) is a region of one stack of device blocks, taken by the
function that needs it and given back when it returns.

  1. Growth: on one fresh context each entry point runs small, then large, then every small call again.  The first
     case, multieval over the same 2^16 points with 1000 and then 2^20 coefficients, grows under a live region: the
     tree fills the first block exactly, so tree_down's buffers and Newton's transform workspaces replace the blocks
     above it while the tree is in use.  The other cases grow their outermost region first (staging, Newton's
     buffers) and then new blocks above it.  Each result equals, bit for bit, the same call on a context that has
     run nothing before it, and the oracle where that is cheap.
  2. Steady state: after larger calls, calls that fit the blocks held allocate, free and wait for nothing.  They run
     behind a gate on the context's stream, built as in test_gpu_streams.py, and the stream must still be busy when
     each returns (no synchronise).  The blocks come from the device's default memory pool in stream order, which
     never waits, so the pool's counters show the rest: its use never rose (nothing allocated) and its use and
     reservation are unchanged (nothing given back).
"""
import os

import numpy as np
import pytest

import oracle
from gpu_util import GL, ctx, dev, host, msm_inputs

pytestmark = pytest.mark.gpu

ENV = {"RONK_TREE_MIN": "1", "RONK_MSM_COORD": "0"}   # the tree at every size it fits; the histogram commit path
SLEEP_CYCLES = 100_000_000   # torch.cuda._sleep: about 50 ms at the H100 SXM's 1.98 GHz boost clock, longer below it


def _p(x):
    from ronkathon_b200 import _lib
    return _lib._ptr(x)


def _context(stream=None, env=ENV):
    """A fresh Context on `stream` (a torch stream; default: torch's current one), with the switches of `env`."""
    import torch
    from ronkathon_b200 import Context
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return Context(0, (stream or torch.cuda.current_stream()).cuda_stream)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _points(n, seed):
    x = oracle.splitmix(GL, seed, n)
    assert len(np.unique(x)) == n
    return x


# ---- 1. growth under live regions --------------------------------------------------------------------------------------
# name → (small size, large size, call(c, size) → result words, oracle check of the small result)
MULTIEVAL_POINTS = 1 << 16


def _multieval(c, d):
    """tree (the same for every d) → tree_down → Newton → transform workspace"""
    from ronkathon_b200 import ops
    xs, f = _points(MULTIEVAL_POINTS, 20), oracle.splitmix(GL, 21, d)
    return host(ops.poly_multieval(c, dev(f), dev(xs)))


def _multieval_check(d, got):
    xs, f = _points(MULTIEVAL_POINTS, 20), oracle.splitmix(GL, 21, d)
    for i in range(0, MULTIEVAL_POINTS, 2047):
        assert oracle.poly_eval_horner(GL, f, int(xs[i])) == got[i], i


def _poly_mul_host(c, n):
    """stage → operands → transform workspace"""
    a, b = oracle.splitmix(GL, 1, n), oracle.splitmix(GL, 2, n)
    out = np.empty(2 * n - 1, np.uint64)
    c.call("ronk_poly_mul_u64_host", GL, 7, _p(a), n, _p(b), n, _p(out))
    return out


def _poly_mul_check(n, got):
    assert np.array_equal(got, oracle.poly_mul(GL, oracle.splitmix(GL, 1, n), oracle.splitmix(GL, 2, n)))


def _divrem_inputs(da):
    a, b = oracle.splitmix(GL, 3, da), oracle.splitmix(GL, 4, da // 2 + 1)
    b[-1] = b[-1] % (GL - 1) + 1   # nonzero top word: the Newton path
    return a, b


def _divrem(c, da):
    """Newton's buffers → transform workspace"""
    from ronkathon_b200 import ops
    a, b = _divrem_inputs(da)
    q, r = ops.poly_divrem(c, dev(a), dev(b))
    return np.concatenate([host(q), host(r)])


def _divrem_check(da, got):
    q, r = oracle.poly_divrem(GL, *_divrem_inputs(da))
    assert np.array_equal(got, np.concatenate([q, r]))


def _tree_inputs(k):
    return _points(k, 5), oracle.splitmix(GL, 6, k), oracle.splitmix(GL, 7, k)


def _tree(c, k):
    """tree → tree_down → Newton → transform workspace: the interpolant through (xs, ys), then f at xs"""
    from ronkathon_b200 import ops
    xs, ys, f = _tree_inputs(k)
    X = dev(xs)
    return np.concatenate([host(ops.poly_interpolate(c, X, dev(ys))), host(ops.poly_multieval(c, dev(f), X))])


def _tree_check(k, got):
    xs, ys, f = _tree_inputs(k)
    for i, x in enumerate(xs):
        assert oracle.poly_eval_horner(GL, got[:k], int(x)) == ys[i], i
        assert oracle.poly_eval_horner(GL, f, int(x)) == got[k + i], i


def _interp_host(c, k):
    """stage (inputs, output and the literal kernels' scratch)"""
    xs, ys, _ = _tree_inputs(k)
    out = np.empty(k, np.uint64)
    c.call("ronk_poly_interpolate_u64_host", GL, _p(xs), _p(ys), k, _p(out))
    return out


def _interp_host_check(k, got):
    xs, ys, _ = _tree_inputs(k)
    for i, x in enumerate(xs):
        assert oracle.poly_eval_horner(GL, got, int(x)) == ys[i], i


def _commit(c, n):
    """the histogram path's partial histograms"""
    import torch
    from ronkathon_b200 import ops
    pts, sc = msm_inputs(n, 8, 9)
    return np.frombuffer(ops.msm(c, torch.from_numpy(pts).cuda(), torch.from_numpy(sc).cuda()), np.uint8)


def _commit_check(n, got):
    pts, sc = msm_inputs(n, 8, 9)
    assert got.tobytes() == oracle.commit(sc, pts, fast=True)


CASES = {
    "multieval_under_tree": (1000, 1 << 20, _multieval, _multieval_check),   # first: on the fresh context
    "poly_mul_host": (300, 1 << 20, _poly_mul_host, _poly_mul_check),
    "divrem_newton": (1 << 12, 1 << 22, _divrem, _divrem_check),
    "tree": (100, 1 << 16, _tree, _tree_check),
    "interpolate_host": (100, 8192, _interp_host, _interp_host_check),
    "commit_hist": (1 << 12, 1 << 22, _commit, _commit_check),
}


def _fresh(call, size):
    c = _context()
    try:
        return call(c, size)
    finally:
        c.close()


def test_growth_under_live_regions():
    """On one fresh context, each case small then large, then every small case again on the grown blocks."""
    c = _context()
    try:
        for name, (small, large, call, check) in CASES.items():
            for size in (small, large):
                got = call(c, size)
                assert np.array_equal(got, _fresh(call, size)), (name, size)
                if size == small:
                    check(size, got)
        for name, (small, _, call, check) in CASES.items():
            got = call(c, small)
            assert np.array_equal(got, _fresh(call, small)), name
            check(small, got)
    finally:
        c.close()


# ---- 2. steady state after larger calls ------------------------------------------------------------------------------
class _DefaultPool:
    """Device 0's default memory pool, which the scratch blocks come from, read through the driver API."""
    RESERVED_MEM_CURRENT, USED_MEM_CURRENT, USED_MEM_HIGH = 5, 7, 8   # CUmemPool_attribute

    def __init__(self):
        import ctypes as C
        self.C, self.cu = C, C.CDLL("libcuda.so.1")
        self.cu.cuMemPoolGetAttribute.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        self.cu.cuMemPoolSetAttribute.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        self.cu.cuMemPoolTrimTo.argtypes = [C.c_void_p, C.c_size_t]
        dev, self.pool = C.c_int(), C.c_void_p()
        assert self.cu.cuDeviceGet(C.byref(dev), 0) == 0
        assert self.cu.cuDeviceGetDefaultMemPool(C.byref(self.pool), dev) == 0

    def get(self, attr):
        v = self.C.c_uint64()
        assert self.cu.cuMemPoolGetAttribute(self.pool, attr, self.C.byref(v)) == 0
        return v.value

    def settle(self):
        """Returns the pool's unused memory and resets its high-water mark of use: afterwards the reservation moves
        only when a block is allocated or freed, and the mark rises above the current use only when one is allocated."""
        assert self.cu.cuMemPoolTrimTo(self.pool, 0) == 0
        zero = self.C.c_uint64(0)
        assert self.cu.cuMemPoolSetAttribute(self.pool, self.USED_MEM_HIGH, self.C.byref(zero)) == 0

    def counters(self):
        return {"reserved": self.get(self.RESERVED_MEM_CURRENT), "used": self.get(self.USED_MEM_CURRENT),
                "used_high": self.get(self.USED_MEM_HIGH)}


@pytest.fixture
def gate():
    """A fresh context c on a non-blocking stream s, and behind(fn): fn(c) enqueued on s behind a spin of about 50 ms
    (torch.cuda._sleep).  behind asserts that s is still busy when fn returns: fn synchronised nothing and waited for
    nothing.  Every kernel fn launches must have run once in the process before (the first launch of a kernel loads
    its module, which waits for the device)."""
    import torch
    s = torch.cuda.Stream()
    c = _context(s, env={})

    def behind(fn):
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            torch.cuda._sleep(SLEEP_CYCLES)
            fn(c)
            assert not s.query(), "s finished before the call returned: the gate was too short, or the call waited"
        s.synchronize()

    yield c, s, behind
    s.synchronize()
    c.close()


def test_smaller_calls_fit_the_blocks_of_larger_ones(gate):
    """After a 2^23 × 2^23 poly_mul (256 MiB of operands, a 128 MiB transform workspace) and a 2^24-point transform, a
    2^18-point transform and a 2^17 × 2^17 poly_mul fit the blocks held: behind the gate, with the default pool's
    counters unchanged.  Both need a transform workspace: the 2^16-point
    transform of batch 1 runs on the cluster kernel and products up to 2^13 points are single-tile, so neither takes
    any."""
    import torch
    from ronkathon_b200 import ops
    c, s, behind = gate
    big, n17 = 1 << 23, 1 << 17
    x = ops.splitmix_fill(ctx(), 1 << 18, 11, GL)
    a, b = ops.splitmix_fill(ctx(), n17, 12, GL), ops.splitmix_fill(ctx(), n17, 13, GL)
    # the same calls on the suite's context first: they load every kernel the gated calls launch
    want_x = x.clone()
    ctx().call("ronk_ntt_u64", GL, 7, _p(want_x), 18, 1, 0)
    want_ab = ops.poly_mul(ctx(), a, b)
    ctx().sync()
    assert np.array_equal(ops.to_host(want_x), oracle.ntt_fast(GL, ops.to_host(x)))

    with torch.cuda.stream(s):
        pa, pb = ops.splitmix_fill(c, big, 14, GL), ops.splitmix_fill(c, big, 15, GL)
        pc = torch.empty(2 * big - 1, dtype=torch.int64, device="cuda")
        c.call("ronk_poly_mul_u64", GL, 7, _p(pa), big, _p(pb), big, _p(pc))
        y = ops.splitmix_fill(c, 1 << 24, 16, GL)
        c.call("ronk_ntt_u64", GL, 7, _p(y), 24, 1, 0)
    s.synchronize()
    del pa, pb, pc, y

    got_x = x.clone()
    got_ab = torch.empty(2 * n17 - 1, dtype=torch.int64, device="cuda")
    pool = _DefaultPool()
    torch.cuda.synchronize()
    pool.settle()
    before = pool.counters()
    assert before["used"] >= (256 + 128) << 20, before   # the blocks of the larger calls are held
    behind(lambda c: c.call("ronk_ntt_u64", GL, 7, _p(got_x), 18, 1, 0))
    behind(lambda c: c.call("ronk_poly_mul_u64", GL, 7, _p(a), n17, _p(b), n17, _p(got_ab)))
    after = pool.counters()
    assert after["used_high"] <= before["used"], (before, after)    # nothing allocated
    assert (after["used"], after["reserved"]) == (before["used"], before["reserved"]), (before, after)   # nothing freed
    assert torch.equal(got_x, want_x)
    assert torch.equal(got_ab, want_ab)
