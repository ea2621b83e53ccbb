"""ronk_poly_mul_batch_u64: many polynomial products in one call, on the device.

The exact reference of every row is ronk_poly_mul_u64 on that row's pair; small shapes are also checked against the
oracle's schoolbook product.  Every call is laid out in poisoned buffers: the operands are views with 0xFFFF…FFFF words
(no residue of any test prime, so reading one changes the result) in front of and behind them, and c has guard words on
both sides that must stay untouched.  A refused call must leave c unwritten.  The launch names of the profile pin the
path each case claims to cover: the fused kernel is one launch whatever the batch."""
import os

import numpy as np
import pytest

import oracle
from gpu_util import GL, MONT_PRIMES, ctx, dev, host

pytestmark = pytest.mark.gpu

POISON = -1
GUARD = 0x5A5A5A5A5A5A5A5
FRONT, BACK = 13, 77
TABLE_BUILDS = {"pow_table", "tw2d_gather", "interpass_table", "ntt3_t1", "ntt3_t2"}
PRIMES = {"gl": (GL, 7), **{n: (p, g) for n, (p, g, _) in MONT_PRIMES.items()},
          "f101": (101, oracle.generator(101)), "f17": (17, oracle.generator(17)), "f127": (127, oracle.generator(127)),
          "gl_g0": (GL, 0)}
_contexts = {}


def context(path=0):
    """The suite's context, or one created with RONK_POLY_BATCH_PATH=path (read once, at creation)."""
    import torch
    from ronkathon_b200 import Context
    c = ctx()
    if not path:
        return c
    if path not in _contexts:
        os.environ["RONK_POLY_BATCH_PATH"] = str(path)
        try:
            _contexts[path] = Context(0, torch.cuda.current_stream().cuda_stream)
        finally:
            del os.environ["RONK_POLY_BATCH_PATH"]
    return _contexts[path]


def poisoned(rows, front=FRONT):
    """A device view holding `rows` (flat) with poison words in front of and behind it."""
    import torch
    flat = np.ascontiguousarray(rows, dtype=np.uint64).reshape(-1)
    buf = torch.full((front + flat.size + BACK,), POISON, dtype=torch.int64, device="cuda")
    view = buf[front:front + flat.size]
    view.copy_(dev(flat))
    return buf, view


class Call:
    """One ronk_poly_mul_batch_u64 call in poisoned buffers; .c is the batch × L result after run()."""

    def __init__(self, p, g, a, b, shared, offsets=(0, 0, 0)):
        import torch
        self.p, self.g, self.a, self.b, self.shared = p, g, a, b, shared
        self.batch, self.da = a.shape
        self.db = b.shape[-1]
        self.L = self.da + self.db - 1
        self.A, self.av = poisoned(a, FRONT + offsets[0])
        self.B, self.bv = poisoned(b, FRONT + offsets[1])
        oc = FRONT + offsets[2]
        self.C = torch.full((oc + self.batch * self.L + BACK,), GUARD, dtype=torch.int64, device="cuda")
        self.oc = oc
        self.cv = self.C[oc:oc + self.batch * self.L]

    def run(self, c=None, batch=None):
        from ronkathon_b200 import _lib
        c = c or context()
        c.call("ronk_poly_mul_batch_u64", self.p, self.g, _lib._ptr(self.av), self.da, _lib._ptr(self.bv), self.db,
               int(self.shared), self.batch if batch is None else batch, _lib._ptr(self.cv))
        return self

    def result(self):
        C = host(self.C).view(np.int64)
        assert np.all(C[:self.oc] == GUARD) and np.all(C[self.oc + self.batch * self.L:] == GUARD), "guard word written"
        A, B = host(self.A).view(np.int64), host(self.B).view(np.int64)
        assert np.count_nonzero(A == POISON) == A.size - self.a.size, "operand a changed"
        assert np.count_nonzero(B == POISON) == B.size - self.b.size, "operand b changed"
        return C[self.oc:self.oc + self.batch * self.L].view(np.uint64).reshape(self.batch, self.L)

    def unwritten(self):
        return bool(np.all(host(self.C).view(np.int64) == GUARD))


def single(p, g, a_row, b_row):
    """ronk_poly_mul_u64 of one pair: the reference of every row."""
    import torch
    from ronkathon_b200 import _lib
    a, b = dev(a_row), dev(b_row)
    c = torch.empty(a.numel() + b.numel() - 1, dtype=torch.int64, device="cuda")
    ctx().call("ronk_poly_mul_u64", p, g, _lib._ptr(a), a.numel(), _lib._ptr(b), b.numel(), _lib._ptr(c))
    return host(c)


def operands(p, da, db, batch, shared, seed):
    a = oracle.splitmix(p, seed, batch * da).reshape(batch, da)
    b = oracle.splitmix(p, seed + 1, db if shared else batch * db)
    b = b if shared else b.reshape(batch, db)
    a[0, 0], a[-1, -1] = p - 1, p - 1     # the largest residue at the rows' ends
    return a, b


def check_rows(call, got, with_oracle):
    for r in range(call.batch):
        brow = call.b if call.shared else call.b[r]
        exp = single(call.p, call.g, call.a[r], brow)
        assert np.array_equal(got[r], exp), (r, int(np.argmax(got[r] != exp)))
        if with_oracle and r < 3:
            assert np.array_equal(got[r], oracle.poly_mul(call.p, call.a[r], brow)), r


def launch_names(c, fn):
    c.sync()
    c.prof_fetch()
    c.prof_enable(True)
    try:
        fn()
        names = [n for n, _ in c.prof_fetch()]
    finally:
        c.prof_enable(False)
    return [n for n in names if n not in TABLE_BUILDS]


# (da, db, batch): L = 1, powers of two and one past them at small N and around the fused cap (2^11), da = 1, db = 1,
# da ≪ db, da ≫ db, one more row than a tile holds, more tiles than co-resident CTAs
SHAPES = [(1, 1, 1), (1, 1, 2), (1, 9, 3), (9, 1, 3), (2, 3, 5), (5, 5, 2), (8, 9, 33), (17, 16, 65), (30, 33, 16001),
          (100, 157, 9), (512, 513, 3), (1024, 1025, 2), (1024, 1026, 2), (7, 2000, 3), (2000, 7, 3), (1500, 1500, 2)]


@pytest.mark.parametrize("shared", [0, 1])
@pytest.mark.parametrize("da,db,batch", SHAPES)
@pytest.mark.parametrize("field", list(PRIMES))
def test_rows_are_the_single_product_words(field, da, db, batch, shared):
    p, g = PRIMES[field]
    if batch > 1000 and field not in ("gl", "babybear", "f101"):
        pytest.skip("the many-tile shape runs on one prime per field policy")
    a, b = operands(p, da, db, batch, shared, seed=da * 7 + db)
    call = Call(p, g, a, b, shared, offsets=((da + db) % 3, db % 5, da % 7)).run()
    got = call.result()
    if batch > 1000:     # the many-tile shape: every row against the oracle would take minutes; a sample of rows
        for r in (0, 1, 31, 32, 33, batch // 2, batch - 2, batch - 1):
            brow = b if shared else b[r]
            assert np.array_equal(got[r], oracle.poly_mul(p, a[r], brow)), r
        return
    check_rows(call, got, with_oracle=da * db <= 1 << 16)


FORCED = {1: "school", 2: "transforms", 3: "long"}


def expected(path, p, da, db, shared, names):
    L = da + db - 1
    n = 1 << max(1, (L - 1).bit_length())
    pow2 = (p - 1) % n == 0
    if path == 1:
        return names == ["poly_mul_schoolbook"]
    core = [x for x in names if x not in ("crt_reduce", "crt_combine")]
    if not pow2:     # multi-modular: one crt_combine last, the rows path over each auxiliary prime before it
        if names[-1] != "crt_combine" or names.count("crt_combine") != 1:
            return False
    fused = n <= 1 << 11 and path == 2
    if fused:
        return core == ["poly_mul_fused"] * (1 if pow2 else len(core))
    pads = ["poly_rows_pad"] if shared else ["poly_rows_pad", "poly_rows_pad"]
    k = core.count("poly_rows_clip")
    return k >= 1 and core[:len(pads)] == pads and core[-1] == "poly_rows_clip" and "poly_mul_fused" not in core


@pytest.mark.parametrize("shared", [0, 1])
@pytest.mark.parametrize("path", list(FORCED))
@pytest.mark.parametrize("field,da,db,batch", [("gl", 3, 4, 5), ("gl", 300, 301, 7), ("gl", 2048, 1, 3),
                                                ("babybear", 700, 900, 4), ("pbig", 5000, 3000, 2),
                                                ("f101", 40, 60, 9), ("f101", 1500, 1000, 3), ("p2adic3", 100, 90, 5),
                                                ("gl_g5", 129, 128, 6)])
def test_every_path_runs_its_kernels(field, da, db, batch, path, shared):
    """Each path forced on its own context (RONK_POLY_BATCH_PATH): its launches are those the path rule names, and the
    words are those of the single product.  The fused kernel is one launch for the whole batch."""
    p, g = PRIMES[field]
    a, b = operands(p, da, db, batch, shared, seed=11 + da)
    call = Call(p, g, a, b, shared, offsets=(1, 2, 3))
    c = context(path)
    names = launch_names(c, lambda: call.run(c))
    assert expected(path, p, da, db, shared, names), (FORCED[path], names)
    check_rows(call, call.result(), with_oracle=False)


def test_config1_shape_at_a_large_batch():
    """BASELINE config 1, 9 × 9 over F101, for 2^16 rows at once (shared and not), against numpy."""
    p, batch = 101, 1 << 16
    for shared in (0, 1):
        a, b = operands(p, 9, 9, batch, shared, seed=101)
        got = Call(p, 2, a, b, shared).run().result()
        B = np.broadcast_to(b, (batch, 9)) if shared else b
        exp = np.zeros((batch, 17), dtype=np.int64)
        for i in range(9):
            exp[:, i:i + 9] += a[:, i:i + 1].astype(np.int64) * B.astype(np.int64)
        assert np.array_equal(got, (exp % p).astype(np.uint64)), shared


@pytest.mark.parametrize("shared", [0, 1])
def test_long_goldilocks_rows_on_the_tile_kernels(shared):
    """4 × (2^20 × 2^20) over Goldilocks: N = 2^21 on the 256-point-tile kernels, batched."""
    p, g, n = GL, 7, 1 << 20
    a, b = operands(p, n, n, 4, shared, seed=5)
    call = Call(p, g, a, b, shared)
    names = launch_names(ctx(), call.run)
    assert "ntt3_pass1" in names and names[-1] == "poly_rows_clip", names
    got = call.result()
    for r in range(4):
        assert np.array_equal(got[r], single(p, g, a[r], b if shared else b[r])), r


@pytest.mark.parametrize("field,da,db", [("f101", 300, 400), ("m31", 700, 600), ("p64", 1100, 1200)])
def test_one_shape_per_prime_count(field, da, db):
    """k = 1, 2, 3 auxiliary primes (101, 2^31 - 1, 2^64 - 279) on the multi-modular rows, forced and by default."""
    p = {"f101": 101, "m31": (1 << 31) - 1, "p64": (1 << 64) - 279}[field]
    g = oracle.generator(p) if p < 1 << 32 else 5
    for path in (0, 2):
        for shared in (0, 1):
            a, b = operands(p, da, db, 3, shared, seed=da)
            call = Call(p, g, a, b, shared)
            c = context(path)
            names = launch_names(c, lambda: call.run(c))
            if path:
                assert names[-1] == "crt_combine", names
            check_rows(call, call.result(), with_oracle=False)


def test_refused_calls_write_nothing():
    from ronkathon_b200 import _lib
    from ronkathon_b200._lib import EINVAL, EUNSUPPORTED, RonkError
    c = ctx()
    a, b = operands(GL, 4, 5, 3, 0, seed=1)
    call = Call(GL, 7, a, b, 0)
    P = _lib._ptr

    def rc(*args):
        return _lib.lib().ronk_poly_mul_batch_u64(c._h, *args)

    av, bv, cv = P(call.av), P(call.bv), P(call.cv)
    cases = [
        (EINVAL, (GL, 7, None, 4, bv, 5, 0, 3, cv)), (EINVAL, (GL, 7, av, 4, None, 5, 0, 3, cv)),
        (EINVAL, (GL, 7, av, 4, bv, 5, 0, 3, None)), (EINVAL, (GL, 7, av, 0, bv, 5, 0, 3, cv)),
        (EINVAL, (GL, 7, av, 4, bv, 0, 0, 3, cv)), (EINVAL, (GL, GL, av, 4, bv, 5, 0, 3, cv)),
        (EINVAL, (100, 3, av, 4, bv, 5, 0, 3, cv)), (EINVAL, (GL - 1, 7, av, 4, bv, 5, 0, 3, cv)),
        (EUNSUPPORTED, (GL, 7, av, (1 << 32) + 1, bv, 5, 0, 1, cv)),
        (EUNSUPPORTED, (GL, 7, av, 1 << 20, bv, 1 << 20, 0, 1 << 20, cv)),
        (EUNSUPPORTED, (GL, 7, av, 3000, bv, 3000, 1, 1 << 20, cv)),    # batch·N = 2^33 on the batched transforms
    ]
    for code, args in cases:
        assert rc(*args) == code, args
        assert call.unwritten(), args
    # c overlapping a or b: views into one buffer
    import torch
    buf = torch.zeros(1000, dtype=torch.int64, device="cuda")
    for ao, bo, co in ((0, 100, 5), (0, 100, 90), (0, 100, 110), (0, 100, 0), (200, 0, 10)):
        assert rc(GL, 7, P(buf[ao:]), 4, P(buf[bo:]), 5, 0, 3, P(buf[co:])) == EINVAL, (ao, bo, co)
    assert rc(GL, 7, av, 4, bv, 5, 0, 0, cv) == 0 and call.unwritten()     # batch 0 does nothing
    with pytest.raises(RonkError):
        c.call("ronk_poly_mul_batch_u64", GL, 7, av, 4, bv, 5, 0, 3, P(call.av))


@pytest.mark.parametrize("field,da,db,batch,shared", [("gl", 5, 6, 7, 0), ("gl", 300, 200, 5, 1), ("f101", 50, 70, 4, 0),
                                                      ("babybear", 3000, 2000, 2, 0), ("f17", 3, 3, 9, 1)])
def test_host_variant_gives_the_device_words(field, da, db, batch, shared):
    from ronkathon_b200 import _lib
    p, g = PRIMES[field]
    a, b = operands(p, da, db, batch, shared, seed=3)
    want = Call(p, g, a, b, shared).run().result()
    out = np.zeros((batch, da + db - 1), dtype=np.uint64)
    ctx().call("ronk_poly_mul_batch_u64_host", p, g, _lib._ptr(np.ascontiguousarray(a)), da,
               _lib._ptr(np.ascontiguousarray(b)), db, shared, batch, _lib._ptr(out))
    assert np.array_equal(out, want)


def test_ops_wrapper():
    from ronkathon_b200 import ops
    a, b = operands(GL, 10, 20, 6, 0, seed=9)
    got = host(ops.poly_mul_batch(ctx(), dev(a), dev(b))).reshape(6, 29)
    shared = host(ops.poly_mul_batch(ctx(), dev(a), dev(b[2]))).reshape(6, 29)
    for r in range(6):
        assert np.array_equal(got[r], oracle.poly_mul(GL, a[r], b[r]))
        assert np.array_equal(shared[r], oracle.poly_mul(GL, a[r], b[2]))
