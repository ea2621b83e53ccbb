"""GPU parity: PrimeField<P> arithmetic through the C ABI vs the reference KATs and the oracle.
Reads like src/algebra/field/prime/{mod,arithmetic}.rs's own tests."""
import numpy as np
import pytest

import oracle
from gpu_util import BABYBEAR, GL, PBIG, ctx, dev, host

pytestmark = pytest.mark.gpu


def test_reference_kats_scalar_api(kats):
    from ronkathon_b200 import PrimeField, RonkPanic
    ctx()
    f = kats["field"]
    for p, a, b, r in f["add"]:
        F = PrimeField(p); assert F.new(a) + F.new(b) == F.new(r)
    for p, a, b, r in f["sub"]:
        F = PrimeField(p); assert F.new(a) - F.new(b) == F.new(r)
    for p, a, b, r in f["mul"]:
        F = PrimeField(p); assert F.new(a) * F.new(b) == F.new(r)
    for p, a, e, r in f["pow"]:
        F = PrimeField(p); assert F.new(a).pow(e) == F.new(r)
    for p, a, r in f["inverse"]:
        F = PrimeField(p); assert F.new(a).inverse() == F.new(r)
    for p in f["inverse_of_zero_panics"]:
        F = PrimeField(p)
        assert F.new(0).inverse() is None          # prime/mod.rs:63-65
        with pytest.raises(RonkPanic):             # Div unwraps the None (arithmetic.rs:54)
            F.new(1) / F.new(0)
    for p, a, r in f["halve"]:
        F = PrimeField(p); assert F.new(a).div(F.new(2)) == F.new(r)
    for p, g in f["generator"].items():
        assert PrimeField(int(p)).PRIMITIVE_ELEMENT.value == g
    for p, n in f["no_root_of_unity"]:
        with pytest.raises(RonkPanic):
            PrimeField(p).primitive_root_of_unity(n)
    with pytest.raises(RonkPanic):                 # prime/mod.rs:293-295 non-prime modulus
        PrimeField(100).new(1) + PrimeField(100).new(1)


@pytest.mark.parametrize("p", [17, 101])
def test_exhaustive_field_laws(p):
    """prime/mod.rs:346-374, arithmetic.rs:136-152 over the whole field, on the GPU."""
    from ronkathon_b200 import ops
    c = ctx()
    a = np.repeat(np.arange(p, dtype=np.uint64), p)
    b = np.tile(np.arange(p, dtype=np.uint64), p)
    da, db = dev(a), dev(b)
    for op, fn in (("add", oracle.add), ("sub", oracle.sub), ("mul", oracle.mul)):
        got = host(ops.field_binop(c, op, da, db, p))
        exp = np.array([fn(p, int(x), int(y)) for x, y in zip(a, b)], dtype=np.uint64)
        assert np.array_equal(got, exp), op
    nz = b != 0
    got = host(ops.field_binop(c, "div", dev(a[nz]), dev(b[nz]), p))
    exp = np.array([oracle.div(p, int(x), int(y)) for x, y in zip(a[nz], b[nz])], dtype=np.uint64)
    assert np.array_equal(got, exp)


def _edge(p):
    v = [0, 1, 2, p - 1, p - 2, p // 2, p // 2 + 1]
    if p > (1 << 33):
        v += [(1 << 32) - 1, 1 << 32, (1 << 32) + 1, p - (1 << 32), p - (1 << 32) + 1, 1 << 63, 0xFFFFFFFF00000000,
              0xFFFFFFFE00000002]
    return [x % p for x in v]


@pytest.mark.parametrize("p", [GL, 0xFFFFFFFFFFFFFFC5, 0x7FFFFFFFFFFFFFE7, 4179340454199820289, 127, BABYBEAR, 4295294977, PBIG])
def test_64bit_field_ops_vs_oracle(p):
    from ronkathon_b200 import ops
    c = ctx()
    ev = _edge(p)
    rng = np.random.default_rng(11)
    rnd = [int(v) % p for v in rng.integers(0, 2**63, 20000, dtype=np.uint64) * 2 + 1]
    a = np.array([x for x in ev for _ in ev] + rnd, dtype=np.uint64)
    b = np.array([y for _ in ev for y in ev] + rnd[::-1], dtype=np.uint64)
    da, db = dev(a), dev(b)
    for op, fn in (("add", oracle.add), ("sub", oracle.sub), ("mul", oracle.mul)):
        got = host(ops.field_binop(c, op, da, db, p))
        exp = np.array([fn(p, int(x), int(y)) for x, y in zip(a, b)], dtype=np.uint64)
        assert np.array_equal(got, exp), (hex(p), op)
    # inverse / pow on a sample
    import torch
    s = a[a != 0][:500]
    ds, out = dev(s), torch.empty(len(s), dtype=torch.int64, device="cuda")
    c.call("ronk_field_inv_u64", p, ds.data_ptr(), out.data_ptr(), len(s))
    assert np.array_equal(host(out), np.array([oracle.inverse(p, int(x)) for x in s], dtype=np.uint64))
    c.call("ronk_field_pow_u64", p, ds.data_ptr(), 0xDEADBEEFCAFE, out.data_ptr(), len(s))
    assert np.array_equal(host(out), np.array([oracle.pow_(p, int(x), 0xDEADBEEFCAFE) for x in s], dtype=np.uint64))
    c.call("ronk_field_neg_u64", p, ds.data_ptr(), out.data_ptr(), len(s))
    assert np.array_equal(host(out), np.array([oracle.neg(p, int(x)) for x in s], dtype=np.uint64))


def test_splitmix_matches_oracle():
    from ronkathon_b200 import ops
    c = ctx()
    for p, seed in ((GL, 42), (GL, 43), (101, 7), (17, 44)):
        assert np.array_equal(host(ops.splitmix_fill(c, 5000, seed, p)), oracle.splitmix(p, seed, 5000))


def test_empty_inputs_are_ok():
    c = ctx()
    c.call("ronk_field_add_u64", GL, None, None, None, 0)
    c.call("ronk_ntt_u64", GL, 7, dev(np.zeros(4, np.uint64)).data_ptr(), 2, 0, 0)
