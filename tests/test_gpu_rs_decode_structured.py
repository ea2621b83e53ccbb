"""ronk_rs_decode_u64 on the structured rows of tests/rs_corpus.py: few errors under a large parity budget, errors on
cosets of subgroups, bursts, prescribed syndrome sequences and a row for every check that refuses one, with n - k on
both sides of every block size of the locator kernel (32, 64, 128, 512 and 1024 threads, 8 coefficients each) and n on
every transform path.  What each row must give is known by construction; at n ≤ 512 the Python model of
tests/test_rs_decode_model.py is compared word for word as well.  Every call runs on sentinel-filled outputs between
guard words and must leave its inputs as they were."""
import numpy as np
import pytest

import rs_corpus as rc
from gpu_util import ctx, dev
from test_gpu_rs_decode import PRIMES, check_bounded, encode
from test_rs_locator_model import decode as model_decode

pytestmark = pytest.mark.gpu

GUARD = 4
SENTINEL = 0x5A5A5A5A5A5A5A5A
FIELDS = ("goldilocks", "babybear", "pbig", "gl_g5")
ODD = {"goldilocks": 3, "babybear": 3, "pbig": 11, "gl_g5": 3}          # an odd factor of p - 1, for Bluestein's path
LITERAL = {"goldilocks": 255, "babybear": 320, "pbig": 11 << 4, "gl_g5": 257}   # gl_g5: g = 7^5 has order (p - 1)/5
PARITIES = (33, 255, 256, 257, 1023, 1024, 4095, 8191)


def _cells():
    out = []
    for name in FIELDS:
        blue = ODD[name] << (12 if ODD[name] == 3 else 10)
        for m in PARITIES:
            if m < 4096:
                out.append((name, 1 << 12, m))               # m = 4095: k = 1
            elif name in ("goldilocks", "pbig"):
                out.append((name, 1 << 16, m))
            if m < 4095 or name == "goldilocks":
                out.append((name, blue, m))
            if m < LITERAL[name]:
                out.append((name, LITERAL[name], m))
        out.append((name, 256, 255))                          # k = 1 at a size the model runs
    return out


CELLS = _cells()


def forward_on_device(c, code):
    """The forward transform of each row of Y: the encoder with k = n."""
    return lambda Y: encode(c, code.p, code.g, Y, code.n)


def guarded_decode(c, code, rows, erased, host=False):
    """One decode call on sentinel-filled outputs between guard words, on the device or through the host-pointer entry
    point: (messages, statuses) after checking the guards, the inputs, and that refused rows are all zero."""
    import torch
    from ronkathon_b200 import _lib
    b, n, k = rows.shape[0], code.n, code.k
    flat_rows, flat_er = np.ascontiguousarray(rows.ravel()), np.ascontiguousarray(erased.ravel())
    if host:
        msg = np.full(b * k + 2 * GUARD, SENTINEL, dtype=np.uint64)
        st = np.full(b + 2 * GUARD, 0x5A5A5A5A, dtype=np.int32)
        d_rows, d_er = flat_rows.copy(), flat_er.copy()
        entry = "ronk_rs_decode_u64_host"
    else:
        msg = dev(np.full(b * k + 2 * GUARD, SENTINEL, dtype=np.uint64))
        st = torch.full((b + 2 * GUARD,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
        d_rows, d_er = dev(flat_rows), torch.from_numpy(flat_er).cuda()
        entry = "ronk_rs_decode_u64"
    c.call(entry, code.p, code.g, _lib._ptr(d_rows), _lib._ptr(d_er), n, k, b, _lib._ptr(msg[GUARD:]), _lib._ptr(st[GUARD:]))
    c.sync()
    if not host:
        d_rows, d_er = d_rows.cpu().numpy().view(np.uint64), d_er.cpu().numpy()
        msg, st = msg.cpu().numpy().view(np.uint64), st.cpu().numpy()
    assert np.array_equal(d_rows, flat_rows) and np.array_equal(d_er, flat_er), "the call changed its inputs"
    for buf, fill in ((msg, SENTINEL), (st, 0x5A5A5A5A)):
        assert (buf[:GUARD] == fill).all() and (buf[-GUARD:] == fill).all(), "a guard word was written"
    msg, st = msg[GUARD:-GUARD].reshape(b, k), st[GUARD:-GUARD]
    assert ((st >= -1) & (st <= code.m)).all()
    assert not msg[st == -1].any(), "a refused row's message is not zero"
    return msg, st


def check_expectations(specs, expect, msg, st):
    for r, (spec, want) in enumerate(zip(specs, expect)):
        if want.status is not None:
            assert st[r] == want.status, (r, spec.name, int(st[r]), want.status)
        if want.msg is not None:
            assert np.array_equal(msg[r], want.msg), (r, spec.name)


@pytest.mark.parametrize("name,n,m", CELLS, ids=[f"{a}-n{b}-m{c}" for a, b, c in CELLS])
def test_structured_rows(name, n, m):
    """Every corpus row gives what it was built to give: the genuine patterns their message and error count, the rows
    built to be refused -1 and zeros, the rest a message within the radius; all of them keep the bounded-distance
    promise on re-encoding.  At n ≤ 512 the constructed rows and every fourth genuine one equal the Python model."""
    p, g = PRIMES[name]
    assert (p - 1) % n == 0
    c = ctx()
    code = rc.Code(p, g, n, n - m)
    specs = rc.everything(code, np.random.default_rng([n, m, len(name)]))
    rows, erased, k, expect = rc.build(code, specs, forward_on_device(c, code))
    msg, st = guarded_decode(c, code, rows, erased)
    check_expectations(specs, expect, msg, st)
    check_bounded(c, p, g, rows, erased, k, msg, st)
    kinds = {s.name.split("-")[0] for s in specs}
    assert {"random", "ends", "burst", "tozero", "delta", "recur_genuine", "recur_double", "erasures"} <= kinds
    assert "coset_equal" in kinds or all(n % e for e in range(2, m // 2 + 1))      # n = 257 has no subgroup to offer
    assert (st == -1).sum() >= 8 and (st > 0).sum() >= 40
    if n <= 512:
        genuine = 0
        for r, spec in enumerate(specs):
            if expect[r].msg is not None:
                genuine += 1
                if genuine % 4:
                    continue
            want, want_st = model_decode(p, g, [int(v) for v in rows[r]], list(erased[r]), k)
            assert st[r] == want_st, (r, spec.name)
            assert msg[r].tolist() == (want if want is not None else [0] * k), (r, spec.name)


MIXED = [("goldilocks", 1 << 12, 1025), ("goldilocks", 3 << 12, 2500), ("babybear", 1 << 12, 1500)]


@pytest.mark.parametrize("name,n,m", MIXED, ids=[f"{a}-n{b}-m{c}" for a, b, c in MIXED])
def test_mixed_batch_equals_separate_calls_and_the_host_entry_point(name, n, m):
    """At least 300 rows, m > 1024 (the locator's block is full), refused rows between decoding ones, every erasure
    flag byte: each row of the batch equals its own one-row call, and the host-pointer call equals the device call."""
    p, g = PRIMES[name]
    c = ctx()
    code = rc.Code(p, g, n, n - m)
    specs = rc.mixed(code, np.random.default_rng([n, m]), rows=300)
    rows, erased, k, expect = rc.build(code, specs, forward_on_device(c, code))
    assert len(specs) >= 300 and set(rc.FLAGS) <= set(np.unique(erased))
    msg, st = guarded_decode(c, code, rows, erased)
    check_expectations(specs, expect, msg, st)
    refused = st == -1
    assert refused.sum() >= 20 and (refused[1:] != refused[:-1]).sum() >= 40, "refused and decoding rows are not interleaved"
    for r in range(len(specs)):
        m1, s1 = guarded_decode(c, code, rows[r:r + 1], erased[r:r + 1])
        assert s1[0] == st[r] and np.array_equal(m1[0], msg[r]), (r, specs[r].name)
    hm, hs = guarded_decode(c, code, rows, erased, host=True)
    assert np.array_equal(hm, msg) and np.array_equal(hs, st)
    check_bounded(c, p, g, rows, erased, k, msg, st)
