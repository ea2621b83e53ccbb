"""ronk_rs_encode_u64 and ronk_rs_decode_u64[_host]: Reed–Solomon encoding and errors-and-erasures decoding.

Messages are compared exactly; a row beyond the radius must give -1 with a zero message, or a message whose codeword
(re-encoded) differs from the row in `status` non-erased positions with 2·status + ε ≤ n - k.  Reference values come
from tests/golden/reference_kats.json, the oracle's encoder and ronk_poly_interpolate_u64_host (Message::decode)."""
import itertools
import os

import numpy as np
import pytest

import oracle
from gpu_util import GL, MONT_PRIMES, ctx, dev, host

pytestmark = pytest.mark.gpu

EINVAL, EUNSUPPORTED = 1, 5
CAP = 8191   # RONK_RS_MAX_PARITY
PRIMES = {**{k: (p, g) for k, (p, g, _) in MONT_PRIMES.items()}, "goldilocks": (GL, 7)}
SENTINEL = -1


def _cap_from_header():
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    return int(re.search(r"#define RONK_RS_MAX_PARITY (\d+)", open(os.path.join(root, "include", "ronk_b200.h")).read()).group(1))


def encode(c, p, g, msgs, n):
    """msgs: batch × k host array → batch × n host codewords"""
    from ronkathon_b200 import ops
    msgs = np.atleast_2d(np.asarray(msgs, dtype=np.uint64))
    out = ops.rs_encode(c, dev(msgs.ravel()), n, msgs.shape[0], p=p, g=g)
    return host(out).reshape(msgs.shape[0], n)


def decode(c, p, g, rows, k, erased=None):
    """rows: batch × n host array → (batch × k messages, statuses)"""
    import torch
    from ronkathon_b200 import ops
    rows = np.atleast_2d(np.asarray(rows, dtype=np.uint64))
    er = None if erased is None else torch.from_numpy(np.ascontiguousarray(erased, dtype=np.uint8).ravel()).cuda()
    msg, st = ops.rs_decode(c, dev(rows.ravel()), k, er, rows.shape[0], p=p, g=g)
    return host(msg).reshape(rows.shape[0], k), st.cpu().numpy()


def check_bounded(c, p, g, rows, erased, k, msgs, st):
    """Every row: -1 with a zero message, or a message within the radius at exactly `status` non-erased differences."""
    b, n = rows.shape
    er = np.zeros((b, n), bool) if erased is None else np.asarray(erased, bool)
    cw = encode(c, p, g, msgs, n)
    dist = ((cw != rows) & ~er).sum(1)
    eps = er.sum(1)
    for r in range(b):
        if st[r] == -1:
            assert not msgs[r].any(), r
        else:
            assert st[r] >= 0 and dist[r] == st[r] and 2 * st[r] + eps[r] <= n - k, (r, st[r], dist[r], eps[r])


def corrupt(p, row, positions, rng, values=None):
    row = row.copy()
    for j, i in enumerate(positions):
        v = int(values[j]) if values is not None else int(rng.integers(1, min(p - 1, 1 << 62))) if p > 3 else 1
        row[i] = (int(row[i]) + v) % p
    return row


# ---- reference KATs ----------------------------------------------------------------------------------------------------
def test_reference_kats(kats):
    c = ctx()
    r = kats["reed_solomon"]
    assert encode(c, r["p"], 3, [r["msg"]], r["n"])[0].tolist() == r["y"]
    d = kats["reed_solomon_decode"]
    p, n = d["p"], d["n"]
    for msg in d["messages"]:
        k = len(msg)
        cw = encode(c, p, 3, [msg], n)
        got, st = decode(c, p, 3, cw, k)
        assert got[0].tolist() == msg and st[0] == 0


def test_every_pattern_of_two_errors_and_three(kats):
    """The K = 3, N = 7 codeword of reed_solomon.rs:177-219 (radius 2): every pattern of ≤ 2 errors (every position set,
    every value pair) in one batched call decodes exactly; every pattern of 3 errors gives -1 or a message within the
    radius, one call per position set."""
    import torch
    from ronkathon_b200 import ops
    c = ctx()
    p, n, g = 127, 7, 3
    msg = kats["reed_solomon_decode"]["messages"][0]
    cw = encode(c, p, g, [msg], n)[0].astype(np.int64)
    rows, want = [cw[None, :]], [0]
    for e in (1, 2):
        vals = np.array(list(itertools.product(range(1, p), repeat=e)), dtype=np.int64)
        for pos in itertools.combinations(range(n), e):
            blk = np.tile(cw, (len(vals), 1))
            blk[:, list(pos)] = (blk[:, list(pos)] + vals) % p
            rows.append(blk)
            want += [e] * len(vals)
    rows = np.concatenate(rows).astype(np.uint64)
    got, st = decode(c, p, g, rows, 3)
    assert (got == np.array(msg, dtype=np.uint64)).all() and (st == np.array(want)).all()
    vals = torch.tensor(list(itertools.product(range(1, p), repeat=3)), dtype=torch.int64, device="cuda")
    base = torch.from_numpy(cw).cuda()
    for pos in itertools.combinations(range(n), 3):
        blk = base.repeat(len(vals), 1)
        blk[:, list(pos)] = (blk[:, list(pos)] + vals) % p
        b = blk.shape[0]
        m_d, st_d = ops.rs_decode(c, blk.reshape(-1).contiguous(), 3, None, b, p=p, g=g)
        re = ops.rs_encode(c, m_d, n, b, p=p, g=g).view(b, n)
        dist = (re != blk).sum(1)
        st_l = st_d.long()
        ok = ((st_l == -1) & (m_d.view(b, 3) == 0).all(1)) | ((st_l >= 0) & (dist == st_l) & (2 * st_l <= n - 3))
        assert bool(ok.all()), pos
        assert bool((st_l != 3).all())


# ---- equivalence with Message::decode -----------------------------------------------------------------------------------
def _domain(p, g, n):
    w = pow(g, (p - 1) // n, p)
    return np.array([pow(w, i, p) for i in range(n)], dtype=np.uint64)


EQUIV = {"goldilocks": [64, 255, 3 << 12], "babybear": [64, 320], "koalabear": [64], "p32": [64, 21 << 4], "p57": [64],
         "pbig": [64], "gl_g5": [64], "p2adic3": [8]}


@pytest.mark.parametrize("name", list(EQUIV))
def test_tail_erased_equals_message_decode(name):
    """Arbitrary rows (not codewords) with positions k..n-1 erased: word for word the interpolant through the first k
    coordinates (ronk_poly_interpolate_u64_host), status 0."""
    p, g = PRIMES[name]
    c = ctx()
    for n in EQUIV[name]:
        # n - k ≤ RONK_RS_MAX_PARITY; the host interpolation takes k ≤ 8192
        for k in sorted({max(1, n - CAP), max(1, n // 3, n - CAP), min(n - 1, 8192)}):
            rows = oracle.splitmix(p, 100 + n + k, 3 * n).reshape(3, n)
            erased = np.zeros((3, n), np.uint8)
            erased[:, k:] = 1
            got, st = decode(c, p, g, rows, k, erased)
            xs = _domain(p, g, n)[:k].copy()
            for r in range(3):
                want = np.empty(k, dtype=np.uint64)
                ys = np.ascontiguousarray(rows[r, :k])
                c.call("ronk_poly_interpolate_u64_host", p, xs.ctypes.data, ys.ctypes.data, k, want.ctypes.data)
                assert np.array_equal(got[r], want), (name, n, k, r)
            assert (st == 0).all()


# ---- exact correction at the radius, on every transform path ------------------------------------------------------------
RADIUS = [("goldilocks", 256, 224), ("babybear", 1024, 900), ("koalabear", 512, 400), ("p32", 256, 200), ("p57", 128, 64),
          ("pbig", 256, 128), ("gl_g5", 64, 32), ("p2adic3", 8, 3),                                       # powers of two
          ("goldilocks", 3 << 12, (3 << 12) - 300), ("goldilocks", 65537 << 4, (65537 << 4) - 64),
          ("babybear", 15 << 10, (15 << 10) - 1000), ("p32", 21 << 10, (21 << 10) - 500),            # Bluestein
          ("goldilocks", 255, 200), ("babybear", 320, 250), ("koalabear", 127, 60), ("p57", 29, 10),
          ("pbig", 11 << 4, 100)]                                                                        # literal


@pytest.mark.parametrize("name,n,k", RADIUS, ids=[f"{a}-{b}-{c}" for a, b, c in RADIUS])
def test_exact_correction_at_the_radius(name, n, k):
    """Row 0: ⌊m/2⌋ errors of value p - 1, at positions 0 and n - 1 among them.  Row 1: ε random erasures and
    ⌊(m - ε)/2⌋ errors.  Row 2: ε = m erasures.  Row 3: the codeword.  Rows 4, 5: one error past the radius, without and
    with erasures, keep the bounded-distance promise."""
    p, g = PRIMES[name]
    assert (p - 1) % n == 0
    c = ctx()
    m = n - k
    rng = np.random.default_rng(n + k)
    msgs = oracle.splitmix(p, 200 + n, 6 * k).reshape(6, k)
    cw = encode(c, p, g, msgs, n)
    if n <= 4096:
        for r in range(2):
            assert np.array_equal(cw[r], oracle.rs_encode(p, msgs[r], n, g)[1])
    rows = cw.copy()
    erased = np.zeros((6, n), np.uint8)
    e0 = m // 2
    pos0 = ([0, n - 1] + [int(v) for v in rng.choice(np.arange(1, n - 1), max(e0 - 2, 0), replace=False)])[:e0]
    rows[0] = corrupt(p, cw[0], pos0, rng, values=[p - 1] * e0)
    eps = m // 3
    perm = rng.permutation(n)
    erased[1, perm[:eps]] = 1
    e1 = (m - eps) // 2
    rows[1] = corrupt(p, cw[1], perm[eps:eps + e1], rng)
    rows[1, perm[:eps]] = rng.integers(0, min(p, 1 << 62), eps).astype(np.uint64)
    erased[2, rng.permutation(n)[:m]] = 1
    rows[2] = np.where(erased[2] == 1, np.uint64(0), cw[2])
    rows[4] = corrupt(p, cw[4], rng.permutation(n)[:min(e0 + 1, n)], rng)
    erased[5, perm[:eps]] = 1
    rows[5] = corrupt(p, cw[5], perm[eps:eps + min(e1 + 1, n - eps)], rng)
    got, st = decode(c, p, g, rows, k, erased)
    for r, e in ((0, e0), (1, e1), (2, 0), (3, 0)):
        assert np.array_equal(got[r], msgs[r]) and st[r] == e, (r, st[r], e)
    check_bounded(c, p, g, rows[4:], erased[4:], k, got[4:], st[4:])


# ---- envelope ----------------------------------------------------------------------------------------------------------
def _radius_row(c, p, g, n, k, seed, eps=0):
    rng = np.random.default_rng(seed)
    msg = oracle.splitmix(p, seed, k)
    cw = encode(c, p, g, [msg], n)[0]
    perm = rng.permutation(n)
    erased = np.zeros(n, np.uint8)
    erased[perm[:eps]] = 1
    e = (n - k - eps) // 2
    row = corrupt(p, cw, perm[eps:eps + e], rng)
    return msg, row, erased, e


@pytest.mark.parametrize("n", [1 << 16, 1 << 20, 3 << 20])
def test_the_cap(n):
    """n - k = RONK_RS_MAX_PARITY with a full radius of errors decodes (Goldilocks 2^16, 2^20 and Bluestein's 3·2^20);
    one more parity symbol is refused with the outputs untouched."""
    assert _cap_from_header() == CAP
    c = ctx()
    k = n - CAP
    msg, row, erased, e = _radius_row(c, GL, 7, n, k, 7 + n)
    assert e == CAP // 2
    got, st = decode(c, GL, 7, row[None, :], k)
    assert np.array_equal(got[0], msg) and st[0] == e
    if n == 1 << 16:
        expect_refused(c, GL, 7, n, n - CAP - 1, EUNSUPPORTED)


def test_erasures_up_to_m_and_edges():
    c = ctx()
    p, g, n, k = GL, 7, 256, 200
    msg, row, erased, e = _radius_row(c, p, g, n, k, 11, eps=n - k)
    assert e == 0
    got, st = decode(c, p, g, row[None, :], k, erased[None, :])
    assert np.array_equal(got[0], msg) and st[0] == 0
    erased[np.flatnonzero(erased == 0)[0]] = 1                     # ε = m + 1
    got, st = decode(c, p, g, row[None, :], k, erased[None, :])
    assert st[0] == -1 and not got.any()
    rows = oracle.splitmix(p, 12, 3 * n).reshape(3, n)             # k = n: every word is a codeword
    got, st = decode(c, p, g, rows, n)
    w = pow(7, (p - 1) // n, p)
    for r in range(3):
        assert oracle.poly_eval(p, got[r], w) == int(rows[r, 1])
    assert (st == 0).all() and np.array_equal(encode(c, p, g, got, n), rows)
    for name in ("goldilocks", "babybear", "p2adic3"):               # n = 1
        p, g = PRIMES[name]
        rows = oracle.splitmix(p, 13, 4).reshape(4, 1)
        got, st = decode(c, p, g, rows, 1)
        assert np.array_equal(got, rows) and (st == 0).all()
        assert np.array_equal(encode(c, p, g, rows, 1), rows)


# ---- batch and variants ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,n,k", [("goldilocks", 256, 200), ("goldilocks", 3 << 12, (3 << 12) - 100),
                                      ("goldilocks", 255, 180), ("babybear", 320, 250)])
def test_batch_equals_separate_calls_and_host_equals_device(name, n, k):
    p, g = PRIMES[name]
    c = ctx()
    rng = np.random.default_rng(n)
    msgs = oracle.splitmix(p, 300 + n, 5 * k).reshape(5, k)
    rows = encode(c, p, g, msgs, n)
    erased = np.zeros((5, n), np.uint8)
    for r in range(5):
        eps = int(rng.integers(0, n - k + 1))
        erased[r, rng.permutation(n)[:eps]] = 1
        rows[r] = corrupt(p, rows[r], rng.permutation(n)[:(n - k - eps) // 2 + (r == 4)], rng)
    got, st = decode(c, p, g, rows, k, erased)
    for r in range(5):
        g1, s1 = decode(c, p, g, rows[r:r + 1], k, erased[r:r + 1])
        assert np.array_equal(g1[0], got[r]) and s1[0] == st[r], r
    hm = np.full(5 * k, 0xFFFFFFFFFFFFFFFF, dtype=np.uint64)
    hs = np.full(5, 7, dtype=np.int32)
    hr = np.ascontiguousarray(rows.ravel())
    he = np.ascontiguousarray(erased.ravel())
    c.call("ronk_rs_decode_u64_host", p, g, hr.ctypes.data, he.ctypes.data, n, k, 5, hm.ctypes.data, hs.ctypes.data)
    assert np.array_equal(hm.reshape(5, k), got) and np.array_equal(hs, st)
    check_bounded(c, p, g, rows, erased, k, got, st)


def test_encode_equals_codes_rs_encode_and_rs_correct():
    from ronkathon_b200 import GoldilocksField, PrimeField, codes
    c = ctx()
    for F, n, k in ((PrimeField(127), 7, 3), (PrimeField(127), 63, 20), (GoldilocksField, 256, 100),
                    (GoldilocksField, 255, 100)):
        p = F.ORDER
        g = F.PRIMITIVE_ELEMENT.value
        msg = [int(v) for v in oracle.splitmix(p, n, k)]
        cw = codes.rs_encode(msg, n, F)
        assert [y.value for _, y in cw] == encode(c, p, g, [msg], n)[0].tolist()
        bad = list(cw)
        errs = (n - k - 2) // 2
        for i in range(errs):
            bad[2 + i] = (cw[2 + i][0], cw[2 + i][1] + F(1 + i))
        bad[0] = (cw[0][0], F(0))
        bad[1] = (cw[1][0], F(5))
        got, e = codes.rs_correct(bad, k, F, erasures=(0, 1))
        assert [v.value for v in got] == msg and e == errs
        bad[2 + errs] = (cw[2 + errs][0], cw[2 + errs][1] + F(1))
        got, e = codes.rs_correct(bad, k, F, erasures=(0, 1))
        assert got is None and e == -1 or 2 * e + 2 <= n - k
    with pytest.raises(AssertionError):
        codes.rs_correct(list(reversed(codes.rs_encode([1, 2, 3], 7, PrimeField(127)))), 3, PrimeField(127))


def record(c, fn):
    """Warm fn once, then the profile names of one profiled call and the launches of one unprofiled call."""
    fn()
    c.sync()
    c.prof_fetch()
    c.prof_enable(True)
    try:
        fn()
        names = [nm for nm, _ in c.prof_fetch()]
    finally:
        c.prof_enable(False)
    before = c.launches
    fn()
    c.sync()
    return names, c.launches - before


def _any_names(c, n, batch, inverse):
    from ronkathon_b200 import ops
    x = dev(oracle.splitmix(GL, 400, batch * n))
    return record(c, lambda: ops.ntt_any_(c, x, n, batch, inverse=inverse))[0]


PINNED = {
    # case → (n, k, profile names of a warm batch-1 decode; None: composed from ronk_ntt_any_u64's records)
    "pow2_256": (256, 200, ["intt_single", "rs_locator", "ntt_single", "rs_correct", "intt_single", "rs_finish"]),
    "literal_255": (255, 200, ["pow_table", "rs_dft", "rs_locator", "rs_dft", "rs_correct", "rs_dft", "rs_finish"]),
    "bluestein_3x2^12": (3 << 12, (3 << 12) - 64, None),
}


@pytest.mark.parametrize("case", list(PINNED))
def test_launches_do_not_depend_on_the_batch(case):
    """Batch 1 and batch 4096 launch the same number of kernels.  The record of batch 1 is the pinned one; on the
    transform paths each record is the transforms' own (ronk_ntt_any_u64 of the same rows) around the decoder's three
    kernels."""
    import torch
    from ronkathon_b200 import ops
    n, k, pinned = PINNED[case]
    c = ctx()
    seen = []
    for batch in (1, 4096):
        x = ops.rs_encode(c, dev(oracle.splitmix(GL, 401, batch * k)), n, batch)
        er = torch.zeros(batch * n, dtype=torch.uint8, device="cuda")
        names, launches = record(c, lambda: ops.rs_decode(c, x, k, er, batch))
        if case.startswith("literal"):
            want = pinned
        else:
            want = (_any_names(c, n, batch, True) + ["rs_locator"] + _any_names(c, n, 3 * batch, False) + ["rs_correct"]
                    + _any_names(c, n, batch, True) + ["rs_finish"])
        assert names == want, (batch, names)
        if batch == 1 and pinned is not None:
            assert names == pinned
        if case.startswith("bluestein"):
            assert names[0] == "anyntt_chirp_in" and names.count("anyntt_chirp_out") == 3
        seen.append(launches)
        _, st = ops.rs_decode(c, x, k, er, batch)
        assert bool((st == 0).all())
    assert seen[0] == seen[1] == len(want)
    names, _ = record(c, lambda: ops.rs_encode(c, dev(oracle.splitmix(GL, 402, k)), n, 1))
    assert names[0] == ("pow_table" if case.startswith("literal") else "rs_pad")


# ---- errors and streams ------------------------------------------------------------------------------------------------
def expect_refused(c, p, g, n, k, code, batch=1, erased=True, alias=False):
    """Decode returns `code` and leaves sentinel-filled device and host outputs untouched."""
    import torch
    from ronkathon_b200 import _lib
    words = max(batch * n, 1) if batch * n <= 1 << 22 else 1 << 10
    rec = torch.zeros(words, dtype=torch.int64, device="cuda")
    er = torch.zeros(words, dtype=torch.uint8, device="cuda") if erased else None
    msg = rec if alias else torch.full((max(batch * k, 1) if batch * k <= 1 << 22 else 1 << 10,), SENTINEL,
                                       dtype=torch.int64, device="cuda")
    st = torch.full((min(max(batch, 1), 1 << 10),), SENTINEL, dtype=torch.int32, device="cuda")
    rc = _lib.lib().ronk_rs_decode_u64(c._h, p, g, _lib._ptr(rec), _lib._ptr(er), n, k, batch, _lib._ptr(msg), _lib._ptr(st))
    assert rc == code, (hex(p), g, n, k, batch, rc)
    c.sync()
    if not alias:
        assert bool((msg == SENTINEL).all())
    assert bool((st == SENTINEL).all())
    if words <= 1 << 20 and not alias:
        hr = np.zeros(words, dtype=np.uint64)
        hm = np.full(msg.numel(), 0xFFFFFFFFFFFFFFFF, dtype=np.uint64)
        hs = np.full(st.numel(), -1, dtype=np.int32)
        rc = _lib.lib().ronk_rs_decode_u64_host(c._h, p, g, _lib._ptr(hr), None, n, k, batch, _lib._ptr(hm), _lib._ptr(hs))
        assert rc == code and bool((hm == 0xFFFFFFFFFFFFFFFF).all()) and bool((hs == -1).all())


def test_errors_leave_outputs_untouched():
    import torch
    from ronkathon_b200 import _lib
    c = ctx()
    for p, g, n, k, code in ((GL, 7, 0, 1, EINVAL), (GL, 7, 8, 0, EINVAL), (GL, 7, 8, 9, EINVAL), (GL, 7, 7, 3, EINVAL),
                             (GL, 0, 8, 3, EINVAL), (GL, GL, 8, 3, EINVAL), (127, 1, 7, 3, EINVAL), (97, 3, 32, 8, EINVAL),
                             (2, 1, 1, 1, EUNSUPPORTED), (GL, 7, 65537 << 9, (65537 << 9) - 10, EUNSUPPORTED),
                             (GL, 7, 1 << 16, (1 << 16) - CAP - 1, EUNSUPPORTED)):
        expect_refused(c, p, g, n, k, code)
    expect_refused(c, GL, 7, 1 << 16, 1 << 15, EUNSUPPORTED, batch=1 << 15)    # 3·batch·n ≥ 2^31
    expect_refused(c, GL, 7, 256, 200, EINVAL, alias=True)                     # msg over received
    rec = torch.zeros(256, dtype=torch.int64, device="cuda")
    msg = torch.full((200,), SENTINEL, dtype=torch.int64, device="cuda")
    st = torch.full((1,), SENTINEL, dtype=torch.int32, device="cuda")
    L = _lib.lib()
    assert L.ronk_rs_decode_u64(c._h, GL, 7, None, None, 256, 200, 1, _lib._ptr(msg), _lib._ptr(st)) == EINVAL
    assert L.ronk_rs_decode_u64(c._h, GL, 7, _lib._ptr(rec), None, 256, 200, 1, None, _lib._ptr(st)) == EINVAL
    assert L.ronk_rs_decode_u64(c._h, GL, 7, _lib._ptr(rec), None, 256, 200, 0, _lib._ptr(msg), _lib._ptr(st)) == 0
    # encode: null, k > n, n ∤ p - 1, output over input; batch 0 does nothing
    cw = torch.full((256,), SENTINEL, dtype=torch.int64, device="cuda")
    assert L.ronk_rs_encode_u64(c._h, GL, 7, None, 200, 256, 1, _lib._ptr(cw)) == EINVAL
    assert L.ronk_rs_encode_u64(c._h, GL, 7, _lib._ptr(rec), 257, 256, 1, _lib._ptr(cw)) == EINVAL
    assert L.ronk_rs_encode_u64(c._h, GL, 7, _lib._ptr(rec), 3, 7, 1, _lib._ptr(cw)) == EINVAL
    assert L.ronk_rs_encode_u64(c._h, GL, 7, _lib._ptr(cw), 200, 256, 1, _lib._ptr(cw)) == EINVAL
    assert L.ronk_rs_encode_u64(c._h, GL, 7, _lib._ptr(rec), 200, 256, 0, _lib._ptr(cw)) == 0
    c.sync()
    assert bool((msg == SENTINEL).all()) and bool((st == SENTINEL).all()) and bool((cw == SENTINEL).all())


def test_behind_a_gated_stream():
    """A warm context on a non-blocking stream s; on s a bounded spin, the real input written over a wrong one, the
    call, a clone.  s must still be busy when the call returns, and the clone must equal the suite context's result."""
    import torch
    from ronkathon_b200 import Context, ops
    n, k, batch = 3 << 12, (3 << 12) - 200, 3
    c0 = ctx()
    msgs = oracle.splitmix(GL, 500, batch * k).reshape(batch, k)
    rows = encode(c0, GL, 7, msgs, n)
    rng = np.random.default_rng(3)
    for r in range(batch):
        rows[r] = corrupt(GL, rows[r], rng.permutation(n)[:100], rng)
    real = dev(rows.ravel())
    want, want_st = ops.rs_decode(c0, real, k, None, batch)
    c0.sync()
    assert np.array_equal(host(want).reshape(batch, k), msgs)
    s = torch.cuda.Stream()
    c = Context(0, s.cuda_stream)
    try:
        buf = real.flip(0).contiguous()
        with torch.cuda.stream(s):
            ops.rs_decode(c, buf.clone(), k, None, batch)      # warm: spectrum and plans
        s.synchronize()
        with torch.cuda.stream(s):
            torch.cuda._sleep(100_000_000)
            buf.copy_(real)
            m, st = ops.rs_decode(c, buf, k, None, batch)
            assert not s.query(), "s finished before the call returned"
            got, got_st = m.clone(), st.clone()
        s.synchronize()
        assert torch.equal(got, want) and torch.equal(got_st, want_st)
    finally:
        c.close()
