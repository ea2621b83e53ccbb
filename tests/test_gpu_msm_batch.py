"""ronk_msm_pluto_ext_batch (ops.msm_batch, kzg.commit_batch): kzg::commit of many scalar rows against one SRS.

Every row must be exactly the point the single-row entry ronk_msm_pluto_ext gives for it, and the oracle's commit: on
points spread over the whole curve group with Infinity terms and zero scalars mixed in, at row lengths around the 4-byte
word and the 2048-scalar column, with rows that start at every byte offset and points that are 4- but not 16-byte aligned.
The oracle is run on every row of the smaller shapes and on the first, a middle and the last row of the larger ones."""
import numpy as np
import pytest

import oracle
from conftest import pt
from gpu_util import ctx

pytestmark = pytest.mark.gpu

EINVAL, EUNSUPPORTED = 1, 5
INF = b"\xff" * 4
POISON = 0xA5
NS = [1, 3, 4, 5, 15, 16, 17, 4095, (1 << 16) + 3, 1 << 20]
BATCHES = [1, 2, 3, 17, 256]
_base = None


def _group():
    """Points of the whole curve group, not only the 17-torsion (test_gpu_kzg's _full_group_points)."""
    global _base
    if _base is None:
        from test_gpu_kzg import _full_group_points
        _base = _full_group_points()
    return _base


def _points(n, seed, lead=0):
    """uint8 [lead + n, 4] on the device: group points with about 2 % Infinity terms."""
    import torch
    rng = np.random.default_rng(seed)
    base = _group()
    pts = base[rng.integers(0, len(base), lead + n)].copy()
    pts[rng.integers(0, lead + n, max(1, (lead + n) // 50))] = 0xFF
    return torch.from_numpy(pts).cuda()


def _scalars(batch, n, seed, lead=0):
    """A device buffer of lead + batch·n scalars < 17 (zeros included) and its (batch, n) view starting at byte lead."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    buf = torch.randint(0, 17, (lead + batch * n,), dtype=torch.uint8, device="cuda", generator=g)
    return buf, buf[lead:].view(batch, n)


def _p(x):
    from ronkathon_b200 import _lib
    return _lib._ptr(x)


def _rc(c, name, *args):
    from ronkathon_b200 import _lib
    c.sync()
    before = c.launches
    rc = getattr(_lib.lib(), name)(c._h, *args)
    c.sync()
    return rc, c.launches - before


def _single(c, P, row):
    from ronkathon_b200 import ops
    return ops.msm(c, P, row)


def _check_rows(c, P, S, rows=None):
    """ops.msm_batch(P, S) row by row against the single-row entry (every row, or `rows`) and the oracle."""
    from ronkathon_b200 import ops
    got = ops.msm_batch(c, P, S).cpu().numpy()
    batch, n = S.shape
    rows = range(batch) if rows is None else rows
    for r in rows:
        assert got[r].tobytes() == _single(c, P, S[r]), (batch, n, r)
    sample = range(batch) if batch * n <= 1 << 22 else sorted({0, batch // 2, batch - 1})
    pts = P[:n].cpu().numpy()
    for r in sample:
        if r in rows:
            assert got[r].tobytes() == oracle.commit(S[r].cpu().numpy(), pts, fast=True), (batch, n, r)
    return got


# ---- words -------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("batch", BATCHES)
def test_rows_equal_single_and_oracle(batch, n):
    """Every row; the scalar view starts 0–3 bytes into its buffer and the point view 0–3 points into its own, so that
    rows start at every byte offset and points are 4- but not 16-byte aligned."""
    c = ctx()
    i = NS.index(n) + BATCHES.index(batch)
    s_lead, p_lead = i % 4, (i // 2) % 4
    P = _points(n, 100 + n, p_lead)[p_lead:]
    _, S = _scalars(batch, n, 200 + 7 * n + batch, s_lead)
    _check_rows(c, P, S)


@pytest.mark.parametrize("s_lead", [1, 2, 3])
@pytest.mark.parametrize("p_lead", [1, 2, 3])
def test_unaligned_views(s_lead, p_lead):
    c = ctx()
    for n, batch in ((5, 17), (2047, 3), (2049, 5), (8191, 2)):
        P = _points(n, 300 + n, p_lead)[p_lead:]
        assert P.data_ptr() % 16 != 0 and P.data_ptr() % 4 == 0
        _, S = _scalars(batch, n, 400 + n, s_lead)
        _check_rows(c, P, S)


def test_longer_srs_and_points_past_the_rows():
    """n_points > n_scalars: only the first n_scalars points are read, so an off-curve point after them is no error."""
    import torch
    from ronkathon_b200 import ops
    c = ctx()
    P = _points(100, 500)
    P[60] = torch.tensor([36, 0, 0, 81], dtype=torch.uint8)
    _, S = _scalars(9, 60, 501)
    got = ops.msm_batch(c, P, S).cpu().numpy()
    for r in range(9):
        assert got[r].tobytes() == oracle.commit(S[r].cpu().numpy(), P[:60].cpu().numpy(), fast=True)


def test_reference_kats_as_rows_of_one_batch(kats):
    """kzg/tests.rs:93-137: [11,11,11,1] → ∞, [7,16,1,11,1] → (32,59), [3,2,1] → (32,59), zero-padded to 5."""
    from ronkathon_b200 import kzg
    ctx()
    g1, _ = kzg.setup()
    cases = kats["kzg"]["commit"]
    got = kzg.commit_batch([cs["coeffs"] for cs in cases], g1)
    assert [p.raw for p in got] == [pt(cs["out"]) for cs in cases]
    assert got[0].raw == INF and got[1].raw == bytes([32, 0, 59, 0]) == got[2].raw


# ---- scale -------------------------------------------------------------------------------------------------------------

def test_more_than_65535_rows():
    from ronkathon_b200 import ops
    c = ctx()
    n, batch = 5, 70001
    P = _points(n, 600)
    buf, S = _scalars(batch, n, 601, 1)
    got = ops.msm_batch(c, P, S).cpu().numpy()
    pts, sc = P.cpu().numpy(), S.cpu().numpy()
    for r in range(batch):
        assert got[r].tobytes() == oracle.commit(sc[r], pts, fast=True), r
    for r in (0, 65535, 65536, batch - 1):
        assert got[r].tobytes() == _single(c, P, S[r])


def test_scalar_block_past_2_32_bytes():
    """4097 rows of 2^20 + 3 scalars: 4.3·10^9 bytes, so the last rows start past 2^32."""
    import torch
    from ronkathon_b200 import ops
    c = ctx()
    n, batch = (1 << 20) + 3, 4097
    assert batch * n > 1 << 32
    P = _points(n, 700)
    buf, S = _scalars(batch, n, 701)
    got = ops.msm_batch(c, P, S).cpu().numpy()
    pts = P.cpu().numpy()
    for r in (0, 4095, 4096):
        assert got[r].tobytes() == _single(c, P, S[r]), r
        assert got[r].tobytes() == oracle.commit(S[r].cpu().numpy(), pts, fast=True), r
    del buf, S
    torch.cuda.empty_cache()


def test_long_row_of_sixteens():
    """One 2^24-term row of all-16 scalars over whole-group points: the largest terms, longest columns of one row."""
    import torch
    from ronkathon_b200 import ops
    c = ctx()
    n = 1 << 24
    P = _points(n, 800)
    S = torch.full((1, n), 16, dtype=torch.uint8, device="cuda")
    got = ops.msm_batch(c, P, S).cpu().numpy()[0].tobytes()
    assert got == _single(c, P, S[0])
    assert got == oracle.commit(np.full(n, 16, np.uint8), P.cpu().numpy(), fast=True)


# ---- refusals ----------------------------------------------------------------------------------------------------------

def _poisoned(batch, extra=0):
    import torch
    return torch.full((batch * 4 + extra,), POISON, dtype=torch.uint8, device="cuda")


def test_rejected_terms_leave_out_unwritten():
    """A scalar 17 in the last byte of the last row, and an off-curve or non-canonical point: RONK_EINVAL after the three
    launches, with out byte for byte as it was; the next call on the context is unaffected."""
    import torch
    from ronkathon_b200 import ops
    c = ctx()
    name = "ronk_msm_pluto_ext_batch"
    for n, batch in ((4095, 17), (5, 3), (1 << 16, 256)):
        P = _points(n, 900 + n)
        _, S = _scalars(batch, n, 901 + n, 1)
        good = ops.msm_batch(c, P, S).clone()
        out = _poisoned(batch)
        bad = S.clone()
        bad[-1, -1] = 17
        assert _rc(c, name, _p(P), n, _p(bad), n, batch, _p(out)) == (EINVAL, 3)
        assert bool((out == POISON).all())
        for w in ([36, 0, 0, 81], [101, 0, 2, 0]):
            Q = P.clone()
            Q[n // 2] = torch.tensor(w, dtype=torch.uint8)
            assert _rc(c, name, _p(Q), n, _p(S), n, batch, _p(out)) == (EINVAL, 3)
            assert bool((out == POISON).all())
        assert torch.equal(ops.msm_batch(c, P, S), good)


def test_argument_refusals_write_nothing():
    import torch
    c = ctx()
    n, batch = 64, 5
    P = _points(n, 950)
    buf, S = _scalars(batch, n, 951)
    out = _poisoned(batch, 4)
    name = "ronk_msm_pluto_ext_batch"
    cases = [
        ((_p(P), n - 1, _p(S), n, batch, _p(out)), EINVAL),                     # n_points < n_scalars
        ((None, n, _p(S), n, batch, _p(out)), EINVAL),                          # null points
        ((_p(P), n, None, n, batch, _p(out)), EINVAL),                          # null scalars
        ((_p(P), n, _p(S), n, batch, None), EINVAL),                            # null out
        ((_p(P), n, _p(S), n, batch, out.data_ptr() + 1), EINVAL),              # misaligned out
        ((P.data_ptr() + 2, n, _p(S), n, batch, _p(out)), EINVAL),              # misaligned points
        ((_p(P), n, _p(S), n, batch, buf.data_ptr()), EINVAL),                  # out over the scalars
        ((_p(P), n, _p(S), n, batch, S.data_ptr() + 4 * n), EINVAL),            # … from inside the block
        ((_p(P), n, _p(S), n, batch, P.data_ptr() + 4 * (n - 1)), EINVAL),      # out over the points
        ((_p(P), n, _p(S), n, 0, _p(out)), 0),                                  # batch 0
        ((None, 0, None, n, 0, None), EINVAL),                                  # batch 0 still checks n_points
        ((None, n, None, n, 0, None), 0),
        ((_p(P), n, _p(S), n, 1 << 20, _p(out)), EUNSUPPORTED),                 # batch·n above 2^40 bytes
    ]
    for args, want in cases:
        if want == EUNSUPPORTED:
            args = (args[0], 1 << 21, args[2], (1 << 20) + 1, args[4], args[5])
        rc, launches = _rc(c, name, *args)
        assert (rc, launches) == (want, 0), (args, rc, launches)
        assert bool((out == POISON).all()), args
    # a refused call has enqueued nothing: the next call still gives the words
    from ronkathon_b200 import ops
    got = ops.msm_batch(c, P, S).cpu().numpy()
    assert got[batch - 1].tobytes() == _single(c, P, S[batch - 1])
    assert _rc(c, name, None, 0, None, 0, 0, None) == (0, 0)
    from ronkathon_b200 import _lib
    assert _lib.lib().ronk_msm_pluto_ext_batch(None, _p(P), n, _p(S), n, batch, _p(out)) == EINVAL
    torch.cuda.synchronize()
    assert bool((out == POISON).all())


def test_empty_rows_are_infinity():
    c = ctx()
    out = _poisoned(7, 4)
    assert _rc(c, "ronk_msm_pluto_ext_batch", None, 0, None, 0, 7, _p(out)) == (0, 0)
    assert bytes(out[:28].cpu().numpy()) == INF * 7 and bool((out[28:] == POISON).all())
    P = _points(3, 960)
    out.fill_(POISON)
    assert _rc(c, "ronk_msm_pluto_ext_batch", _p(P), 3, None, 0, 7, _p(out)) == (0, 0)
    assert bytes(out[:28].cpu().numpy()) == INF * 7


def test_host_twin_refuses_before_staging():
    c = ctx()
    pts = np.full((4, 4), 0xFF, np.uint8)
    sc = np.zeros(8, np.uint8)
    out = np.full(16, POISON, np.uint8)
    name = "ronk_msm_pluto_ext_batch_host"
    for args, want in [
        ((_p(pts), 3, _p(sc), 4, 2, _p(out)), EINVAL),                          # n_points < n_scalars
        ((None, 4, _p(sc), 4, 2, _p(out)), EINVAL),
        ((_p(pts), 4, _p(sc), 4, 2, None), EINVAL),
        ((_p(pts), 1 << 21, _p(sc), (1 << 20) + 1, 1 << 20, _p(out)), EUNSUPPORTED),   # would stage 2^40 bytes
        ((_p(pts), 4, _p(sc), 4, 0, _p(out)), 0),
    ]:
        assert _rc(c, name, *args) == (want, 0), args
    assert np.all(out == POISON)


# ---- launches, host twin, streams --------------------------------------------------------------------------------------

def test_launch_count_does_not_depend_on_the_batch():
    from ronkathon_b200 import ops
    c = ctx()
    n = 4095
    P = _points(n, 1000)
    counts = []
    for batch in (2, 17, 256):
        _, S = _scalars(batch, n, 1001 + batch)
        ops.msm_batch(c, P, S)   # warm: tables and scratch
        c.sync()
        before = c.launches
        ops.msm_batch(c, P, S)
        counts.append(c.launches - before)
    assert counts == [3, 3, 3]


def test_host_twin_gives_the_device_words():
    from ronkathon_b200 import ops
    c = ctx()
    for n, batch in ((7, 4096), (4095, 3), ((1 << 16) + 3, 17)):
        P = _points(n + 5, 1100 + n)
        _, S = _scalars(batch, n, 1101 + n)
        want = ops.msm_batch(c, P, S).cpu().numpy()
        pts, sc = P.cpu().numpy(), S.cpu().numpy()
        out = np.full((batch, 4), POISON, np.uint8)
        c.call("ronk_msm_pluto_ext_batch_host", _p(pts), n + 5, _p(sc), n, batch, _p(out))
        assert np.array_equal(out, want), (n, batch)


def test_gated_non_blocking_stream():
    """A batched commit on a fresh context's non-blocking stream behind a spin: it waits for the stream's earlier work
    (the real scalars are written behind the spin), and its words are the default stream's."""
    import torch
    from ronkathon_b200 import Context, ops
    c0 = ctx()
    n, batch = 4095, 17
    P = _points(n, 1200)
    _, S = _scalars(batch, n, 1201)
    want = ops.msm_batch(c0, P, S).cpu().numpy()
    s = torch.cuda.Stream()
    c = Context(0, s.cuda_stream)
    try:
        with torch.cuda.stream(s):
            ops.msm_batch(c, P, S)   # warm: tables and scratch
        s.synchronize()
        Sg = torch.flip(S, dims=[1]).contiguous()   # valid but wrong rows until the gate opens
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            torch.cuda._sleep(100_000_000)
            Sg.copy_(S)
            got = ops.msm_batch(c, P, Sg)
        s.synchronize()
        assert np.array_equal(got.cpu().numpy(), want)
    finally:
        c.close()


# ---- Python layer ------------------------------------------------------------------------------------------------------

def test_commit_batch_equals_commit_on_ragged_rows():
    from ronkathon_b200 import RonkPanic, kzg
    ctx()
    g1, _ = kzg.setup()
    rng = np.random.default_rng(1300)
    rows = [[int(v) for v in rng.integers(-40, 200, int(k))] for k in rng.integers(0, 8, 40)]
    rows += [[], [0, 0, 0], [17, 34], list(range(7))]
    assert kzg.commit_batch(rows, g1) == [kzg.commit(r, g1) for r in rows]
    assert kzg.commit_batch([], g1) == []
    with pytest.raises(RonkPanic):          # kzg/setup.rs:53, as commit panics on the long row
        kzg.commit_batch([[1, 2], [1] * 8], g1)
    with pytest.raises(RonkPanic):
        kzg.commit([1] * 8, g1)


def test_open_batch_through_commit_batch():
    from ronkathon_b200 import kzg
    ctx()
    g1, _ = kzg.setup()
    assert kzg.open_batch([[11, 11, 11, 1]], 4, g1)[0].raw == bytes([26, 0, 45, 0])   # kzg/tests.rs:327-337
    polys = [[int(v) % 17 for v in oracle.splitmix(17, 1400 + i, 2 + (i % 6))] for i in range(12)]
    assert kzg.open_batch(polys, 9, g1) == [kzg.open_(f, 9, g1) for f in polys]


def test_commit_preprocessed_equals_commit_lagrange():
    import plonk_vectors as pv
    from ronkathon_b200 import AffinePoint, kzg
    ctx()
    for n in (4, 8, 16):
        polys = pv.REFERENCE_N4 if n == 4 else pv.padded(n)
        srs = [AffinePoint(bytes(r)) for r in pv.srs(oracle, n)]
        assert kzg.commit_preprocessed(polys, srs) == {k: kzg.commit_lagrange(v, srs) for k, v in polys.items()}
