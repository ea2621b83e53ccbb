"""ronk_sha256 and its _host twin (hashes.Sha256, ops.sha256): batches of the reference's SHA-256 (src/hashes/sha.rs)
against Python's hashlib.

The reference's known answers, ragged batches (empty messages, the padding edges 55/56/63/64/119/120, every start
alignment, one 1 MiB message), batches around a warp, a CTA and one grid, poisoned slack around the output, refusals
in the header's order with nothing written, device-flagged offsets, the _host twin and a gated non-blocking stream."""
import hashlib
import json
import os

import numpy as np
import pytest

from gpu_util import ctx

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
EINVAL, EUNSUPPORTED = 1, 5
POISON = 0xA5
CTA = 128   # threads per CTA of sha256_kernel


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


def _u8(b: bytes, lead: int = 0):
    """A uint8 device tensor holding b after `lead` filler bytes, and the view of b in it."""
    import torch
    t = torch.full((lead + len(b) + 1,), POISON, dtype=torch.uint8, device="cuda")
    if b:
        t[lead:lead + len(b)] = torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda()
    return t[lead:lead + len(b)]


def _i64(a):
    from ronkathon_b200 import ops
    return ops.to_device(np.asarray(a, dtype=np.uint64))


def _batch(msgs, lead=0):
    offs = np.zeros(len(msgs) + 1, np.uint64)
    offs[1:] = np.cumsum([len(m) for m in msgs])
    return _u8(b"".join(msgs), lead), _i64(offs)


def _digests(c, msgs, lead=0):
    """(digests [n] as bytes, launches) through ronk_sha256."""
    import torch
    data, offs = _batch(msgs, lead)
    out = torch.empty((max(len(msgs), 1), 32), dtype=torch.uint8, device="cuda")
    code, launches = _rc(c, "ronk_sha256", _p(data) if data.numel() else None, data.numel(), _p(offs), len(msgs), _p(out))
    assert code == 0, c.check(code)
    h = out.cpu().numpy()
    return [h[i].tobytes() for i in range(len(msgs))], launches


def _want(msgs):
    return [hashlib.sha256(m).digest() for m in msgs]


# ---- the reference's known answers -----------------------------------------------------------------------------------

def test_reference_known_answers():
    from ronkathon_b200.hashes import Sha256
    with open(os.path.join(HERE, "golden", "sha_merkle_kats.json")) as f:
        cases = json.load(f)["sha256"]
    c = ctx()
    msgs = [k["input"].encode() for k in cases]
    got, launches = _digests(c, msgs)
    assert launches == 1 and [g.hex() for g in got] == [k["digest"] for k in cases]
    for k in cases:
        assert Sha256().digest(k["input"].encode()).hex() == k["digest"], k["src"]


# ---- ragged batches --------------------------------------------------------------------------------------------------

def test_ragged_batch_padding_edges_and_alignments():
    c = ctx()
    rng = np.random.default_rng(3)
    lengths = [0, 1, 3, 4, 5, 31, 32, 33, 55, 56, 57, 63, 64, 65, 119, 120, 121, 127, 128, 0, 200, 0]
    msgs = [rng.integers(0, 256, n, dtype=np.uint8).tobytes() for n in lengths]
    for lead in range(8):   # the batch's first byte at every alignment mod 8; each message then lands where it lands
        got, launches = _digests(c, msgs, lead)
        assert launches == 1 and got == _want(msgs), lead
    # every length 0 … 130 starting at each alignment mod 4
    for a in range(4):
        ms = [bytes([7] * a)] + [rng.integers(0, 256, n, dtype=np.uint8).tobytes() for n in range(131)]
        data, offs = _batch(ms)
        sub = offs[1:].contiguous()   # the batch without the alignment filler
        import torch
        out = torch.empty((131, 32), dtype=torch.uint8, device="cuda")
        assert _rc(c, "ronk_sha256", _p(data), data.numel(), _p(sub), 131, _p(out)) == (0, 1)
        h = out.cpu().numpy()
        assert [h[i].tobytes() for i in range(131)] == _want(ms[1:]), a


def test_one_mebibyte_message_among_small_ones():
    c = ctx()
    rng = np.random.default_rng(4)
    msgs = [b"abc", rng.integers(0, 256, 1 << 20, dtype=np.uint8).tobytes(), b"", b"x" * 77]
    got, launches = _digests(c, msgs, lead=3)
    assert launches == 1 and got == _want(msgs)


def test_batches_around_a_warp_a_cta_and_one_grid():
    import torch
    c = ctx()
    rng = np.random.default_rng(5)
    grid = torch.cuda.get_device_properties(0).multi_processor_count * 8 * CTA
    for n in (1, 31, 32, 33, CTA - 1, CTA, CTA + 1, grid - 1, grid, grid + 1):
        lens = rng.integers(0, 70, n)
        blob = rng.integers(0, 256, int(lens.sum()), dtype=np.uint8).tobytes()
        offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
        msgs = [blob[offs[i]:offs[i + 1]] for i in range(n)]
        got, launches = _digests(c, msgs, lead=1)
        assert launches == 1 and got == _want(msgs), n
    assert _rc(c, "ronk_sha256", None, 0, None, 0, None) == (0, 0)


def test_ops_sha256_and_offsets_starting_past_zero():
    from ronkathon_b200 import ops
    c = ctx()
    blob = bytes(range(256)) * 4
    offs = [5, 5, 17, 80, 81, 700]
    got = ops.sha256(c, _u8(blob), _i64(offs)).cpu().numpy()
    assert got.shape == (5, 32)
    assert [got[i].tobytes() for i in range(5)] == _want([blob[offs[i]:offs[i + 1]] for i in range(5)])


# ---- slack, refusals, flags ------------------------------------------------------------------------------------------

def test_slack_around_output_stays_poisoned():
    import torch
    c = ctx()
    msgs = [b"a" * i for i in range(37)]
    data, offs = _batch(msgs, lead=2)
    buf = torch.full((37 * 32 + 2 * 19,), POISON, dtype=torch.uint8, device="cuda")
    out = buf[19:19 + 37 * 32]
    assert _rc(c, "ronk_sha256", _p(data), data.numel(), _p(offs), 37, _p(out)) == (0, 1)
    h = buf.cpu().numpy()
    assert (h[:19] == POISON).all() and (h[-19:] == POISON).all()
    assert [h[19 + 32 * i:19 + 32 * i + 32].tobytes() for i in range(37)] == _want(msgs)


def test_refusals_in_order_write_nothing():
    import torch
    c = ctx()
    data, offs = _batch([b"abc", b"defg"])
    out = torch.full((64,), POISON, dtype=torch.uint8, device="cuda")
    raw = torch.zeros(8, dtype=torch.int64, device="cuda")
    mis = raw.view(torch.uint8)[1:41]   # offsets one byte off 8-byte alignment
    P = _p

    def call(d=data, dl=7, o=offs, n=2, out_=out):
        return _rc(c, "ronk_sha256", P(d) if d is not None else None, dl, P(o) if o is not None else None, n,
                   P(out_) if out_ is not None else None)

    cases = [
        ("null data with bytes, before n ≥ 2^32", call(d=None, n=1 << 32), EINVAL),
        ("null offsets", call(o=None), EINVAL),
        ("null out", call(out_=None), EINVAL),
        ("misaligned offsets before n ≥ 2^32", call(o=mis, n=1 << 32), EINVAL),
        ("n ≥ 2^32", call(n=1 << 32), EUNSUPPORTED),
        ("data_len above 2^40", call(dl=(1 << 40) + 1), EUNSUPPORTED),
        ("size before overlap", call(out_=data, dl=(1 << 40) + 1), EUNSUPPORTED),
        ("out overlaps data", call(out_=data), EINVAL),
        ("out overlaps offsets", call(out_=offs), EINVAL),
    ]
    for name, (code, launches), want in cases:
        assert (code, launches) == (want, 0), name
    assert (out.cpu().numpy() == POISON).all()
    assert call(d=None, dl=0, n=0, o=None, out_=None) == (0, 0)
    # data may be null when there are no bytes: n empty messages
    empty = _i64([0, 0, 0])
    assert call(d=None, dl=0, o=empty, n=2) == (0, 1)
    h = out.cpu().numpy()
    assert h[:32].tobytes() == h[32:].tobytes() == hashlib.sha256(b"").digest()


@pytest.mark.parametrize("offs", [[0, 4, 3], [0, 3, 8], [2, 1, 3], [0, 7, 7, 2]])
def test_bad_offsets_are_flagged_after_one_launch(offs):
    import torch
    c = ctx()
    data = _u8(b"abcdefg")
    out = torch.empty((len(offs) - 1, 32), dtype=torch.uint8, device="cuda")
    assert _rc(c, "ronk_sha256", _p(data), 7, _p(_i64(offs)), len(offs) - 1, _p(out)) == (EINVAL, 1)
    assert _rc(c, "ronk_sha256", _p(data), 7, _p(_i64([0, 3, 7])), 2, _p(out)) == (0, 1)   # the flag is cleared


def test_host_twin():
    c = ctx()
    rng = np.random.default_rng(6)
    msgs = [rng.integers(0, 256, n, dtype=np.uint8).tobytes() for n in (0, 55, 56, 64, 1000, 3)]
    blob = np.frombuffer(b"".join(msgs), np.uint8).copy()
    offs = np.concatenate([[0], np.cumsum([len(m) for m in msgs])]).astype(np.uint64)
    out = np.zeros((6, 32), np.uint8)
    assert _rc(c, "ronk_sha256_host", _p(blob), blob.size, _p(offs), 6, _p(out)) == (0, 1)
    assert [out[i].tobytes() for i in range(6)] == _want(msgs)
    # bad offsets are refused on the host before anything is staged or launched, with nothing written
    out[:] = POISON
    for bad in ([0, 5, 4], [0, 5, blob.size + 1]):
        o = np.array(bad, np.uint64)
        assert _rc(c, "ronk_sha256_host", _p(blob), blob.size, _p(o), 2, _p(out)) == (EINVAL, 0)
    assert (out == POISON).all()


def test_gated_non_blocking_stream():
    import torch
    from ronkathon_b200 import Context, ops
    rng = np.random.default_rng(7)
    msgs = [rng.integers(0, 256, int(n), dtype=np.uint8).tobytes() for n in rng.integers(0, 200, 3000)]
    data, offs = _batch(msgs)
    s = torch.cuda.Stream()
    c = Context(0, s.cuda_stream)
    try:
        g = torch.zeros_like(data)
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            torch.cuda._sleep(100_000_000)
            g.copy_(data)
            got = ops.sha256(c, g, offs)
        s.synchronize()
        h = got.cpu().numpy()
        assert [h[i].tobytes() for i in range(len(msgs))] == _want(msgs)
    finally:
        c.close()
