"""ronk_poseidon_permute_u64 and ronk_poseidon_sponge_u64 (hashes.Poseidon / PoseidonSponge, ops.poseidon_permute_,
ops.poseidon_hash, ops.poseidon_sponge): batches of the reference's Poseidon permutation and sponge.

Every width 2 … 16, each test prime (both field policies) and each class of S-box exponent and round count is checked
against the C restatement of the reference (tests/poseidon_oracle.c), as are the sponge's rate and length edges, batches
around a warp and past one grid, the _host twins and a gated non-blocking stream.  Refusals must come in the header's
order with nothing written and nothing launched."""
import json
import os

import numpy as np
import pytest

import poseidon_oracle as po
from gpu_util import GL, ctx

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
EINVAL, EUNSUPPORTED = 1, 5
PRIMES = [17, 101, 127, GL, (1 << 61) - 1, (1 << 64) - 59]
POISON = 0x5A5A5A5A5A5A5A5A


def _kats():
    with open(os.path.join(HERE, "golden", "poseidon_kats.json")) as f:
        return json.load(f)


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


def _rand(rng, p, n):
    return rng.integers(0, 2**64, size=n, dtype=np.uint64) % np.uint64(p)


def _cfg(rng, p, width, alpha=5, num_f=8, num_p=11):
    return po.Config(p, width, alpha, num_p, num_f, _rand(rng, p, (num_f + num_p) * width).tolist(),
                     _rand(rng, p, width * width).reshape(width, width).tolist())


def _dev(a):
    from ronkathon_b200 import ops
    return ops.to_device(np.ascontiguousarray(a, dtype=np.uint64))


def _host(t):
    from ronkathon_b200 import ops
    ctx().sync()
    return ops.to_host(t)


def _consts(cfg):
    return _dev(cfg.rc), _dev(cfg.mds)


def _permute_dev(c, cfg, states):
    """States through ronk_poseidon_permute_u64; (words, launches)."""
    s = _dev(states)
    rc, mds = _consts(cfg)
    code, launches = _rc(c, "ronk_poseidon_permute_u64", cfg.p, cfg.width, cfg.alpha, cfg.num_f, cfg.num_p, _p(rc), _p(mds),
                         _p(s), np.asarray(states).shape[0])
    assert code == 0, c.check(code)
    return _host(s).reshape(np.asarray(states).shape), launches


def _sponge_dev(c, cfg, rate, rows, n_out):
    import torch
    rows = np.ascontiguousarray(rows, dtype=np.uint64)
    batch, length = rows.shape
    inp = _dev(rows) if rows.size else torch.empty(1, dtype=torch.int64, device="cuda")
    out = torch.empty(max(batch * n_out, 1), dtype=torch.int64, device="cuda")
    rc, mds = _consts(cfg)
    code, launches = _rc(c, "ronk_poseidon_sponge_u64", cfg.p, cfg.width, cfg.alpha, cfg.num_f, cfg.num_p, _p(rc), _p(mds),
                         rate, _p(inp), length, batch, _p(out), n_out)
    assert code == 0, c.check(code)
    return _host(out)[:batch * n_out].reshape(batch, n_out), launches


# ---- the reference's known answer ------------------------------------------------------------------------------------

def test_reference_kat_through_hash_and_ops():
    import torch
    from ronkathon_b200 import RonkPanic, ops
    from ronkathon_b200.field import PlutoBaseField
    from ronkathon_b200.hashes import Poseidon, PoseidonConfig
    k = _kats()
    c = ctx()
    h = Poseidon(k["width"], k["alpha"], k["num_p"], k["num_f"], [PlutoBaseField(v) for v in k["rc16"]],
                 [[PlutoBaseField(v) for v in r] for r in k["mds16"]])
    assert h.hash([PlutoBaseField(0)] * 16) == PlutoBaseField(20)
    assert h.hash([]) == PlutoBaseField(20)
    cfg = PoseidonConfig(k["width"], k["alpha"], k["num_p"], k["num_f"], k["rc16"], k["mds16"], field=PlutoBaseField)
    orc = po.Config(101, 16, k["alpha"], k["num_p"], k["num_f"], k["rc16"], k["mds16"])
    rng = np.random.default_rng(5)
    rows = _rand(rng, 101, 40 * 7).reshape(40, 7)
    rows[0] = 0
    got = _host(ops.poseidon_hash(c, _dev(rows), cfg))
    assert int(got[0]) == 20
    assert got.tolist() == [po.hash_(orc, r.tolist()) for r in rows]
    with pytest.raises(RonkPanic):
        h.hash([0] * 17)
    with pytest.raises(RonkPanic):
        ops.poseidon_hash(c, torch.zeros((1, 17), dtype=torch.int64, device="cuda"), cfg)


# ---- every width, prime and exponent class -----------------------------------------------------------------------------

@pytest.mark.parametrize("p", PRIMES)
def test_every_width_both_entries(p):
    c = ctx()
    rng = np.random.default_rng(p % 10007)
    for width in range(2, 17):
        cfg = _cfg(rng, p, width)
        states = _rand(rng, p, 33 * width).reshape(33, width)
        assert np.array_equal(_permute_dev(c, cfg, states)[0], po.permute(cfg, states)), (p, width)
        rate = max(1, width - 2)
        rows = _rand(rng, p, 5 * (2 * rate + 1)).reshape(5, 2 * rate + 1)
        got, _ = _sponge_dev(c, cfg, rate, rows, rate + 2)
        assert np.array_equal(got, po.sponge_rows(cfg, rate, rows, rate + 2)), (p, width)


@pytest.mark.parametrize("p", PRIMES)
def test_alpha_and_round_classes(p):
    c = ctx()
    rng = np.random.default_rng(p % 4099)
    for alpha in (0, 1, 2, 3, 5, 7, p - 2):
        for num_f, num_p in ((8, 11), (7, 3), (3, 0), (0, 4), (0, 0)):
            for width in (2, 9, 16):
                cfg = _cfg(rng, p, width, alpha, num_f, num_p)
                states = _rand(rng, p, 6 * width).reshape(6, width)
                states[0] = 0
                assert np.array_equal(_permute_dev(c, cfg, states)[0], po.permute(cfg, states)), (p, alpha, num_f, num_p, width)


def test_zero_rounds_takes_null_constants():
    c = ctx()
    rng = np.random.default_rng(2)
    states = _rand(rng, 101, 3 * 4)
    s = _dev(states)
    assert _rc(c, "ronk_poseidon_permute_u64", 101, 4, 3, 0, 0, None, None, _p(s), 3) == (0, 1)
    assert np.array_equal(_host(s), states)


# ---- sponge edges ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("p", [101, GL, (1 << 64) - 59])
def test_sponge_rate_and_length_edges(p):
    c = ctx()
    rng = np.random.default_rng(p % 811)
    for width in (2, 5, 16):
        cfg = _cfg(rng, p, width, 7, 4, 5)
        for rate in sorted({1, width - 1, width}):
            for length in (0, 1, rate, 3 * rate, 3 * rate + 1):
                for n_out in (1, rate, 2 * rate, 2 * rate + 1, 3):
                    rows = _rand(rng, p, 4 * length).reshape(4, length)
                    got, launches = _sponge_dev(c, cfg, rate, rows, n_out)
                    assert launches == 1
                    assert np.array_equal(got, po.sponge_rows(cfg, rate, rows, n_out)), (width, rate, length, n_out)
                    if length == 0:
                        assert not got[:, :rate].any()    # no permutation before the first squeeze: the zero state
        got, launches = _sponge_dev(c, cfg, 1, _rand(rng, p, 8).reshape(2, 4), 0)
        assert launches == 0 and got.shape == (2, 0)


# ---- batches ---------------------------------------------------------------------------------------------------------

def test_batches_around_a_warp_and_past_one_grid():
    import torch
    c = ctx()
    rng = np.random.default_rng(9)
    grid_rows = torch.cuda.get_device_properties(0).multi_processor_count * 8 * 128
    for p, width in ((GL, 3), (101, 4)):
        cfg = _cfg(rng, p, width, 7, 2, 1)
        for batch in (1, 31, 32, 33, grid_rows + 1):
            states = _rand(rng, p, batch * width).reshape(batch, width)
            got, launches = _permute_dev(c, cfg, states)
            assert launches == 1 and np.array_equal(got, po.permute(cfg, states)), (p, batch)
        for batch in (1, 33, grid_rows + 1):
            rows = _rand(rng, p, batch * 5).reshape(batch, 5)
            got, launches = _sponge_dev(c, cfg, 2, rows, 3)
            assert launches == 1 and np.array_equal(got, po.sponge_rows(cfg, 2, rows, 3)), (p, batch)
    s = _dev(np.zeros(4, np.uint64))
    rc, mds = _consts(cfg)
    assert _rc(c, "ronk_poseidon_permute_u64", 101, 4, 7, 2, 1, _p(rc), _p(mds), _p(s), 0) == (0, 0)
    assert _rc(c, "ronk_poseidon_sponge_u64", 101, 4, 7, 2, 1, _p(rc), _p(mds), 2, _p(s), 4, 0, _p(s), 4) == (0, 0)


def test_slack_around_outputs_stays_poisoned():
    import torch
    c = ctx()
    rng = np.random.default_rng(11)
    p, width, batch, slack = GL, 6, 37, 19
    cfg = _cfg(rng, p, width)
    rc, mds = _consts(cfg)
    states = _rand(rng, p, batch * width)
    buf = torch.full((batch * width + 2 * slack,), POISON, dtype=torch.int64, device="cuda")
    buf[slack:slack + batch * width] = _dev(states)
    view = buf[slack:slack + batch * width]
    assert _rc(c, "ronk_poseidon_permute_u64", p, width, cfg.alpha, cfg.num_f, cfg.num_p, _p(rc), _p(mds), _p(view), batch)[0] == 0
    h = _host(buf)
    assert (h[:slack] == POISON).all() and (h[-slack:] == POISON).all()
    assert np.array_equal(h[slack:-slack], po.permute(cfg, states.reshape(batch, width)).reshape(-1))
    length, n_out = 9, 7
    rows = _rand(rng, p, batch * length)
    inp = _dev(rows)
    buf = torch.full((batch * n_out + 2 * slack,), POISON, dtype=torch.int64, device="cuda")
    out = buf[slack:slack + batch * n_out]
    assert _rc(c, "ronk_poseidon_sponge_u64", p, width, cfg.alpha, cfg.num_f, cfg.num_p, _p(rc), _p(mds), 4, _p(inp), length,
               batch, _p(out), n_out)[0] == 0
    h = _host(buf)
    assert (h[:slack] == POISON).all() and (h[-slack:] == POISON).all()
    assert np.array_equal(h[slack:-slack].reshape(batch, n_out), po.sponge_rows(cfg, 4, rows.reshape(batch, length), n_out))


# ---- refusals ----------------------------------------------------------------------------------------------------------

def test_refusals_in_order_write_nothing():
    import torch
    c = ctx()
    rng = np.random.default_rng(13)
    cfg = _cfg(rng, 101, 4, 3, 2, 1)
    rc, mds = _consts(cfg)
    big_rc = _dev(np.zeros(369 * 16, np.uint64))
    out = torch.full((64,), POISON, dtype=torch.int64, device="cuda")
    inp = _dev(_rand(rng, 101, 64))
    P, N = _p, None

    def perm(p=101, w=4, nf=2, np_=1, rc_=rc, mds_=mds, s=out, b=3):
        return _rc(c, "ronk_poseidon_permute_u64", p, w, 3, nf, np_, P(rc_) if rc_ is not None else N,
                   P(mds_) if mds_ is not None else N, P(s) if s is not None else N, b)

    def sponge(p=101, w=4, nf=2, np_=1, rc_=rc, mds_=mds, rate=2, i=inp, ln=5, b=3, o=out, n=4):
        return _rc(c, "ronk_poseidon_sponge_u64", p, w, 3, nf, np_, P(rc_) if rc_ is not None else N,
                   P(mds_) if mds_ is not None else N, rate, P(i) if i is not None else N, ln, b, P(o) if o is not None else N, n)

    cases = [
        ("null states before a bad modulus", perm(p=100, s=None), EINVAL),
        ("null rc", perm(rc_=None), EINVAL),
        ("null mds", perm(mds_=None), EINVAL),
        ("p = 2 before width", perm(p=2, w=1), EUNSUPPORTED),
        ("composite p before width", perm(p=100, w=1), EINVAL),
        ("width 1", perm(w=1, nf=0, np_=0), EINVAL),
        ("width 17", perm(w=17), EUNSUPPORTED),
        ("constants past 48 KiB", perm(w=16, nf=8, np_=361, rc_=big_rc), EUNSUPPORTED),
        ("batch·width past 2^40", perm(b=1 << 39), EUNSUPPORTED),
        ("states overlap rc", perm(s=rc, b=1), EINVAL),
        ("sponge: null in", sponge(i=None), EINVAL),
        ("sponge: null out", sponge(o=None), EINVAL),
        ("sponge: composite p before rate", sponge(p=100, rate=0), EINVAL),
        ("sponge: rate 0", sponge(rate=0), EINVAL),
        ("sponge: rate > width before width 17", sponge(w=17, rate=18), EINVAL),
        ("sponge: width 17", sponge(w=17, rate=2), EUNSUPPORTED),
        ("sponge: batch·len past 2^40", sponge(ln=1 << 40, b=2), EUNSUPPORTED),
        ("sponge: batch·n_out past 2^40", sponge(n=1 << 40, b=2), EUNSUPPORTED),
        ("sponge: size before overlap", sponge(o=inp, n=1 << 40, b=2), EUNSUPPORTED),
        ("sponge: out overlaps in", sponge(o=inp), EINVAL),
        ("sponge: out overlaps mds", sponge(o=mds), EINVAL),
    ]
    for name, (code, launches), want in cases:
        assert (code, launches) == (want, 0), name
    assert (_host(out) == POISON).all()
    assert perm(rc_=None, mds_=None, nf=0, np_=0) == (0, 1)     # zero rounds read neither table
    assert sponge(i=None, ln=0, n=0, o=None) == (0, 0)
    assert _rc(c, "ronk_poseidon_permute_u64", 101, 4, 3, 2, 1, None, None, None, 0) == (0, 0)


def test_host_twins():
    c = ctx()
    rng = np.random.default_rng(17)
    from ronkathon_b200 import _lib
    for p in (101, GL, (1 << 64) - 59):
        cfg = _cfg(rng, p, 7)
        states = _rand(rng, p, 9 * 7).reshape(9, 7)
        s = states.copy()
        assert _lib.lib().ronk_poseidon_permute_u64_host(c._h, p, 7, cfg.alpha, cfg.num_f, cfg.num_p, _p(cfg.rc), _p(cfg.mds),
                                                         _p(s), 9) == 0
        assert np.array_equal(s, po.permute(cfg, states))
        rows = _rand(rng, p, 9 * 11).reshape(9, 11)
        out = np.zeros((9, 5), np.uint64)
        assert _lib.lib().ronk_poseidon_sponge_u64_host(c._h, p, 7, cfg.alpha, cfg.num_f, cfg.num_p, _p(cfg.rc), _p(cfg.mds), 3,
                                                        _p(rows), 11, 9, _p(out), 5) == 0
        assert np.array_equal(out, po.sponge_rows(cfg, 3, rows, 5))
    # non-canonical words are refused before staging, with nothing written
    cfg = _cfg(rng, 101, 3, 3, 2, 1)
    bad_rc = cfg.rc.copy()
    bad_rc[-1] = 101
    for rc_, st in ((bad_rc, np.zeros(3, np.uint64)), (cfg.rc, np.array([0, 101, 0], np.uint64))):
        s = st.copy()
        code, launches = _rc(c, "ronk_poseidon_permute_u64_host", 101, 3, 3, 2, 1, _p(rc_), _p(cfg.mds), _p(s), 1)
        assert (code, launches) == (EINVAL, 0) and np.array_equal(s, st)
    out = np.full(4, POISON, np.uint64)
    inp = np.array([5, 101], np.uint64)
    assert _rc(c, "ronk_poseidon_sponge_u64_host", 101, 3, 3, 2, 1, _p(cfg.rc), _p(cfg.mds), 2, _p(inp), 2, 1, _p(out), 4) == (EINVAL, 0)
    assert (out == POISON).all()
    assert _rc(c, "ronk_poseidon_sponge_u64_host", 101, 3, 3, 2, 1, _p(cfg.rc), _p(cfg.mds), 4, _p(inp), 1, 1, _p(out), 4) == (EINVAL, 0)


# ---- streams and launch counts ---------------------------------------------------------------------------------------

def test_gated_non_blocking_stream():
    import torch
    from ronkathon_b200 import Context, ops
    from ronkathon_b200.hashes import PoseidonConfig
    rng = np.random.default_rng(19)
    orc = _cfg(rng, GL, 12, 7, 8, 22)
    cfg = PoseidonConfig(12, 7, 22, 8, orc.rc.tolist(), orc.mds.reshape(orc.width, orc.width).tolist())
    rows = _rand(rng, GL, 300 * 20).reshape(300, 20)
    want = po.sponge_rows(orc, 8, rows, 8)
    d = _dev(rows)
    s = torch.cuda.Stream()
    c = Context(0, s.cuda_stream)
    try:
        with torch.cuda.stream(s):
            ops.poseidon_sponge(c, d, 8, 8, cfg)            # warm: uploads the constants for this context
        s.synchronize()
        g = torch.zeros_like(d)
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            torch.cuda._sleep(100_000_000)
            g.copy_(d)
            got = ops.poseidon_sponge(c, g, 8, 8, cfg)
        s.synchronize()
        assert np.array_equal(got.cpu().numpy().view(np.uint64), want)
    finally:
        c.close()


def test_one_launch_per_call_whatever_the_batch():
    from ronkathon_b200 import ops
    from ronkathon_b200.hashes import PoseidonConfig
    c = ctx()
    rng = np.random.default_rng(23)
    orc = _cfg(rng, GL, 8, 7, 8, 22)
    cfg = PoseidonConfig(8, 7, 22, 8, orc.rc.tolist(), orc.mds.reshape(orc.width, orc.width).tolist())
    for batch in (1, 1000, 200_000):
        st = _dev(_rand(rng, GL, batch * 8)).view(batch, 8)
        ops.poseidon_permute_(c, st, cfg)                   # constants uploaded by the first call
        c.sync()
        before = c.launches
        ops.poseidon_permute_(c, st, cfg)
        out = ops.poseidon_sponge(c, st, 5, 4, cfg)
        c.sync()
        assert c.launches - before == 2 and out.shape == (batch, 5)


# ---- the Python typestate --------------------------------------------------------------------------------------------

def test_python_sponge_typestate_and_splits():
    from ronkathon_b200 import RonkPanic, ops
    from ronkathon_b200.field import PlutoBaseField
    from ronkathon_b200.hashes import PoseidonConfig, PoseidonSponge, SpongeStateError
    k = _kats()
    c = ctx()
    F = PlutoBaseField

    def sponge(rate=k["rate"]):
        return PoseidonSponge(k["width"], k["alpha"], k["num_p"], k["num_f"], rate, [F(v) for v in k["rc16"]],
                              [[F(v) for v in r] for r in k["mds16"]])

    orc = po.Config(101, 16, k["alpha"], k["num_p"], k["num_f"], k["rc16"], k["mds16"])
    cfg = PoseidonConfig(16, k["alpha"], k["num_p"], k["num_f"], k["rc16"], k["mds16"], field=F)
    rng = np.random.default_rng(29)
    for case in k["sponge_cases"]:
        size, times = case["absorb_size"], case.get("absorb_time", 1)
        sq, sq_times = case["squeeze_size"], case.get("squeeze_time", 1)
        words = [int(v) for v in rng.integers(0, 101, size)]
        s = sponge().start_absorbing()
        for _ in range(times):
            s.absorb([F(v) for v in words])
        s.start_squeezing()
        got = [v.value for _ in range(sq_times) for v in s.squeeze(sq)]
        want = po.sponge(orc, k["rate"], [words] * times, [sq] * sq_times)
        assert got == want, case
        row = _dev(np.array(words * times, np.uint64)).view(1, -1)
        assert _host(ops.poseidon_sponge(c, row, sq * sq_times, k["rate"], cfg)).reshape(-1).tolist() == want, case
    # abosrb_after_squeeze (tests/mod.rs:151-172): absorb on a squeezing sponge is the reference's Err
    s = sponge().start_absorbing()
    s.absorb([F(2)] * 5)
    s.start_squeezing()
    s.squeeze(2)
    with pytest.raises(SpongeStateError):
        s.absorb([F(2)] * 5)
    with pytest.raises(SpongeStateError):
        sponge().start_absorbing().squeeze(1)
    with pytest.raises(SpongeStateError):
        sponge().absorb([F(1)])
    assert sponge().start_absorbing().start_squeezing().squeeze(3) == [F(0)] * 3
    with pytest.raises(RonkPanic):
        sponge(rate=0)
    with pytest.raises(RonkPanic):
        sponge(rate=17)
