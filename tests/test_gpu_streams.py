"""The library off the legacy default stream: every context here enqueues on a torch stream, which is non-blocking.

The rest of the suite runs on stream 0, the legacy default stream, which synchronises implicitly with every blocking
stream; there a kernel, memset or copy on the wrong stream, a "synchronous" call that returns early or a missing
pipeline event goes unseen.  Here each case runs behind a gate on the context's own stream s:

  1. the inputs hold valid but wrong data (the real inputs reversed, or other seeds where reversing would not change
     the result) and the device is synchronised;
  2. on s: torch.cuda._sleep (a bounded spin of about 50 ms), the real inputs written, the outputs filled with a
     sentinel that is no residue of any test prime, the library call, clones of the results;
  3. right after an asynchronous call, s must still be busy, which shows that the call was enqueued behind the gate;
  4. after synchronising s the results must equal, bit for bit, those of the same call on the suite's context on
     stream 0 (which the rest of the suite pins to the oracle), and the oracle itself where that is cheap.

Work enqueued anywhere but on s runs during the sleep: it reads the wrong inputs, or the sentinel overwrites what it
wrote.  So a misplaced launch fails deterministically, without a race.  Nothing here loops to provoke a race.
An entry point that synchronises s before its kernels (division after reading the divisor's top word, the strided and
the fused cross-rank stage, the first call of a commit path on a context) opens the gate itself.  The commit tests warm
their context first; for the others, a second probe runs warm calls while the legacy default stream spins, and a
kernel of theirs enqueued there would run only after the spin.

The ops layer allocates its outputs on torch's current stream, so the tests call it inside `torch.cuda.stream(s)`
only; where the library's stream must differ from torch's, they use `Context.call` on buffers allocated beforehand.
"""
import ctypes as C
import os
import threading

import numpy as np
import pytest

import oracle
from gpu_util import BABYBEAR, GL, PBIG, ctx, dev, host, msm_inputs

pytestmark = pytest.mark.gpu

SLEEP_CYCLES = 100_000_000   # torch.cuda._sleep: about 50 ms at the H100 SXM's 1.98 GHz boost clock, longer below it
SENTINEL = -1                # 0xFFFFFFFFFFFFFFFF: not a canonical residue of any test prime
FAMILIES = {"goldilocks": (GL, 7), "babybear": (BABYBEAR, 31), "pbig": (PBIG, 3)}


def _ptr(t):
    return t.data_ptr()


def _context(stream, env=None):
    """A fresh Context on `stream` (a torch stream), with the tuning switches of `env` read at its creation."""
    from ronkathon_b200 import Context
    env = env or {}
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return Context(0, stream.cuda_stream)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _res(n, seed, p=GL):
    """n canonical residues mod p on the device (splitmix, generated on the suite's context)."""
    from ronkathon_b200 import ops
    return ops.splitmix_fill(ctx(), n, seed, p)


def _nonzero(t):
    """t with every zero replaced by 1: inputs for inverse and division."""
    import torch
    return torch.where(t == 0, torch.ones_like(t), t)


def _divisor(n, seed, p=GL):
    b = oracle.splitmix(p, seed, n)
    b[-1] = b[-1] % (p - 1) + 1   # nonzero top word
    return dev(b)


def _wrong(t):
    """Valid but wrong data of t's shape and type: its rows reversed."""
    import torch
    w = t.flip(0).contiguous()
    assert not torch.equal(w, t), "a palindromic input cannot show a misplaced read"
    return w


def _outputs(n_outs):
    import torch
    return [torch.empty(n, dtype=dt, device="cuda") for n, dt in n_outs]


def _warm_torch(ins, outs):
    """The torch copy and fill kernels of the gate, launched once before it: the first launch of a kernel in the
    process loads its module, which waits for the whole device."""
    for t in ins:
        t.clone().copy_(t)
    for o in outs:
        o.fill_(SENTINEL)


def _reference(ins, n_outs, call):
    """The same call on the suite's context (stream 0) with the real inputs: in-place buffers, then outputs."""
    c0 = ctx()
    bufs = [t.clone() for t in ins]
    outs = _outputs(n_outs)
    ret = call(c0, bufs, outs)
    c0.sync()
    return bufs + outs, ret


def _gated(s, c, ins, n_outs, call, asynchronous, wrong=None, warm=False):
    """call(c, bufs, outs) on stream s behind the gate; returns the clones taken on s after it and its return value.
    `wrong`: the valid but wrong inputs (default: the real ones reversed).  `warm`: run the call once on the wrong
    inputs first, for entry points whose first use on a context synchronises its stream before their kernels."""
    import torch
    bufs = [_wrong(t) for t in ins] if wrong is None else [w.clone() for w in wrong]
    outs = _outputs(n_outs)
    if warm:
        with torch.cuda.stream(s):
            call(c, [b.clone() for b in bufs], _outputs(n_outs))
        s.synchronize()
    _warm_torch(ins, outs)
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
        for b, t in zip(bufs, ins):
            b.copy_(t)
        for o in outs:
            o.fill_(SENTINEL)
        ret = call(c, bufs, outs)
        if asynchronous:
            assert not s.query(), "s finished before the call returned: the gate was too short, or the call waited"
        got = [t.clone() for t in bufs + outs]
    s.synchronize()
    return got, ret


def _through_gate(ins, n_outs, call, asynchronous=True, env=None, wrong=None, warm=False):
    """Runs one case on a fresh context behind the gate and checks it against the reference; returns the results.  The
    reference runs first: the first launch of a kernel in the process loads its module, which waits for the device."""
    import torch
    want, wret = _reference(ins, n_outs, call)
    s = torch.cuda.Stream()
    c = _context(s, env)
    try:
        got, ret = _gated(s, c, ins, n_outs, call, asynchronous, wrong, warm)
    finally:
        c.close()
    for i, (x, y) in enumerate(zip(got, want)):
        assert x.shape == y.shape and torch.equal(x, y), f"result {i} differs from the default-stream context"
    assert ret == wret
    return got, ret


# ---- 1. every entry point behind the gate -----------------------------------------------------------------------------
NTT_SHAPES = [(10, 7), (16, 1), (16, 3), (18, 1), (18, 17), (20, 1), (22, 1), (24, 1), (25, 1)]


@pytest.mark.parametrize("log_n,batch", NTT_SHAPES, ids=[f"2^{l}x{b}" for l, b in NTT_SHAPES])
@pytest.mark.parametrize("family", list(FAMILIES))
def test_transforms_behind_the_gate(family, log_n, batch):
    """Forward, fused-multiply and inverse transforms on a non-blocking stream: single tile (2^10 × 7), the 2^16
    cluster kernel (batch 1) and tiles (batch 3), the Montgomery two-pass and split 2^18 (also × 17), ntt3c at 2^20 and
    the three-pass 2^24 (both with programmatic dependent launch), the 2^22 mid path and the split 2^25."""
    p, g = FAMILIES[family]
    n = batch << log_n
    ins = [_res(n, 11, p), _res(n, 12, p), _res(n, 13, p), _res(n, 14, p)]

    def call(c, b, o):
        x, y, m, z = b
        c.call("ronk_ntt_u64", p, g, _ptr(x), log_n, batch, 0)
        c.call("ronk_ntt_mul_u64", p, g, _ptr(y), _ptr(m), log_n, batch)
        c.call("ronk_ntt_u64", p, g, _ptr(z), log_n, batch, 1)

    got, _ = _through_gate(ins, [], call)
    if log_n == 10:
        from ronkathon_b200 import ops
        a, z = ops.to_host(ins[0]), ops.to_host(ins[3])
        x, zi = ops.to_host(got[0]), ops.to_host(got[3])
        for k in range(batch):
            sl = slice(k << log_n, (k + 1) << log_n)
            assert np.array_equal(x[sl], oracle.ntt_fast(p, a[sl], g=g)), k
            assert np.array_equal(zi[sl], oracle.ntt_fast(p, z[sl], inverse=True, g=g)), k


@pytest.mark.parametrize("da,db", [(40, 30), ((1 << 20) + 5, (1 << 20) - 100)], ids=["schoolbook", "ntt_2^21"])
def test_poly_mul_behind_the_gate(da, db):
    import torch
    ins = [_res(da, 21), _res(db, 22)]

    def call(c, b, o):
        c.call("ronk_poly_mul_u64", GL, 7, _ptr(b[0]), da, _ptr(b[1]), db, _ptr(o[0]))

    got, _ = _through_gate(ins, [(da + db - 1, torch.int64)], call)
    if da < 100:
        from ronkathon_b200 import ops
        assert np.array_equal(ops.to_host(got[2]), oracle.poly_mul(GL, ops.to_host(ins[0]), ops.to_host(ins[1])))


DIVREM = {
    "newton": lambda: (_res(1 << 18, 31), _divisor((1 << 17) + 1, 32), 7),
    "linear": lambda: (_res(5000, 33), dev(np.array([GL - 5, 1], np.uint64)), 7),
    "da_lt_db": lambda: (_res(5, 34), _divisor(9, 35), 7),
    "literal": lambda: (_res(600, 36), _divisor(70, 37), 0),   # g = 0 keeps the literal kernel
}


@pytest.mark.parametrize("path", list(DIVREM))
def test_divrem_behind_the_gate(path):
    """ronk_poly_divrem_u64 on each path.  It reads the divisor's top word on the host to choose one and synchronises
    s for it, so the gate checks that read (it must see the real divisor); the kernels that follow run after the gate
    has opened, and the legacy-stream test below checks where they are enqueued."""
    import torch
    a, b, g = DIVREM[path]()
    da, db = a.numel(), b.numel()

    def call(c, bf, o):
        c.call("ronk_poly_divrem_u64", GL, g, _ptr(bf[0]), da, _ptr(bf[1]), db, _ptr(o[0]), _ptr(o[1]))

    got, _ = _through_gate([a, b], [(da, torch.int64), (da, torch.int64)], call, asynchronous=False)
    if da <= 5000:
        from ronkathon_b200 import ops
        q, r = oracle.poly_divrem(GL, ops.to_host(a), ops.to_host(b))
        assert np.array_equal(ops.to_host(got[2]), q) and np.array_equal(ops.to_host(got[3]), r)


def test_div_linear_eval_and_dft_behind_the_gate():
    import torch
    d, m, nd = (1 << 20) + 3, (1 << 16) + 1, 4080   # 4080 = 2^4·3·5·17 divides p - 1
    b0, b1 = 0x123456789 % GL, 0xABCDEF % GL
    ins = [_res(d, 41), _res(1000, 42), _res(m, 43), _res(nd, 44)]

    def call(c, b, o):
        c.call("ronk_poly_div_linear_u64", GL, _ptr(b[0]), d, b0, b1, _ptr(o[0]), _ptr(o[1]))
        c.call("ronk_poly_eval_u64", GL, _ptr(b[1]), 1000, _ptr(b[2]), m, _ptr(o[2]))
        c.call("ronk_dft_u64", GL, 7, _ptr(b[3]), nd, _ptr(o[3]))

    got, _ = _through_gate(ins, [(d, torch.int64), (1, torch.int64), (m, torch.int64), (nd, torch.int64)], call)
    from ronkathon_b200 import ops
    assert np.array_equal(ops.to_host(got[7]), oracle.dft(GL, ops.to_host(ins[3])))
    xs, cs, ev = ops.to_host(ins[2]), ops.to_host(ins[1]), ops.to_host(got[6])
    for i in (0, 1, m - 1):
        assert int(ev[i]) == oracle.poly_eval_horner(GL, cs, int(xs[i])), i


@pytest.mark.parametrize("family", list(FAMILIES))
def test_field_ops_powers_and_splitmix_behind_the_gate(family):
    import torch
    p, g = FAMILIES[family]
    n = (1 << 20) + 3
    ins = [_res(n, 51, p), _res(n, 52, p)]
    e = 0xFEDCBA9876543210
    w = oracle.root_of_unity(p, 1 << 16, g)

    def call(c, b, o):
        c.call("ronk_field_add_u64", p, _ptr(b[0]), _ptr(b[1]), _ptr(o[0]), n)
        c.call("ronk_field_mul_u64", p, _ptr(b[0]), _ptr(b[1]), _ptr(o[1]), n)
        c.call("ronk_field_pow_u64", p, _ptr(b[0]), e, _ptr(o[2]), n)
        c.call("ronk_field_neg_u64", p, _ptr(b[1]), _ptr(o[3]), n)
        c.call("ronk_field_powers_u64", p, w, 5, _ptr(o[4]), n)
        c.call("ronk_splitmix_fill_u64", p, 4242, _ptr(o[5]), n)

    got, _ = _through_gate(ins, [(n, torch.int64)] * 6, call)
    from ronkathon_b200 import ops
    a, b = ops.to_host(ins[0]), ops.to_host(ins[1])
    for i in (0, 1, n - 1):
        assert int(ops.to_host(got[2])[i]) == oracle.add(p, int(a[i]), int(b[i]))
        assert int(ops.to_host(got[3])[i]) == oracle.mul(p, int(a[i]), int(b[i]))
        assert int(ops.to_host(got[4])[i]) == oracle.pow_(p, int(a[i]), e)
    assert np.array_equal(ops.to_host(got[7]), oracle.splitmix(p, 4242, n))


def test_strided_small_behind_the_gate():
    """It stages its table from the stack and synchronises s before its kernel, so the gate opens inside the call and
    this checks only the result; the legacy-stream test below checks where the kernel is enqueued."""
    log_g, stride = 3, (1 << 16) + 1
    ins = [_res(stride << log_g, 61)]

    def call(c, b, o):
        c.call("ronk_ntt_strided_small_u64", GL, 7, _ptr(b[0]), log_g, stride, stride, 0)
        c.call("ronk_ntt_strided_small_u64", GL, 7, _ptr(b[0]), log_g, stride, stride - 3, 1)

    _through_gate(ins, [], call, asynchronous=False)


@pytest.mark.parametrize("path,env", [("coord", {}), ("hist", {"RONK_MSM_COORD": "0"}),
                                      ("buckets", {"RONK_MSM_COORD": "0", "RONK_MSM_HIST": "0"})])
def test_msm_behind_the_gate(path, env):
    """kzg::commit on all three paths (msm_hist_finish with programmatic dependent launch); synchronous, with a host
    output.  The wrong inputs come from other seeds: reversing points and scalars together would only reorder the
    terms of the same sum.  The context is warmed first, because the first call of the coordinate and histogram paths
    builds its tables and synchronises the stream before any commit kernel is enqueued."""
    import torch
    from ronkathon_b200 import ops
    n = (1 << 16) + 3
    pts, sc = msm_inputs(n, 71, 72)
    wpts, wsc = msm_inputs(n, 73, 74)
    assert oracle.commit(wsc, wpts, fast=True) != oracle.commit(sc, pts, fast=True)
    ins = [torch.from_numpy(pts).cuda(), torch.from_numpy(sc).cuda()]
    wrong = [torch.from_numpy(wpts).cuda(), torch.from_numpy(wsc).cuda()]

    def call(c, b, o):
        return ops.msm(c, b[0], b[1])

    _, ret = _through_gate(ins, [], call, asynchronous=False, env=env, wrong=wrong, warm=True)
    assert ret == oracle.commit(sc, pts, fast=True)


@pytest.mark.parametrize("flavour", [0, 1], ids=["nccl_layout", "fused"])
def test_dist_virtual_behind_the_gate(flavour):
    log_n, batch, log_g = 20, 2, 2
    ins = [_res(batch << log_n, 81)]

    def call(c, b, o):
        c.call("ronk_ntt_u64_dist_virtual", GL, 7, _ptr(b[0]), log_n, batch, log_g, flavour)

    _through_gate(ins, [], call, asynchronous=False)


def test_cross_rank_fused_behind_the_gate():
    """G = 4: every rank's output from the same four peer buffers.  Like the strided stage it synchronises s before
    its kernels, so this checks the result; the legacy-stream test below checks where the kernels are enqueued."""
    import torch
    log_g, log_n = 2, 20
    G, m = 1 << log_g, 1 << (log_n - log_g)
    ins = [_res(m, 90 + r) for r in range(G)]

    def call(c, b, o):
        peers = (C.c_void_p * G)(*[_ptr(y) for y in b])
        for r in range(G):
            c.call("ronk_ntt_cross_rank_fused_u64", GL, 7, C.cast(peers, C.c_void_p), log_g, r, log_n, _ptr(o[r]))

    _through_gate(ins, [(m, torch.int64)] * G, call, asynchronous=False)


# ---- 2. the documented-synchronous entry points ---------------------------------------------------------------------
def test_synchronous_calls_are_complete_on_return():
    """field_inv, field_div, Newton division at 2^22 / 2^21 + 1 (milliseconds of work follow its read of the divisor's
    top word), msm and memcpy_h2d: right after each returns, an unrelated stream copies the outputs with no wait."""
    import torch
    from ronkathon_b200 import RonkPanic, ops
    s, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    c = _context(s)
    n = (1 << 20) + 3
    da, db = 1 << 22, (1 << 21) + 1
    h = oracle.splitmix(GL, 109, n)
    pts, sc = msm_inputs(1 << 20, 107, 108)
    wpts, wsc = msm_inputs(1 << 20, 111, 112)   # other seeds: reversed inputs would give the same commitment
    assert oracle.commit(wsc, wpts, fast=True) != oracle.commit(sc, pts, fast=True)
    wrong = {"msm": [torch.from_numpy(wpts).cuda(), torch.from_numpy(wsc).cuda()]}
    cases = {
        "inv": ([_nonzero(_res(n, 101))], [(n, torch.int64)],
                lambda c, b, o: c.call("ronk_field_inv_u64", GL, _ptr(b[0]), _ptr(o[0]), n)),
        "div": ([_res(n, 102), _nonzero(_res(n, 103))], [(n, torch.int64)],
                lambda c, b, o: c.call("ronk_field_div_u64", GL, _ptr(b[0]), _ptr(b[1]), _ptr(o[0]), n)),
        "divrem": ([_res(da, 104), _divisor(db, 105)], [(da, torch.int64), (da, torch.int64)],
                   lambda c, b, o: c.call("ronk_poly_divrem_u64", GL, 7, _ptr(b[0]), da, _ptr(b[1]), db, _ptr(o[0]),
                                          _ptr(o[1]))),
        "msm": ([torch.from_numpy(pts).cuda(), torch.from_numpy(sc).cuda()], [],
                lambda c, b, o: ops.msm(c, b[0], b[1])),
        "h2d": ([], [(n, torch.int64)],
                lambda c, b, o: c.call("ronk_memcpy_h2d", _ptr(o[0]), h.ctypes.data_as(C.c_void_p), n * 8)),
    }
    try:
        for name, (ins, n_outs, call) in cases.items():
            want, wret = _reference(ins, n_outs, call)
            bufs = [w.clone() for w in wrong[name]] if name in wrong else [_wrong(t) for t in ins]
            outs = _outputs(n_outs)
            with torch.cuda.stream(s):   # plans and workspaces first built on other data: no waits inside the call
                call(c, [b.clone() for b in bufs], _outputs(n_outs))
            s.synchronize()
            _warm_torch(ins, outs)
            torch.cuda.synchronize()
            with torch.cuda.stream(s):
                torch.cuda._sleep(SLEEP_CYCLES)
                for b, t in zip(bufs, ins):
                    b.copy_(t)
                for o in outs:
                    o.fill_(SENTINEL)
                ret = call(c, bufs, outs)
            with torch.cuda.stream(s2):
                got = [o.clone() for o in outs]
            s2.synchronize()
            s.synchronize()
            for i, (x, y) in enumerate(zip(got, want[len(ins):])):
                assert torch.equal(x, y), (name, i)
            assert ret == wret, name
            if name == "msm":
                assert ret == oracle.commit(sc, pts, fast=True)
            if name == "h2d":
                assert np.array_equal(ops.to_host(got[0]), h)
        # the flag path on s: a zero input raises, and the next call is right
        a = _nonzero(_res(n, 110))
        a[-1] = 0
        out = torch.empty_like(a)
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            torch.cuda._sleep(SLEEP_CYCLES)
            with pytest.raises(RonkPanic):
                c.call("ronk_field_inv_u64", GL, _ptr(a), _ptr(out), n)
            a[-1] = 5
            c.call("ronk_field_inv_u64", GL, _ptr(a), _ptr(out), n)
            got = out.clone()
        s.synchronize()
        want, _ = _reference([a], [(n, torch.int64)], cases["inv"][2])
        assert torch.equal(got, want[1])
        assert int(ops.to_host(got)[-1]) == oracle.inverse(GL, 5)
    finally:
        c.close()


def test_legacy_stream_work_neither_delays_nor_corrupts_a_context_on_its_own_stream():
    """With the legacy default stream spinning, warm calls on a context on a non-blocking stream finish on their own:
    nothing the library does for them may be enqueued on, or wait for, the legacy stream.  This is the probe for the
    kernels of entry points that synchronise their stream before launching (every division path after its top-word
    read, the strided and the fused cross-rank stage), which the gate cannot reach: a kernel of theirs on the legacy
    stream would run after the spin, so the results read when s is done would be wrong."""
    import torch
    s = torch.cuda.Stream()
    c = _context(s)
    da, db, n = 1 << 18, (1 << 17) + 1, 1 << 20
    log_g, stride, log_n = 3, (1 << 16) + 1, 20                  # strided stage; G = 4 fused stage at 2^20
    m = 1 << (log_n - 2)
    divs = [(_res(5000, 126), dev(np.array([GL - 5, 1], np.uint64)), 7),   # linear
            (_res(5, 127), _divisor(9, 128), 7),                            # da < db
            (_res(600, 129), _divisor(70, 130), 0)]                         # literal (g = 0)
    ins = [_res(da, 121), _divisor(db, 122), _res(n, 123), _res(n >> 1, 124), _nonzero(_res(n, 125)),
           *[t for a, b, _ in divs for t in (a, b)], _res(stride << log_g, 131), *[_res(m, 132 + r) for r in range(4)]]
    n_outs = [(da, torch.int64), (da, torch.int64), (n + (n >> 1) - 1, torch.int64), (n, torch.int64),
              *[(a.numel(), torch.int64) for a, _, _ in divs for _ in range(2)], *[(m, torch.int64)] * 4]

    def call(c, b, o):
        c.call("ronk_poly_divrem_u64", GL, 7, _ptr(b[0]), da, _ptr(b[1]), db, _ptr(o[0]), _ptr(o[1]))
        c.call("ronk_ntt_u64", GL, 7, _ptr(b[2]), 20, 1, 0)
        c.call("ronk_poly_mul_u64", GL, 7, _ptr(b[2]), n, _ptr(b[3]), n >> 1, _ptr(o[2]))
        c.call("ronk_field_inv_u64", GL, _ptr(b[4]), _ptr(o[3]), n)
        for k, (a, dv, g) in enumerate(divs):
            x, y, q, r = b[5 + 2 * k], b[6 + 2 * k], o[4 + 2 * k], o[5 + 2 * k]
            c.call("ronk_poly_divrem_u64", GL, g, _ptr(x), a.numel(), _ptr(y), dv.numel(), _ptr(q), _ptr(r))
        c.call("ronk_ntt_strided_small_u64", GL, 7, _ptr(b[11]), log_g, stride, stride, 0)
        peers = (C.c_void_p * 4)(*[_ptr(y) for y in b[12:16]])
        for r in range(4):
            c.call("ronk_ntt_cross_rank_fused_u64", GL, 7, C.cast(peers, C.c_void_p), 2, r, log_n, _ptr(o[10 + r]))

    try:
        want, _ = _reference(ins, n_outs, call)
        with torch.cuda.stream(s):   # first use: plans, tables and workspaces, on other data (another top word)
            call(c, [_wrong(t) for t in ins], _outputs(n_outs))
        s.synchronize()
        bufs, outs = [t.clone() for t in ins], _outputs(n_outs)
        torch.cuda.synchronize()
        legacy = torch.cuda.default_stream()
        assert legacy.cuda_stream == 0
        with torch.cuda.stream(legacy):
            torch.cuda._sleep(2 * SLEEP_CYCLES)
        with torch.cuda.stream(s):
            call(c, bufs, outs)
        s.synchronize()
        assert not legacy.query(), "a call on the context's own stream waited for the legacy default stream"
        torch.cuda.synchronize()
        for i, (x, y) in enumerate(zip(bufs + outs, want)):
            assert torch.equal(x, y), i
    finally:
        c.close()


# ---- 3. concurrent contexts ---------------------------------------------------------------------------------------------
def _mixed_inputs(seed):
    import torch
    n20, n24, nd = 1 << 20, 1 << 24, 4080
    pts, sc = msm_inputs(n20, seed, seed + 1)
    return {"x24": _res(n24, seed + 2), "y24": _res(n24, seed + 3), "bb20": _res(n20, seed + 4, BABYBEAR),
            "ma": _res(n20 >> 1, seed + 5), "mb": _res((n20 >> 1) + 1, seed + 6),
            "da": _res(n20, seed + 7), "db": _divisor((n20 >> 1) + 1, seed + 8),
            "pts": torch.from_numpy(pts).cuda(), "sc": torch.from_numpy(sc).cuda(),
            "inv": _nonzero(_res(n20, seed + 9)), "dft": _res(nd, seed + 10)}


def _mixed_run(c, x):
    """2^24 forward and inverse, a Montgomery 2^20 transform, poly_mul at 2^20, Newton division, msm of 2^20 terms,
    field_inv and dft, all on c's stream, which is torch's current stream; no host synchronisation in between."""
    import torch
    from ronkathon_b200 import ops
    r = {k: x[k].clone() for k in ("x24", "y24", "bb20")}
    ops.ntt_(c, r["x24"], 24)
    ops.ntt_(c, r["y24"], 24, inverse=True)
    ops.ntt_(c, r["bb20"], 20, p=BABYBEAR, g=31)
    r["mul"] = ops.poly_mul(c, x["ma"], x["mb"])
    r["q"], r["r"] = ops.poly_divrem(c, x["da"], x["db"])
    r["msm"] = ops.msm(c, x["pts"], x["sc"])
    r["inv"] = torch.empty_like(x["inv"])
    c.call("ronk_field_inv_u64", GL, _ptr(x["inv"]), _ptr(r["inv"]), x["inv"].numel())
    r["dft"] = torch.empty_like(x["dft"])
    c.call("ronk_dft_u64", GL, 7, _ptr(x["dft"]), x["dft"].numel(), _ptr(r["dft"]))
    return r


def _same(got, want):
    import torch
    assert got.keys() == want.keys()
    for k in want:
        ok = torch.equal(got[k], want[k]) if hasattr(want[k], "data_ptr") else got[k] == want[k]
        assert ok, k


def test_four_threads_with_their_own_contexts_and_streams():
    """Four host threads, each with a fresh context (plans, tables, cluster probe and shared-memory attributes all first
    built concurrently), its own stream and its own seeds, run the mixed list twice; everything equals the serial
    results of the suite's context."""
    import torch
    T = 4
    inputs = [_mixed_inputs(1000 + 100 * t) for t in range(T)]
    want = []
    for x in inputs:
        want.append(_mixed_run(ctx(), x))
        ctx().sync()
    torch.cuda.synchronize()
    results, errors = [None] * T, []
    start = threading.Barrier(T, timeout=120)

    def worker(t):
        try:
            s = torch.cuda.Stream()
            c = _context(s)
            start.wait()
            with torch.cuda.stream(s):
                runs = [_mixed_run(c, inputs[t]) for _ in range(2)]
            s.synchronize()
            c.close()
            results[t] = runs
        except BaseException as e:   # re-raised in the main thread
            errors.append((t, e))
            start.abort()            # the others stop waiting for this thread

    threads = [threading.Thread(target=worker, args=(t,)) for t in range(T)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    for t in range(T):
        for run in results[t]:
            _same(run, want[t])


def test_two_contexts_on_one_thread_hand_over_through_events():
    """Two contexts on two streams, interleaved on one thread; data passes from one to the other only through a torch
    Event and wait_event.  x → NTT on A (behind the gate) → inverse on B → NTT ⊙ m on A."""
    import torch
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    ca, cb = _context(sa), _context(sb)
    x0, m = _res(1 << 20, 131), _res(1 << 20, 132)
    want = x0.clone()
    ctx().call("ronk_ntt_mul_u64", GL, 7, _ptr(want), _ptr(m), 20, 1)
    ctx().sync()
    x = _wrong(x0)
    torch.cuda.synchronize()
    try:
        def hand(src, dst):
            ev = torch.cuda.Event()
            ev.record(src)
            dst.wait_event(ev)

        with torch.cuda.stream(sa):
            torch.cuda._sleep(SLEEP_CYCLES)
            x.copy_(x0)
            ca.call("ronk_ntt_u64", GL, 7, _ptr(x), 20, 1, 0)
        hand(sa, sb)
        with torch.cuda.stream(sb):
            cb.call("ronk_ntt_u64", GL, 7, _ptr(x), 20, 1, 1)
            assert not sb.query(), "B ran ahead of A's gate"
            back = x.clone()
        hand(sb, sa)
        with torch.cuda.stream(sa):
            ca.call("ronk_ntt_mul_u64", GL, 7, _ptr(x), _ptr(m), 20, 1)
            got = x.clone()
        sa.synchronize()
        assert torch.equal(back, x0)
        assert torch.equal(got, want)
    finally:
        sa.synchronize()
        ca.close()
        cb.close()


# ---- 4. ronk_ctx_set_stream ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("plan", ["built_before", "built_on_a"])
def test_set_stream_orders_the_old_stream_before_the_new(plan):
    """A forward transform enqueued on the gated stream A, set_stream(B), the inverse of the same buffer on B: the
    buffer comes back as the input.  Either with the plan built beforehand or first built by the call on A."""
    import torch
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    c = _context(sa)
    p, g, log_n, batch = (GL, 7, 20, 1) if plan == "built_before" else (BABYBEAR, 31, 18, 3)
    x0 = _res(batch << log_n, 141, p)
    x = _wrong(x0)
    try:
        if plan == "built_before":
            with torch.cuda.stream(sa):
                c.call("ronk_ntt_u64", p, g, _ptr(x.clone()), log_n, batch, 0)
        torch.cuda.synchronize()
        with torch.cuda.stream(sa):
            torch.cuda._sleep(SLEEP_CYCLES)
            x.copy_(x0)
            c.call("ronk_ntt_u64", p, g, _ptr(x), log_n, batch, 0)
            assert not sa.query(), "the gate was too short"
        c.set_stream(sb.cuda_stream)
        with torch.cuda.stream(sb):
            c.call("ronk_ntt_u64", p, g, _ptr(x), log_n, batch, 1)
            got = x.clone()
        sb.synchronize()
        assert torch.equal(got, x0)
    finally:
        c.close()


# ---- 5. the host pipeline over all three slots ---------------------------------------------------------------------------
@pytest.mark.parametrize("memory", ["pinned", "pageable"])
def test_host_pipeline_all_three_slots(memory):
    """Submits over slots 0, 1, 2 in rotation with per-slot sizes growing 2^12 → 2^18 → 2^22 (every slot buffer is
    reallocated twice), batches, inverse transforms and Montgomery primes, behind a gate on the context's stream so the
    uploads run ahead of compute; a 2^24 device transform that grows the workspace sits between a submit and its
    wait.  Then the argument errors; after a failed submit, a wait on its slot succeeds, its host buffer is as it was,
    and the next submit on that slot is right."""
    import torch
    from ronkathon_b200 import RonkError, RonkPanic, _lib
    s = torch.cuda.Stream()
    c = _context(s)
    fams = [(GL, 7), (BABYBEAR, 31), (PBIG, 3)]
    batches = {12: 6, 18: 3, 22: 1}
    jobs = []
    for i in range(9):
        slot, log_n = i % 3, (12, 18, 22)[i // 3]
        p, g = fams[(slot + i // 3) % 3]
        jobs.append((slot, p, g, log_n, batches[log_n], i % 2))

    def host_buf(a):
        if memory == "pinned":
            t = torch.from_numpy(a.copy().view(np.int64)).pin_memory()
            return t, t.data_ptr(), lambda: t.numpy().view(np.uint64)
        h = a.copy()
        return h, h.ctypes.data, lambda: h

    def expect(a, p, g, log_n, batch, inv):
        d = dev(a)
        ctx().call("ronk_ntt_u64", p, g, _ptr(d), log_n, batch, inv)
        return host(d)

    data = [oracle.splitmix(p, 150 + i, batch << log_n) for i, (_, p, _, log_n, batch, _) in enumerate(jobs)]
    want = [expect(a, *j[1:]) for a, j in zip(data, jobs)]
    bufs = [host_buf(a) for a in data]
    z0 = _res(1 << 24, 160)
    z_want = z0.clone()
    ctx().call("ronk_ntt_u64", GL, 7, _ptr(z_want), 24, 1, 0)
    z = z0.clone()
    torch.cuda.synchronize()
    try:
        with torch.cuda.stream(s):
            torch.cuda._sleep(SLEEP_CYCLES)
        for i, (slot, p, g, log_n, batch, inv) in enumerate(jobs):
            c.call("ronk_ntt_u64_host_submit", p, g, bufs[i][1], log_n, batch, inv, slot)
            if i == 4:
                c.call("ronk_ntt_u64", GL, 7, _ptr(z), 24, 1, 0)
            if i >= 2:
                c.call("ronk_ntt_u64_host_wait", jobs[i - 2][0])
        for slot in range(3):
            c.call("ronk_ntt_u64_host_wait", slot)
        for i, b in enumerate(bufs):
            assert np.array_equal(b[2](), want[i]), jobs[i]
        s.synchronize()
        assert torch.equal(z, z_want)
        # errors
        a = oracle.splitmix(GL, 170, 1 << 12)
        hb = host_buf(a)
        for bad in (-1, 3):
            with pytest.raises(RonkPanic):
                c.call("ronk_ntt_u64_host_submit", GL, 7, hb[1], 12, 1, 0, bad)
            with pytest.raises(RonkPanic):
                c.call("ronk_ntt_u64_host_wait", bad)
        with pytest.raises(RonkError) as e:
            c.call("ronk_ntt_u64_host_submit", GL, 7, hb[1], 27, 1, 0, 1)
        assert e.value.code == _lib.EUNSUPPORTED
        with pytest.raises(RonkPanic):
            c.call("ronk_ntt_u64_host_submit", 100, 3, hb[1], 12, 1, 0, 1)
        c.call("ronk_ntt_u64_host_wait", 1)
        assert np.array_equal(hb[2](), a)
        c.call("ronk_ntt_u64_host_submit", GL, 7, hb[1], 12, 1, 0, 1)
        c.call("ronk_ntt_u64_host_wait", 1)
        assert np.array_equal(hb[2](), oracle.ntt_fast(GL, a))
    finally:
        s.synchronize()
        c.close()
