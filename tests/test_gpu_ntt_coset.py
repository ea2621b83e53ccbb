"""Coset transforms (ronk_ntt_coset_u64) and the low-degree extension (ronk_poly_lde_u64) on the device.

The coset factor s^j rides on the load of a transform's first pass (forward) or the store of its last (inverse), in
instantiations of the tile kernels and of the 256-point-tile passes that nothing else takes.  Every kernel family meets
its size edges here, with shifts whose answer is known exactly:

* s = ω_n^t: the plain transform rotated by t (X_s[k] = A(ω^(k + t))), at every size;
* s = ω_2n: the odd outputs of the plain 2n-point transform of the zero-padded row;
* s = 1, g, p - 1 and a seeded element: the plain transform of a ⊙ s^j, the factor built by ronk_field_powers_u64 and
  ronk_field_mul_u64, against the oracle's transforms up to 2^12 and Horner's rule at five points at every size;
* round trips in both orders, launch records pinned per family, other tuning contexts, guarded buffers, refused calls,
  the host-pointer twins and a gated non-blocking stream."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle
from gpu_util import GL, MONT_PRIMES, ctx, dev, host

pytestmark = pytest.mark.gpu

POISON = -1   # 0xFFFFFFFFFFFFFFFF: no canonical residue of any test prime
FIELDS = {"gl": (GL, 7, 32), **MONT_PRIMES}
EDGE_SIZES = [1, 4, 12, 13, 14, 20, 21, 24, 26]   # the size edges of the kernel families
TABLE_BUILDS = {"pow_table", "tw2d_gather", "interpass_table", "ntt3_t1", "ntt3_t2"}   # first use of a plan


def sizes(name):
    p, g, adicity = FIELDS[name]
    if name == "gl":
        return list(range(1, 27))
    return sorted({k for k in EDGE_SIZES if k <= adicity} | {min(adicity, 26)})


GRID = [(name, k) for name in FIELDS for k in sizes(name)]


_ctx = None


@pytest.fixture(scope="module", autouse=True)
def _module_context():
    """The module's calls run on a context of its own, destroyed when the module is done: they build plans for every
    test prime at every size (hundreds of small device tables) and grow the scratch to 2^26-point workspaces, and
    none of that should stay on the suite's shared context, where every later test would carry it.  The several GiB
    the 2^26-point cases leave in torch's caching allocator go back to the device as well."""
    global _ctx
    import torch
    from ronkathon_b200 import Context
    ctx()   # binds the device and the suite's default context first
    _ctx = Context(0, torch.cuda.current_stream().cuda_stream)
    try:
        yield
    finally:
        _ctx.close()
        _ctx = None
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


def _c():
    return _ctx


def fill(n, seed, p):
    from ronkathon_b200 import ops
    return ops.splitmix_fill(_c(), n, seed, p)


def ntt(t, log_n, batch, p, g, inverse=False):
    from ronkathon_b200 import ops
    return ops.ntt_(_c(), t, log_n, batch=batch, inverse=inverse, p=p, g=g)


def coset(t, log_n, s, batch, p, g, inverse=False):
    from ronkathon_b200 import ops
    return ops.ntt_coset_(_c(), t, log_n, s, batch=batch, inverse=inverse, p=p, g=g)


def root(p, g, log_n):
    return pow(g, (p - 1) >> log_n, p)


def three_call_reference(a, log_n, s, batch, p, g):
    """ronk_ntt_u64 of a ⊙ s^j, the factor built by ronk_field_powers_u64 and applied by ronk_field_mul_u64."""
    import torch
    n = 1 << log_n
    pw = torch.empty(n, dtype=torch.int64, device="cuda")
    _c().call("ronk_field_powers_u64", p, s, 1, pw.data_ptr(), n)
    factor, b = pw.repeat(batch), torch.empty_like(a)
    _c().call("ronk_field_mul_u64", p, a.data_ptr(), factor.data_ptr(), b.data_ptr(), batch * n)
    return ntt(b, log_n, batch, p, g)


def batch_for(name, log_n):
    """Batches above 1 for every family: small sizes and the three-pass Goldilocks sizes, within 2^23 words."""
    return 3 if log_n <= 21 else (2 if name == "gl" and log_n <= 22 else 1)


# ---- exact words ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,log_n", GRID, ids=[f"{n}-2^{k}" for n, k in GRID])
def test_coset_words(name, log_n):
    import torch
    p, g, _ = FIELDS[name]
    n = 1 << log_n
    for batch in sorted({1, batch_for(name, log_n)}):
        a = fill(batch * n, 1000 * log_n + batch, p)
        X = ntt(a.clone(), log_n, batch, p, g)
        rows = X.view(batch, n)
        # s = ω_n^t: the plain transform rotated by t
        w = root(p, g, log_n)
        for t in sorted({1, n // 2, n - 1, 3 % n}):
            got = coset(a.clone(), log_n, pow(w, t, p), batch, p, g)
            assert torch.equal(got.view(batch, n), torch.roll(rows, -t, 1)), f"ω^{t}"
            back = coset(torch.roll(rows, -t, 1).contiguous().view(-1), log_n, pow(w, t, p), batch, p, g, inverse=True)
            assert torch.equal(back, a), f"inverse at ω^{t}"
        # s = 1: exactly the plain words, both directions
        assert torch.equal(coset(a.clone(), log_n, 1, batch, p, g), X)
        assert torch.equal(coset(X.clone(), log_n, 1, batch, p, g, inverse=True), ntt(X.clone(), log_n, batch, p, g, True))
        # general shifts against the three-call route, with round trips in both orders
        for s in (g, p - 1, int(oracle.splitmix(p, log_n, 1)[0]) or 2):
            got = coset(a.clone(), log_n, s, batch, p, g)
            assert torch.equal(got, three_call_reference(a, log_n, s, batch, p, g)), f"s = {s}"
            assert torch.equal(coset(got.clone(), log_n, s, batch, p, g, inverse=True), a), f"inverse∘forward, s = {s}"
            assert torch.equal(coset(coset(a.clone(), log_n, s, batch, p, g, inverse=True), log_n, s, batch, p, g), a), \
                f"forward∘inverse, s = {s}"
            if s == g:
                check_points(host(a).reshape(batch, n), host(got).reshape(batch, n), log_n, s, p, g)


def check_points(a, got, log_n, s, p, g):
    """The oracle's transform of a ⊙ s^j up to 2^12; Horner's rule at s·ω^k for five k at every size (rows 0 and last)."""
    n = 1 << log_n
    w = root(p, g, log_n)
    rows = sorted({0, len(a) - 1})
    if log_n <= 12:
        pw = np.array([pow(s, j, p) for j in range(n)], dtype=np.uint64)
        for r in rows:
            assert np.array_equal(got[r], oracle.ntt_fast(p, oracle.vec_mul(p, a[r], pw), g=g))
    for r in rows:
        for k in sorted({0, 1 % n, n // 2, n - 1, int(oracle.splitmix(n, r, 1)[0])}):
            assert int(got[r][k]) == oracle.poly_eval_horner(p, a[r], s * pow(w, k, p) % p), (r, k)


@pytest.mark.parametrize("name,log_n", [(n, k) for n, k in GRID if k < min(FIELDS[n][2], 26)],
                         ids=[f"{n}-2^{k}" for n, k in GRID if k < min(FIELDS[n][2], 26)])
def test_half_step_shift_gives_odd_outputs(name, log_n):
    """s = ω_2n: the odd outputs of the 2n-point transform of the row zero-padded to 2n words."""
    import torch
    p, g, _ = FIELDS[name]
    n = 1 << log_n
    a = fill(n, 77 + log_n, p)
    padded = torch.cat([a, torch.zeros_like(a)])
    big = ntt(padded, log_n + 1, 1, p, g)
    assert torch.equal(coset(a.clone(), log_n, root(p, g, log_n + 1), 1, p, g), big[1::2])


# ---- low-degree extension ---------------------------------------------------------------------------------------------
LDE_CASES = [("gl", 10), ("gl", 18), ("babybear", 10), ("babybear", 18), ("pbig", 12), ("p32", 8)]


@pytest.mark.parametrize("blowup", range(5))
@pytest.mark.parametrize("name,log_n", LDE_CASES, ids=[f"{n}-2^{k}" for n, k in LDE_CASES])
def test_lde(name, log_n, blowup):
    import torch
    from ronkathon_b200 import ops
    p, g, adicity = FIELDS[name]
    LN = log_n + blowup
    if LN > min(adicity, 26):
        pytest.skip("N does not divide p - 1")
    n, N = 1 << log_n, 1 << LN
    for batch in (1, 5 if LN <= 20 else 2):
        for d in sorted({1, n // 2 + 1, n, N}):
            coeffs = fill(batch * d, d + batch, p).view(batch, d)
            padded = torch.zeros((batch, N), dtype=torch.int64, device="cuda")
            padded[:, :d] = coeffs
            for s in (1, g, int(oracle.splitmix(p, LN, 1)[0]) or 2):
                out = ops.lde(_c(), coeffs, LN, s, p=p, g=g)
                assert out.shape == (batch, N)
                want = coset(padded.clone().view(-1), LN, s, batch, p, g).view(batch, N)
                assert torch.equal(out, want), (d, s)
                if s == 1:
                    assert torch.equal(out.view(-1), ntt(padded.clone().view(-1), LN, batch, p, g))
                if d <= n:   # every 2^blowup-th point is the n-point coset transform with the same shift
                    small = torch.zeros((batch, n), dtype=torch.int64, device="cuda")
                    small[:, :d] = coeffs
                    assert torch.equal(out[:, ::1 << blowup], coset(small.view(-1), log_n, s, batch, p, g).view(batch, n))
    one = ops.lde(_c(), fill(3, 5, p), LN, 5, p=p, g=g)   # 1-D input: one row, 1-D output
    assert one.shape == (N,)


# ---- launch records ---------------------------------------------------------------------------------------------------
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


RECORDS = [
    ("gl", 12, 1, False, ["ntt_coset_table", "ntt_single_coset"]),
    ("gl", 12, 1, True, ["ntt_coset_table", "intt_single_coset"]),
    ("gl", 16, 1, False, ["ntt_coset_table", "ntt_pass1_coset", "ntt_pass2_coset"]),
    ("gl", 20, 1, True, ["ntt_coset_table", "intt_pass1_coset", "intt_pass2_coset"]),
    ("gl", 22, 2, False, ["ntt_coset_table", "ntt3_pass1_coset", "ntt3_pass2_coset", "ntt3_pass3_coset"]),
    ("gl", 24, 1, False, ["ntt_coset_table", "ntt3_pass1_coset", "ntt3_pass2_coset", "ntt3_pass3_coset"]),
    ("gl", 24, 1, True, ["ntt_coset_table", "intt3_pass1_coset", "intt3_pass2_coset", "intt3_pass3_coset"]),
    ("gl", 26, 1, False, ["ntt_coset_table", "ntt_pass1_coset", "ntt_pass2_coset"]),
    ("babybear", 24, 1, False, ["ntt_coset_table", "ntt_pass1_coset", "ntt_pass2_coset"]),
    ("babybear", 13, 3, True, ["ntt_coset_table", "intt_single_coset"]),
]


@pytest.mark.parametrize("name,log_n,batch,inverse,want", RECORDS, ids=[f"{r[0]}-2^{r[1]}x{r[2]}-{'inv' if r[3] else 'fwd'}" for r in RECORDS])
def test_launch_record(name, log_n, batch, inverse, want):
    """One warmed call per family; at 2^24 the table launch plus the three passes: no pass over the data beyond the
    plain transform's."""
    p, g, _ = FIELDS[name]
    a = fill(batch << log_n, 3, p)
    coset(a, log_n, g, batch, p, g, inverse)
    c0 = _c().launches
    assert launch_names(_c(), lambda: coset(a, log_n, g, batch, p, g, inverse)) == want
    assert _c().launches - c0 == len(want)


def test_launch_record_lde_and_shift_one():
    from ronkathon_b200 import ops
    coeffs = fill(1 << 20, 4, GL)
    ops.lde(_c(), coeffs, 22, 7)
    assert launch_names(_c(), lambda: ops.lde(_c(), coeffs, 22, 7)) == \
        ["lde_pad", "ntt_coset_table", "ntt3_pass1_coset", "ntt3_pass2_coset", "ntt3_pass3_coset"]
    a = fill(1 << 16, 5, GL)
    plain = launch_names(_c(), lambda: ntt(a, 16, 1, GL, 7))
    assert launch_names(_c(), lambda: coset(a, 16, 1, 1, GL, 7)) == plain


# ---- other tuning contexts --------------------------------------------------------------------------------------------
ENVS = [{"RONK_NTT3": "0"}, {"RONK_NTT3_MID": "0"}, {"RONK_TILE_ADAPT": "0"}, {"RONK_PDL": "0"}, {"RONK_TW_TABLE": "1"}]


def context_with(env, stream=None):
    import torch
    from ronkathon_b200 import Context
    _c()
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


@pytest.mark.parametrize("env", ENVS, ids=[next(iter(e)) for e in ENVS])
def test_other_contexts_give_the_same_words(env):
    from ronkathon_b200 import ops
    c = context_with(env)
    try:
        for log_n in (16, 20, 22, 24):
            a = fill(1 << log_n, log_n, GL)
            for inverse in (False, True):
                want = coset(a.clone(), log_n, 7, 1, GL, 7, inverse)
                got = a.clone()
                ops.ntt_coset_(c, got, log_n, 7, inverse=inverse)
                c.sync()
                assert (got == want).all(), (log_n, inverse)
    finally:
        c.close()


# ---- memory safety, refused calls, host twins, streams ----------------------------------------------------------------
FRONT = 16


def arena(words):
    import torch
    return torch.full((FRONT + words + FRONT,), POISON, dtype=torch.int64, device="cuda")


@pytest.mark.parametrize("name,log_n,batch", [("gl", 5, 3), ("gl", 13, 2), ("gl", 14, 3), ("gl", 21, 2), ("gl", 24, 1),
                                              ("babybear", 9, 5), ("babybear", 17, 2), ("pbig", 22, 1)])
def test_guard_words_and_odd_offsets(name, log_n, batch):
    """In-place coset transforms and the LDE inside poisoned arenas, at an odd word offset: nothing outside the view
    moves and the LDE's input is left as it was."""
    import torch
    p, g, _ = FIELDS[name]
    n = 1 << log_n
    a = fill(batch * n, 9, p)
    for inverse in (False, True):
        buf = arena(batch * n + 1)
        view = buf[FRONT + 1:FRONT + 1 + batch * n]
        view.copy_(a)
        _c().call("ronk_ntt_coset_u64", p, g, view.data_ptr(), log_n, batch, g, int(inverse))
        want = coset(a.clone(), log_n, g, batch, p, g, inverse)
        assert torch.equal(view, want)
        assert (buf[:FRONT + 1] == POISON).all() and (buf[FRONT + 1 + batch * n:] == POISON).all()
    d = n // 2 + 1
    LN = log_n + (1 if log_n < 24 else 0)
    cin = arena(batch * d + 1)
    cview = cin[FRONT + 1:FRONT + 1 + batch * d]
    cview.copy_(fill(batch * d, 10, p))
    before = cin.clone()
    out = arena((batch << LN) + 1)
    oview = out[FRONT + 1:FRONT + 1 + (batch << LN)]
    _c().call("ronk_poly_lde_u64", p, g, cview.data_ptr(), d, LN, g, batch, oview.data_ptr())
    _c().sync()
    assert torch.equal(cin, before), "the LDE wrote to its input"
    assert (out[:FRONT + 1] == POISON).all() and (out[FRONT + 1 + (batch << LN):] == POISON).all()
    padded = torch.zeros((batch, 1 << LN), dtype=torch.int64, device="cuda")
    padded[:, :d] = cview.view(batch, d)
    assert torch.equal(oview, coset(padded.view(-1), LN, g, batch, p, g))


def test_refused_calls_write_nothing():
    import torch
    from ronkathon_b200 import _lib
    lib, h = _lib.lib(), _c()._h
    a = fill(1 << 12, 11, GL)
    out = arena(1 << 14)
    snap_a, snap_o = a.clone(), out.clone()
    P, O = a.data_ptr(), out.data_ptr() + 8 * FRONT
    EI, EU = _lib.EINVAL, _lib.EUNSUPPORTED
    cases = [
        (lib.ronk_ntt_coset_u64, (h, GL, 7, P, 12, 1, 0, 0), EI),            # shift 0
        (lib.ronk_ntt_coset_u64, (h, GL, 7, P, 12, 1, GL, 1), EI),           # shift p
        (lib.ronk_ntt_coset_u64, (h, GL, 7, P, 12, 1, GL + 5, 0), EI),       # shift > p
        (lib.ronk_ntt_coset_u64, (h, GL, 0, P, 12, 1, 3, 0), EI),            # g = 0
        (lib.ronk_ntt_coset_u64, (h, GL, 7, None, 12, 1, 3, 0), EI),         # null
        (lib.ronk_ntt_coset_u64, (h, 101, 2, P, 3, 1, 3, 0), EI),            # 8 does not divide 100
        (lib.ronk_ntt_coset_u64, (h, GL, 7, P, 27, 1, 3, 0), EU),            # log_n > 26
        (lib.ronk_ntt_coset_u64, (h, 100, 3, P, 1, 1, 3, 0), EI),            # not a prime modulus
        (lib.ronk_poly_lde_u64, (h, GL, 7, P, 0, 14, 3, 1, O), EI),          # d = 0
        (lib.ronk_poly_lde_u64, (h, GL, 7, P, (1 << 14) + 1, 14, 3, 1, O), EI),   # d > N
        (lib.ronk_poly_lde_u64, (h, GL, 7, P, 16, 14, 0, 1, O), EI),         # shift 0
        (lib.ronk_poly_lde_u64, (h, GL, 7, None, 16, 14, 3, 1, O), EI),      # null coeffs
        (lib.ronk_poly_lde_u64, (h, GL, 7, P, 16, 14, 3, 1, None), EI),      # null out
        (lib.ronk_poly_lde_u64, (h, GL, 7, O + 8, 16, 14, 3, 1, O), EI),     # out overlaps coeffs
        (lib.ronk_poly_lde_u64, (h, GL, 7, P, 16, 26, 3, 65, O), EU),        # batch·N > 2^32
        (lib.ronk_poly_lde_u64, (h, GL, 7, P, 16, 27, 3, 1, O), EU),         # log_n > 26
        (lib.ronk_poly_lde_u64, (h, 101, 2, P, 1, 3, 3, 1, O), EI),          # 8 does not divide 100
    ]
    for fn, args, code in cases:
        assert fn(*args) == code, (fn.__name__, args[1:])
        _c().sync()
        assert torch.equal(a, snap_a) and torch.equal(out, snap_o), (fn.__name__, args[1:])
    # batch 0 does nothing; log_n 0 is the identity
    assert lib.ronk_ntt_coset_u64(h, GL, 7, P, 12, 0, 3, 0) == 0
    assert lib.ronk_poly_lde_u64(h, GL, 7, P, 16, 14, 3, 0, O) == 0
    assert lib.ronk_ntt_coset_u64(h, GL, 7, P, 0, 7, 3, 0) == 0 and lib.ronk_ntt_coset_u64(h, GL, 7, P, 0, 7, 3, 1) == 0
    _c().sync()
    assert torch.equal(a, snap_a) and torch.equal(out, snap_o)
    assert lib.ronk_poly_lde_u64(h, GL, 7, P, 1, 0, 3, 5, O) == 0   # N = 1: the rows' constant terms
    _c().sync()
    assert torch.equal(out[FRONT:FRONT + 5], a[:5]) and (out[FRONT + 5:] == POISON).all()


@pytest.mark.parametrize("name,log_n,batch", [("gl", 11, 3), ("gl", 22, 1), ("babybear", 16, 2)])
def test_host_variants_equal_device(name, log_n, batch):
    from ronkathon_b200 import _lib
    p, g, _ = FIELDS[name]
    n = 1 << log_n
    a = oracle.splitmix(p, 12, batch * n)
    for inverse in (0, 1):
        h = a.copy()
        _c().call("ronk_ntt_coset_u64_host", p, g, h.ctypes.data_as(C.c_void_p), log_n, batch, g, inverse)
        assert np.array_equal(h, host(coset(dev(a), log_n, g, batch, p, g, bool(inverse))))
    d = n // 2 + 1
    coeffs = oracle.splitmix(p, 13, batch * d)
    out = np.zeros(batch * 2 * n, dtype=np.uint64)
    _c().call("ronk_poly_lde_u64_host", p, g, coeffs.ctypes.data_as(C.c_void_p), d, log_n + 1, g, batch,
              out.ctypes.data_as(C.c_void_p))
    from ronkathon_b200 import ops
    assert np.array_equal(out, host(ops.lde(_c(), dev(coeffs).view(batch, d), log_n + 1, g, p=p, g=g)).reshape(-1))
    assert _lib.lib().ronk_ntt_coset_u64_host(_c()._h, p, g, a.ctypes.data_as(C.c_void_p), log_n, batch, 0, 0) == _lib.EINVAL


@pytest.mark.parametrize("log_n,batch", [(10, 7), (16, 1), (24, 1)])
def test_gated_non_blocking_stream(log_n, batch):
    """On a fresh context on a non-blocking stream held behind a 50 ms sleep: the calls return before the stream has
    run, read the inputs copied in behind the gate and give the default context's words."""
    import torch
    from ronkathon_b200 import ops
    n = batch << log_n
    a = fill(n, 14, GL)
    coeffs = fill(batch << (log_n - 1), 15, GL).view(batch, -1)
    want_c = coset(a.clone(), log_n, 7, batch, GL, 7)
    want_i = coset(a.clone(), log_n, 7, batch, GL, 7, inverse=True)
    want_l = ops.lde(_c(), coeffs, log_n, 7)
    _c().sync()
    s = torch.cuda.Stream()
    c = context_with({}, s)
    try:
        bufs = [a.flip(0).contiguous() for _ in range(2)]
        cin = coeffs.flip(0).contiguous()
        with torch.cuda.stream(s):   # once on wrong inputs: first uses of kernels and plans out of the timed gate
            ops.ntt_coset_(c, bufs[0].clone(), log_n, 7, batch=batch)
            ops.ntt_coset_(c, bufs[1].clone(), log_n, 7, batch=batch, inverse=True)
            ops.lde(c, cin, log_n, 7)
        s.synchronize()
        with torch.cuda.stream(s):
            torch.cuda._sleep(100_000_000)
            for b in bufs:
                b.copy_(a)
            cin.copy_(coeffs)
            ops.ntt_coset_(c, bufs[0], log_n, 7, batch=batch)
            ops.ntt_coset_(c, bufs[1], log_n, 7, batch=batch, inverse=True)
            out = ops.lde(c, cin, log_n, 7)
            assert not s.query(), "the stream finished before the calls returned"
            got = [bufs[0].clone(), bufs[1].clone(), out.clone()]
        s.synchronize()
    finally:
        c.close()
    assert torch.equal(got[0], want_c) and torch.equal(got[1], want_i) and torch.equal(got[2], want_l)
