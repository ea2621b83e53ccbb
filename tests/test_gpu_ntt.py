"""GPU parity: Polynomial::fft / ifft / dft through the C ABI vs the reference KATs, the faithful
oracle and the independent golden vectors.  Bit-exact everywhere (integer path)."""
import numpy as np
import pytest

import oracle
from gpu_util import GL, MONT_PRIMES, PBIG, BABYBEAR, ctx, dev, host, s64, summary

pytestmark = pytest.mark.gpu


def gpu_ntt(a, log_n, batch=1, inverse=False, p=GL, g=7):
    from ronkathon_b200 import ops
    d = dev(a)
    ops.ntt_(ctx(), d, log_n, batch, inverse, p, g)
    return host(d)


def test_reference_kat_polynomial_api(kats):
    """polynomial/tests.rs:119-142: dft == fft == [10,79,99,18]; ifft(fft(p)) == p."""
    from ronkathon_b200 import PlutoBaseField, Polynomial, RonkPanic
    ctx()
    k = kats["polynomial"]
    poly = Polynomial(k["a"], PlutoBaseField)
    assert [int(v) for v in poly.fft().coefficients] == k["fft_a"]
    assert [int(v) for v in poly.dft().coefficients] == k["dft_a"]
    assert poly.fft().ifft() == poly
    with pytest.raises(RonkPanic):                      # polynomial/tests.rs:46-55
        Polynomial(k["dft_3_terms_panics"], PlutoBaseField).dft()
    with pytest.raises(RonkPanic):                      # not a power of two (mod.rs:274)
        Polynomial([1, 2, 3], PlutoBaseField).fft()
    with pytest.raises(RonkPanic):                      # 8 ∤ 100: no 8th root of unity in F101
        Polynomial([1] * 8, PlutoBaseField).fft()


@pytest.mark.parametrize("p,log_n", [(101, 1), (101, 2), (17, 1), (17, 2), (17, 3), (17, 4), (127, 1)])
def test_small_moduli_every_size(p, log_n):
    g = oracle.generator(p)
    n = 1 << log_n
    rng = np.random.default_rng(log_n + p)
    for batch in (1, 5, 1000):
        a = rng.integers(0, p, n * batch).astype(np.uint64)
        X = gpu_ntt(a, log_n, batch, p=p, g=g)
        for b in (0, batch // 2, batch - 1):
            assert np.array_equal(X[b * n:(b + 1) * n], oracle.fft(p, a[b * n:(b + 1) * n]))
        assert np.array_equal(gpu_ntt(X, log_n, batch, True, p, g), a)


@pytest.mark.parametrize("n", [2, 4, 5, 10, 20, 25, 50, 100])
def test_dft_any_divisor_of_p_minus_1(n):
    """dft works for every n | 100 over F101 (polynomial/mod.rs:240-258), not only powers of two."""
    from ronkathon_b200 import PlutoBaseField, Polynomial
    ctx()
    a = list(np.random.default_rng(n).integers(0, 101, n))
    assert [int(v) for v in Polynomial(a, PlutoBaseField).dft().coefficients] == list(oracle.dft(101, a))


@pytest.mark.parametrize("log_n", list(range(1, 15)))
def test_goldilocks_single_tile_sizes(log_n):
    n = 1 << log_n
    batch = 7 if log_n <= 11 else 2
    a = oracle.splitmix(GL, 100 + log_n, n * batch)
    X = gpu_ntt(a, log_n, batch)
    for b in range(batch):
        ref = oracle.fft(GL, a[b * n:(b + 1) * n]) if log_n <= 12 else oracle.ntt_fast(GL, a[b * n:(b + 1) * n])
        assert np.array_equal(X[b * n:(b + 1) * n], ref), (log_n, b)
    assert np.array_equal(gpu_ntt(X, log_n, batch, inverse=True), a)


@pytest.mark.parametrize("log_n,batch", [(15, 3), (16, 2), (17, 1), (18, 2), (19, 1), (20, 1), (21, 1), (22, 1)])
def test_goldilocks_two_pass_sizes(log_n, batch):
    n = 1 << log_n
    a = oracle.splitmix(GL, 42, n * batch)
    X = gpu_ntt(a, log_n, batch)
    for b in range(batch):
        assert np.array_equal(X[b * n:(b + 1) * n], oracle.ntt_fast(GL, a[b * n:(b + 1) * n])), (log_n, b)
    assert np.array_equal(gpu_ntt(X, log_n, batch, inverse=True), a)


def _montgomery_cases():
    sizes = {"babybear": range(1, 27), "pbig": range(1, 27), "koalabear": (1, 5, 9, 12, 13, 14, 15, 18, 21, 24),
             "p32": range(1, 17), "p57": (1, 9, 13, 14, 15, 17, 20, 23, 26),
             "gl_g5": (1, 2, 10, 13, 14, 15, 16, 20, 24, 25, 26), "p2adic3": (1, 2, 3)}
    cases = [(name, lg, 1) for name in MONT_PRIMES for lg in sizes[name]]
    return cases + [(name, lg, b) for name in ("babybear", "pbig") for lg, b in ((12, 64), (16, 3), (18, 17))]


@pytest.mark.parametrize("name,log_n,batch", _montgomery_cases())
def test_montgomery_transform_every_size(name, log_n, batch):
    """Every (p, g) except Goldilocks with g = 7 runs on the run-time-modulus Montgomery kernels: the single-tile kernel up
    to 2^13, the two-pass tile kernel from 2^14 to 2^26.  Single transforms shrink the tiles until the grid fills the GPU
    (2^20: pass-1 tiles of 2^12 points, 128 threads; pass-2 tiles of 2^11, 128 threads); from 2^22 up the preferred
    2^14-point pass-1 tile (512 threads) and 2^13-point pass-2 tile (256 threads) run.  The batches reach the same
    preferred tiles at 17 × 2^18, 2^12-point single tiles (128 threads) at 64 × 2^12, and shrunken tiles at 3 × 2^16.
    Forward against the oracle (bit for bit up to 2^22 words, else X[k] = a(ω^k) by Horner at sampled k), Goldilocks with
    g = 7^5 against the g = 7 transform permuted by k → 5k mod n at full length, the fused point-wise multiply and the
    inverse round trip.  The first two inputs are p - 1 and p - 2."""
    _check_montgomery_transform(name, log_n, batch)


def test_generic_montgomery_path_on_goldilocks_and_other_64bit_primes():
    """A different generator sends Goldilocks through the run-time-modulus Montgomery kernels — the path p = 101
    uses — and must agree with the oracle; so must another NTT-friendly prime.  The original cases (Goldilocks with
    g = 7^5 at 2^10 and 2^16, 29·2^57 + 1 at 2^9, 2^13 and 2^17) with the checks of the every-size test above."""
    for name, log_n in (("gl_g5", 10), ("gl_g5", 16), ("p57", 9), ("p57", 13), ("p57", 17)):
        _check_montgomery_transform(name, log_n, 1)


def _check_montgomery_transform(name, log_n, batch):
    from ronkathon_b200 import ops
    c = ctx()
    p, g, _ = MONT_PRIMES[name]
    n = 1 << log_n
    a = host(ops.splitmix_fill(c, n * batch, 800 + log_n, p)).copy()
    a[0], a[1] = p - 1, p - 2
    m = ops.splitmix_fill(c, n * batch, 900 + log_n, p)
    x = dev(a)
    ops.ntt_(c, x, log_n, batch, False, p, g)
    X = host(x)
    if n * batch <= 1 << 22:
        members = range(batch)
    elif n <= 1 << 22:
        members = sorted({0, batch // 2, batch - 1})
    else:
        members = []
        w = oracle.root_of_unity(p, n, g)
        for k in sorted({0, 1, n // 2 + 3, (n // 3) | 1, n - 1}):
            assert int(X[k]) == oracle.poly_eval_horner(p, a[:n], oracle.pow_(p, w, k)), (name, log_n, k)
    for b in members:
        assert np.array_equal(X[b * n:(b + 1) * n], oracle.ntt_fast(p, a[b * n:(b + 1) * n], g=g)), (name, log_n, b)
    if name == "gl_g5":
        X7 = gpu_ntt(a, log_n, batch)
        perm = (np.arange(n, dtype=np.uint64) * np.uint64(5)) % np.uint64(n)
        assert np.array_equal(X.reshape(batch, n), X7.reshape(batch, n)[:, perm])
        del X7, perm
    y = dev(a)
    ops.ntt_mul_(c, y, m, log_n, batch, p, g)
    assert np.array_equal(host(y), oracle.vec_mul(p, X, host(m)))
    del y, m
    ops.ntt_(c, x, log_n, batch, True, p, g)
    assert np.array_equal(host(x), a)


def _context_with(env):
    import os
    import torch
    from ronkathon_b200 import Context
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return Context(0, torch.cuda.current_stream().cuda_stream)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def test_montgomery_opt_in_variants_agree_with_the_default():
    """The n-word inter-pass twiddle table (RONK_TW_TABLE=1: interpass_table<MontField>, twiddles in Montgomery form)
    and launches without programmatic dependent launch (RONK_PDL=0) reproduce the default context's Montgomery
    transforms bit for bit, with a prime above 2^63: forward, fused multiply and inverse at 2^20 and 2^24."""
    import torch
    from ronkathon_b200 import ops
    c0 = ctx()
    p, g = PBIG, 3
    ref = {}
    for lg in (20, 24):
        a = ops.splitmix_fill(c0, 1 << lg, 31 + lg, p)
        m = ops.splitmix_fill(c0, 1 << lg, 41 + lg, p)
        x = a.clone()
        ops.ntt_(c0, x, lg, 1, False, p, g)
        y = a.clone()
        ops.ntt_mul_(c0, y, m, lg, 1, p, g)
        z = x.clone()
        ops.ntt_(c0, z, lg, 1, True, p, g)
        c0.sync()
        assert torch.equal(z, a)
        ref[lg] = (a, m, x, y)
    for env in ({"RONK_TW_TABLE": "1"}, {"RONK_PDL": "0"}):
        c1 = _context_with(env)
        for lg, (a, m, x0, y0) in ref.items():
            x = a.clone()
            ops.ntt_(c1, x, lg, 1, False, p, g)
            y = a.clone()
            ops.ntt_mul_(c1, y, m, lg, 1, p, g)
            z = x.clone()
            ops.ntt_(c1, z, lg, 1, True, p, g)
            c1.sync()
            assert torch.equal(x, x0) and torch.equal(y, y0) and torch.equal(z, a), (env, lg)
        c1.close()


def _edge_cases():
    gl = [("gl", lg, 1) for lg in range(1, 16)]                         # single tile 2^1 … 2^13; two-pass 2^14, 2^15
    gl += [("gl", 16, 1), ("gl", 16, 2), ("gl", 16, 3)]                 # cluster kernel (batch ≤ 2), 256-point tiles
    gl += [("gl", lg, 1) for lg in range(17, 27)]                       # split, 2^20, mid, 2^24, split over 2^24
    return gl + [("pbig", lg, 1) for lg in (1, 4, 9, 13, 14, 16, 19, 22, 24, 26)]


@pytest.mark.parametrize("name,log_n,batch", _edge_cases())
def test_exact_edge_inputs_through_every_dispatch_branch(name, log_n, batch):
    """Inputs at the edge of the range whose transforms are known exactly, at full length, through every branch of
    run_ntt for Goldilocks (g = 7) and through the Montgomery kernels with a prime above 2^63:
    all p - 1 → X[0] = -n, the rest 0; the inverse of all c → [c, 0, …, 0]; p - 1 at odd j → X[0] = -n/2, X[n/2] = n/2,
    the rest 0; an impulse at j = 1 / j = n - 1 → X[k] = ω^(±k) (the powers kernel, itself spot-checked against the
    oracle); a fused multiply by all p - 1 → -X."""
    import torch
    from ronkathon_b200 import _lib, ops
    c = ctx()
    p, g = (GL, 7) if name == "gl" else (PBIG, 3)
    n, total = 1 << log_n, batch << log_n

    def ntt(t, inverse=False, mul=None):
        if mul is None:
            ops.ntt_(c, t, log_n, batch, inverse, p, g)
        else:
            ops.ntt_mul_(c, t, mul, log_n, batch, p, g)
        return t.view(batch, n)

    def full(v):
        return torch.full((total,), s64(v), dtype=torch.int64, device="cuda")

    def want(*pairs):
        e = torch.zeros((batch, n), dtype=torch.int64, device="cuda")
        for k, v in pairs:
            e[:, k] = s64(v % p)
        return e

    assert torch.equal(ntt(full(p - 1)), want((0, -n)))
    assert torch.equal(ntt(full(p - 2), inverse=True), want((0, p - 2)))
    alt = torch.zeros(total, dtype=torch.int64, device="cuda")
    alt[1::2] = s64(p - 1)
    assert torch.equal(ntt(alt), want((0, -(n // 2)), (n // 2, n // 2)))
    w = oracle.root_of_unity(p, n, g)
    for j, root in ((1, w), (n - 1, oracle.inverse(p, w))):
        imp = torch.zeros((batch, n), dtype=torch.int64, device="cuda")
        imp[:, j] = 1
        pw = torch.empty(n, dtype=torch.int64, device="cuda")
        c.call("ronk_field_powers_u64", p, root, 1, _lib._ptr(pw), n)
        pwh = host(pw)
        for k in sorted({0, 1, n // 2, n // 3, n - 1}):
            assert int(pwh[k]) == oracle.pow_(p, root, k), (j, k)
        assert torch.equal(ntt(imp.view(-1)), pw.expand(batch, n)), j
    a = ops.splitmix_fill(c, total, 60 + log_n, p)
    X = host(ntt(a.clone()))
    negX = np.where(X == 0, np.uint64(0), np.uint64(p) - X)
    assert np.array_equal(host(ntt(a, mul=full(p - 1))), negX)


@pytest.mark.parametrize("name,log_l", [("gl", 21), ("gl", 22), ("gl", 23), ("gl", 24), ("pbig", 21), ("pbig", 24)])
def test_poly_mul_of_all_minus_one_operands_is_the_trapezoid(name, log_l):
    """poly_mul with 2^21 … 2^24-point transforms (Goldilocks: the bounded 256-point-tile route; the prime above 2^63: the
    bounded Montgomery two-pass route).  Two all-(p - 1) operands multiply like two all-ones operands, so coefficient i
    of the product is min(i + 1, da, db, da + db - 1 - i), exactly."""
    from ronkathon_b200 import ops
    c = ctx()
    p, g = (GL, 7) if name == "gl" else (PBIG, 3)
    L = (1 << log_l) - 5 if log_l < 24 else (1 << 24) - 1
    da = L // 3 + 7
    db = L + 1 - da
    a = dev(np.full(da, p - 1, dtype=np.uint64))
    b = dev(np.full(db, p - 1, dtype=np.uint64))
    got = host(ops.poly_mul(c, a, b, p, g))
    i = np.arange(L, dtype=np.uint64)
    exp = np.minimum(np.minimum(i + np.uint64(1), np.uint64(min(da, db))), np.uint64(L) - i)
    assert len(got) == L and np.array_equal(got, exp)


def test_golden_vectors(gold64):
    """BASELINE config 2 (2^20 forward NTT, bit-exact vs CPU) + the independent pure-Python vectors."""
    assert list(gpu_ntt(np.arange(1, 9, dtype=np.uint64), 3)) == gold64["ntt8_1to8"]
    assert list(gpu_ntt(oracle.splitmix(GL, 42, 1024), 10)) == gold64["ntt_2_10_full"]
    for lg in (16, 20):
        X = gpu_ntt(oracle.splitmix(GL, 42, 1 << lg), lg)
        g = gold64["ntt_2_%d" % lg]
        s = summary(X)
        for key in s:
            assert s[key] == g[key], (lg, key)
        for k, v in g["horner_checks"].items():
            assert int(X[int(k)]) == v


def test_metric_size_2_24_bit_exact_and_properties():
    """The BASELINE metric size: 2^24 forward NTT, bit-exact vs the oracle, plus the
    size-independent properties (round trip, linearity, spot X[k] == a(ω^k))."""
    from ronkathon_b200 import ops
    c = ctx()
    lg, n = 24, 1 << 24
    a = oracle.splitmix(GL, 42, n)
    X = gpu_ntt(a, lg)
    assert np.array_equal(X, oracle.ntt_fast(GL, a))
    w = oracle.root_of_unity(GL, n)
    for k in (0, 1, n // 2 + 3, n - 1):
        assert int(X[k]) == oracle.poly_eval_horner(GL, a, oracle.pow_(GL, w, k))
    assert np.array_equal(gpu_ntt(X, lg, inverse=True), a)
    # linearity: NTT(a + b) == NTT(a) + NTT(b), all on the GPU
    b = ops.splitmix_fill(c, n, 43)
    da = dev(a)
    s = ops.field_binop(c, "add", da, b)
    ops.ntt_(c, s, lg); ops.ntt_(c, b, lg)
    assert np.array_equal(host(s), host(ops.field_binop(c, "add", dev(X), b)))


@pytest.mark.parametrize("log_n", [23, 25, 26])
def test_largest_sizes(log_n):
    """Up to the largest supported transform (2^26: N1 = N2 = 2^13, 13-bit sub-transforms in both passes,
    512 MiB of data + 512 MiB workspace): X[k] = a(ω^k) at sampled k against the oracle's Horner
    evaluation, full bit-exact comparison where the CPU transform is quick, and the round trip."""
    from ronkathon_b200 import ops
    c = ctx()
    n = 1 << log_n
    d = ops.splitmix_fill(c, n, 4242)
    a = host(d).copy()
    assert np.array_equal(a[:1000], oracle.splitmix(GL, 4242, 1000))
    ops.ntt_(c, d, log_n)
    X = host(d)
    w = oracle.root_of_unity(GL, n)
    for k in (0, 1, n // 2 + 3, (n // 3) | 1, n - 1):
        assert int(X[k]) == oracle.poly_eval_horner(GL, a, oracle.pow_(GL, w, k)), (log_n, k)
    if log_n <= 23:
        assert np.array_equal(X, oracle.ntt_fast(GL, a))
    ops.ntt_(c, d, log_n, inverse=True)
    assert np.array_equal(host(d), a)
    del d


def test_fused_pointwise_multiply(gold64):
    from ronkathon_b200 import ops
    c = ctx()
    for lg in (10, 16):
        n = 1 << lg
        a, b = oracle.splitmix(GL, 42, n), oracle.splitmix(GL, 43, n)
        A, B = dev(a), dev(b)
        ops.ntt_(c, A, lg)
        ops.ntt_mul_(c, B, A, lg)
        assert np.array_equal(host(B), oracle.vec_mul(GL, oracle.ntt_fast(GL, a), oracle.ntt_fast(GL, b)))
        ops.ntt_(c, B, lg, inverse=True)
        if lg == 16:
            g = gold64["cyclic_conv_2_16_seed42_seed43"]
            s = summary(host(B))
            for key in s:
                assert s[key] == g[key], key


def test_batched_config5_shape():
    """BASELINE config 5's per-GPU shard shape, reduced: 64 × 2^16 contiguous transforms."""
    lg, batch = 16, 64
    n = 1 << lg
    a = oracle.splitmix(GL, 77, n * batch)
    X = gpu_ntt(a, lg, batch)
    for b in (0, 1, 31, 63):
        assert np.array_equal(X[b * n:(b + 1) * n], oracle.ntt_fast(GL, a[b * n:(b + 1) * n]))
    assert np.array_equal(gpu_ntt(X, lg, batch, inverse=True), a)


def test_host_pointer_variant_and_errors():
    from ronkathon_b200 import RonkError, RonkPanic
    c = ctx()
    a = oracle.splitmix(GL, 3, 1 << 13)
    buf = a.copy()
    c.call("ronk_ntt_u64_host", GL, 7, buf.ctypes.data, 13, 1, 0)
    assert np.array_equal(buf, oracle.ntt_fast(GL, a))
    with pytest.raises(RonkPanic):   # 2^33 ∤ p-1
        c.call("ronk_ntt_u64", GL, 7, dev(a).data_ptr(), 33, 1, 0)
    with pytest.raises(RonkError) as ei:
        c.call("ronk_ntt_u64", GL, 7, dev(a).data_ptr(), 27, 1, 0)
    assert ei.value.code == 5
    with pytest.raises(RonkPanic):   # composite modulus
        c.call("ronk_ntt_u64", 100, 7, dev(a).data_ptr(), 2, 1, 0)


def test_distributed_building_blocks():
    """ronk_field_powers_u64 and ronk_ntt_strided_small_u64 (cross-rank butterflies) vs the oracle."""
    import torch
    c = ctx()
    w = oracle.root_of_unity(GL, 1 << 20)
    for n, scale in ((1, 1), (5, 3), (4097, 12345678901234567)):
        out = torch.empty(n, dtype=torch.int64, device="cuda")
        c.call("ronk_field_powers_u64", GL, w, scale, out.data_ptr(), n)
        exp = [oracle.mul(GL, scale, oracle.pow_(GL, w, i)) for i in range(n)]
        assert list(host(out)) == exp
    for log_g in (1, 2, 3, 4):
        G, stride, count = 1 << log_g, 37, 29
        a = oracle.splitmix(GL, log_g, G * stride)
        d = dev(a)
        c.call("ronk_ntt_strided_small_u64", GL, 7, d.data_ptr(), log_g, stride, count, 0)
        got = host(d)
        exp = a.copy()
        for k in range(count):
            exp[k:k + G * stride:stride] = oracle.fft(GL, a[k:k + G * stride:stride].copy())
        assert np.array_equal(got, exp)
        c.call("ronk_ntt_strided_small_u64", GL, 7, d.data_ptr(), log_g, stride, count, 1)
        assert np.array_equal(host(d), a)


def test_distributed_transform_single_rank_group():
    """ntt_distributed / msm_distributed with a 1-rank NCCL group: the whole code path on one GPU."""
    import os
    import torch
    import torch.distributed as dist
    from ronkathon_b200 import dist as rd
    c = ctx()
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29617")
    dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device("cuda", 0))
    try:
        ops_ = rd.LocalOps(c)
        a = oracle.splitmix(GL, 42, 1 << 14)
        out = rd.ntt_distributed(ops_, dev(a), 14)
        assert np.array_equal(host(rd.gather_distributed_output(out, 14)), oracle.ntt_fast(GL, a))
    finally:
        dist.destroy_process_group()


def test_pipelined_host_submit_wait():
    """ronk_ntt_u64_host_submit/_wait: several host buffers in flight over the two slots."""
    import torch
    c = ctx()
    lg = 18
    bufs, exps = [], []
    for i in range(5):
        a = oracle.splitmix(GL, 900 + i, 1 << lg)
        t = torch.from_numpy(a.copy().view(np.int64)).pin_memory()
        bufs.append(t); exps.append(oracle.ntt_fast(GL, a))
    for i, t in enumerate(bufs):
        c.call("ronk_ntt_u64_host_submit", GL, 7, t.data_ptr(), lg, 1, 0, i & 1)
        if i >= 1:
            c.call("ronk_ntt_u64_host_wait", (i - 1) & 1)
    c.call("ronk_ntt_u64_host_wait", (len(bufs) - 1) & 1)
    for t, e in zip(bufs, exps):
        assert np.array_equal(t.numpy().view(np.uint64), e)
    c.call("ronk_ntt_u64_host_wait", 0)  # idempotent on an idle slot


def test_opt_in_kernel_variants_agree_with_the_default():
    """The switches read at ronk_ctx_create select alternative formulations of the same transform: the default 2^24 path
    is the three-pass kernel (ntt3_kernel.cuh, with programmatic dependent launch); RONK_NTT3=0 is the two-pass tile
    kernel, optionally with the specialised 4096-point-per-tile kernel (RONK_FAST12=1: pairs, additive shared-memory
    layout, round 0 fed from HBM) or the n-word inter-pass twiddle table (RONK_TW_TABLE=1); RONK_PDL=0 launches the
    passes without overlap.  Each must reproduce the default context's 2^24 and 2^23 transforms bit for bit, forward,
    fused-multiply and inverse."""
    import os
    import torch
    from ronkathon_b200 import Context, ops
    c0 = ctx()
    a = ops.splitmix_fill(c0, 1 << 24, 11, GL, "cuda")
    m = ops.splitmix_fill(c0, 1 << 24, 12, GL, "cuda")
    ref = {}
    for lg in (24, 23):
        x = a[: 1 << lg].clone()
        ops.ntt_(c0, x, lg)
        y = a[: 1 << lg].clone()
        ops.ntt_mul_(c0, y, m[: 1 << lg].clone(), lg)
        z = x.clone()
        ops.ntt_(c0, z, lg, inverse=True)
        c0.sync()
        assert torch.equal(z, a[: 1 << lg])
        ref[lg] = (x, y)
    for env in ({"RONK_NTT3": "0"}, {"RONK_NTT3": "0", "RONK_FAST12": "1"}, {"RONK_NTT3": "0", "RONK_TW_TABLE": "1"}, {"RONK_PDL": "0"},
                {"RONK_NTT3_T1": "24"}, {"RONK_NTT3_PDL": "0"}):   # the 128 MiB pass-1 twiddle table (default: stepped), no PDL
        old = {k: os.environ.get(k) for k in env}
        os.environ.update(env)
        try:
            c1 = Context(0, torch.cuda.current_stream().cuda_stream)
        finally:
            for k, v in old.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
        for lg in (24, 23):
            x = a[: 1 << lg].clone()
            ops.ntt_(c1, x, lg)
            y = a[: 1 << lg].clone()
            ops.ntt_mul_(c1, y, m[: 1 << lg].clone(), lg)
            z = x.clone()
            ops.ntt_(c1, z, lg, inverse=True)
            c1.sync()
            assert torch.equal(x, ref[lg][0]) and torch.equal(y, ref[lg][1]) and torch.equal(z, a[: 1 << lg]), (env, lg)
        c1.close()


def test_three_pass_batch_of_2_24():
    """A batch of two 2^24-point transforms through the three-pass kernel equals the two transforms done singly
    (which test_metric_size_2_24_bit_exact_and_properties pins against the oracle)."""
    import torch
    from ronkathon_b200 import ops
    c = ctx()
    a = ops.splitmix_fill(c, 2 << 24, 21, GL, "cuda")
    one = [a[: 1 << 24].clone(), a[1 << 24:].clone()]
    for t in one:
        ops.ntt_(c, t, 24)
    both = a.clone()
    ops.ntt_(c, both, 24, batch=2)
    c.sync()
    assert torch.equal(both[: 1 << 24], one[0]) and torch.equal(both[1 << 24:], one[1])
    ops.ntt_(c, both, 24, batch=2, inverse=True)
    c.sync()
    assert torch.equal(both, a)



def test_2_20_interleaved_tile_path():
    """BASELINE config 2's size through the 256-point-tile kernels (16 interleaved 2^16-point transforms + the radix-16
    pass): a batch of 3 bit-exact against the oracle, fused multiply, inverse round trip, out-of-place source — and
    bit-for-bit agreement with the two-pass tile kernel (RONK_NTT3_20=0)."""
    import os
    import torch
    from ronkathon_b200 import Context, ops
    c0 = ctx()
    n, batch = 1 << 20, 3
    a = oracle.splitmix(GL, 77, n * batch)
    m = oracle.splitmix(GL, 78, n * batch)
    x = dev(a)
    ops.ntt_(c0, x, 20, batch)
    X = host(x)
    for b in range(batch):
        assert np.array_equal(X[b * n:(b + 1) * n], oracle.ntt_fast(GL, a[b * n:(b + 1) * n])), b
    y = dev(a)
    ops.ntt_mul_(c0, y, dev(m), 20, batch)
    assert np.array_equal(host(y), oracle.vec_mul(GL, X, m))
    ops.ntt_(c0, x, 20, batch, inverse=True)
    assert np.array_equal(host(x), a)
    for env in ("RONK_NTT3_20", "RONK_NTT3_T1"):   # the two-pass tile kernel; the stepped pass-A2 twiddle (default: 8 MiB table)
        os.environ[env] = "0"
        try:
            c1 = Context(0, torch.cuda.current_stream().cuda_stream)
        finally:
            os.environ.pop(env)
        z = dev(a)
        ops.ntt_(c1, z, 20, batch)
        c1.sync()
        assert np.array_equal(host(z), X), env
        ops.ntt_(c1, z, 20, batch, inverse=True)
        c1.sync()
        assert np.array_equal(host(z), a), env
        c1.close()


def test_2_16_cluster_kernel_matches_the_two_launch_path():
    """Small batches of 2^16-point transforms take ntt16c_kernel (one launch, a 16-CTA cluster per transform, the
    pass-2 → pass-3 exchange through distributed shared memory, in place).  Forward against the oracle, fused
    multiply, inverse round trip, for every batch size up to the switch-over and one beyond it, and bit-for-bit
    agreement with a context that never uses the cluster kernel."""
    import os
    import torch
    from ronkathon_b200 import Context, ops
    c0 = ctx()
    os.environ["RONK_NTT16_CLUSTER_MAX_BATCH"] = "0"
    try:
        c1 = Context(0, torch.cuda.current_stream().cuda_stream)
    finally:
        os.environ.pop("RONK_NTT16_CLUSTER_MAX_BATCH")
    n = 1 << 16
    os.environ["RONK_NTT16_CLUSTER_MAX_BATCH"] = "8"   # the default switch-over is 2: widen it for this test
    try:
        c8 = Context(0, torch.cuda.current_stream().cuda_stream)
    finally:
        os.environ.pop("RONK_NTT16_CLUSTER_MAX_BATCH")
    for batch in (1, 2, 3, 8, 9):
        c0 = c8
        a = oracle.splitmix(GL, 300 + batch, n * batch)
        m = oracle.splitmix(GL, 400 + batch, n * batch)
        x = dev(a)
        ops.ntt_(c0, x, 16, batch)
        X = host(x)
        for b in (0, batch - 1):
            assert np.array_equal(X[b * n:(b + 1) * n], oracle.ntt_fast(GL, a[b * n:(b + 1) * n])), (batch, b)
        z = dev(a)
        ops.ntt_(c1, z, 16, batch)
        c1.sync()
        assert np.array_equal(host(z), X), batch
        y = dev(a)
        ops.ntt_mul_(c0, y, dev(m), 16, batch)
        assert np.array_equal(host(y), oracle.vec_mul(GL, X, m)), batch
        ops.ntt_(c0, x, 16, batch, inverse=True)
        assert np.array_equal(host(x), a), batch
    # the launch counter shows which path ran: one launch per call through the cluster kernel
    c0 = ctx()                                          # the default context: one transform → one launch
    x = dev(oracle.splitmix(GL, 5, n))
    ops.ntt_(c0, x, 16, 1)
    before = c0.launches
    ops.ntt_(c0, x, 16, 1)
    assert c0.launches - before == 1
    c1.close()
    c8.close()


@pytest.mark.parametrize("log_g", [1, 2, 3, 4])
def test_virtual_rank_distributed_transform(log_g):
    """ronk_ntt_u64_dist with G = 2, 4, 8, 16 VIRTUAL ranks on one device (ronk_ntt_u64_dist_virtual): the local
    transforms with the twiddle column ω_n^(r·k') in their store phase, the pack kernel and cross_rank_kernel<log G> —
    every kernel and index formula of both exchange flavours of the multi-GPU call — reassembled and compared with the
    oracle bit for bit; Goldilocks and a generic (Montgomery) modulus, single transforms and batches."""
    from ronkathon_b200 import _lib
    from ronkathon_b200 import dist as rd
    c = ctx()
    G = 1 << log_g
    cases = [(GL, 7, max(2 * log_g, 4), 1), (GL, 7, 12, 3), (GL, 7, 16 + log_g, 2), (GL, 7, 20, 1), (GL, 7, 21 + log_g, 1),
             (2013265921, 31, 10, 2), (GL, pow(7, 5, GL), 12, 2),
             (PBIG, 3, 20 + log_g, 1), (BABYBEAR, 31, 16 + log_g, 2)]   # shared multiplier through the Montgomery two-pass kernel
    for p, g, log_n, batch in cases:
        n, m = 1 << log_n, (1 << log_n) // G
        blk = m // G
        full = [oracle.splitmix(p, 600 + 7 * b + log_n, n) for b in range(batch)]
        want = [oracle.ntt_fast(p, a, g=g) for a in full]
        for flavour in (rd.DIST_NCCL, rd.DIST_FUSED):
            loc = np.concatenate([np.concatenate([a[r::G] for a in full]) for r in range(G)])   # [rank][batch][m]
            d = dev(loc)
            c.call("ronk_ntt_u64_dist_virtual", p, g, _lib._ptr(d), log_n, batch, log_g, flavour)
            out = host(d).reshape(G, batch, G, blk)                                             # [rank s][b][q][k]
            for b in range(batch):
                X = np.empty(n, dtype=np.uint64)
                for s in range(G):
                    for q in range(G):
                        X[s * blk + m * q: s * blk + m * q + blk] = out[s, b, q]
                assert np.array_equal(X, want[b]), (p, log_n, batch, flavour, b)


@pytest.mark.parametrize("log_n,batch", [(21, 2), (22, 1), (23, 1)])
def test_mid_sizes_through_the_tile_kernels(log_n, batch):
    """2^21 … 2^23 through the 256-point-tile kernels (first pass of 32 / 64 / 128 points, passes 2 and 3 as for 2^24):
    bit-exact against the oracle, fused multiply, inverse round trip, and bit-for-bit agreement with the two-pass
    tile kernel (RONK_NTT3_MID=0) and with the table-fed first-pass twiddle (RONK_NTT3_T1=24)."""
    import os
    import torch
    from ronkathon_b200 import Context, ops
    c0 = ctx()
    n = 1 << log_n
    a = oracle.splitmix(GL, 500 + log_n, n * batch)
    m = oracle.splitmix(GL, 510 + log_n, n * batch)
    x = dev(a)
    ops.ntt_(c0, x, log_n, batch)
    X = host(x)
    for b in range(batch):
        assert np.array_equal(X[b * n:(b + 1) * n], oracle.ntt_fast(GL, a[b * n:(b + 1) * n])), b
    y = dev(a)
    ops.ntt_mul_(c0, y, dev(m), log_n, batch)
    assert np.array_equal(host(y), oracle.vec_mul(GL, X, m))
    ops.ntt_(c0, x, log_n, batch, inverse=True)
    assert np.array_equal(host(x), a)
    for env, val in (("RONK_NTT3_MID", "0"), ("RONK_NTT3_T1", "24")):
        os.environ[env] = val
        try:
            c1 = Context(0, torch.cuda.current_stream().cuda_stream)
        finally:
            os.environ.pop(env)
        z = dev(a)
        ops.ntt_(c1, z, log_n, batch)
        c1.sync()
        assert np.array_equal(host(z), X), env
        ops.ntt_(c1, z, log_n, batch, inverse=True)
        c1.sync()
        assert np.array_equal(host(z), a), env
        c1.close()


@pytest.mark.parametrize("log_n,batch", [(17, 32), (18, 17), (19, 8), (25, 1)])
def test_split_transforms_match_oracle_and_the_two_pass_path(log_n, batch):
    """n = R·2^16 (batches of 2^17 … 2^19) and n = 2·2^24: a radix-R register pass, then R tile transforms whose last
    pass interleaves their outputs.  Sampled transforms against the oracle, fused multiply against a separate
    point-wise product, inverse round trip, and bit-for-bit agreement with RONK_NTT3_SPLIT=0."""
    import os
    import torch
    from ronkathon_b200 import Context, ops
    c0 = ctx()
    n = 1 << log_n
    a = ops.splitmix_fill(c0, n * batch, 700 + log_n, GL)
    m = ops.splitmix_fill(c0, n * batch, 710 + log_n, GL)
    ah = host(a)
    x = a.clone()
    ops.ntt_(c0, x, log_n, batch)
    X = host(x)
    for b in sorted({0, batch // 2, batch - 1}):
        assert np.array_equal(X[b * n:(b + 1) * n], oracle.ntt_fast(GL, ah[b * n:(b + 1) * n])), b
    y = a.clone()
    ops.ntt_mul_(c0, y, m, log_n, batch)
    assert np.array_equal(host(y), oracle.vec_mul(GL, X, host(m)))
    ops.ntt_(c0, x, log_n, batch, inverse=True)
    assert np.array_equal(host(x), ah)
    os.environ["RONK_NTT3_SPLIT"] = "0"
    try:
        c1 = Context(0, torch.cuda.current_stream().cuda_stream)
    finally:
        os.environ.pop("RONK_NTT3_SPLIT")
    z = a.clone()
    ops.ntt_(c1, z, log_n, batch)
    c1.sync()
    assert np.array_equal(host(z), X)
    c1.close()
