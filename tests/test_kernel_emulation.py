"""CPU emulation of the CUDA kernel logic (tests/emu/ntt_emu.cpp compiles the product's own
field.cuh / ntt_kernel.cuh for the host and runs the tile phases thread by thread).  Checks index
maps, round schedule, twiddle tables and field arithmetic against the oracle.  The emulator is
test infrastructure; the product library never executes on the CPU."""
import ctypes as C

import numpy as np
import pytest

import field_corpus as fc
import oracle
from gpu_util import BABYBEAR, PBIG

GL = oracle.GOLDILOCKS
P64 = C.POINTER(C.c_uint64)


@pytest.fixture(scope="module")
def emu():
    return fc.host_twin()


def _ptr(a):
    return a.ctypes.data_as(P64) if a is not None else None


def emu_ntt(emu, p, g, data, log_n, batch=1, inverse=False, mul=None, tile_cap=12, tiles=(13, 13)):
    d = np.ascontiguousarray(data, dtype=np.uint64).copy()
    m = None if mul is None else np.ascontiguousarray(mul, dtype=np.uint64)
    rc = emu.emu_ntt(p, g, _ptr(d), _ptr(m), log_n, batch, int(inverse), tile_cap, tiles[0], tiles[1])
    assert rc == 0
    return d


_EXTRA_MONT = [p for p in fc.MONT_PRIMES.values() if p not in (GL, 101, 17, 127, 0xFFFFFFFFFFFFFFC5, 0x7FFFFFFFFFFFFFE7,
                                                                4179340454199820289)]


@pytest.mark.parametrize("p,force_mont", [(GL, 0), (GL, 1), (101, 0), (17, 0), (127, 0),
                                          (0xFFFFFFFFFFFFFFC5, 0), (0x7FFFFFFFFFFFFFE7, 0), (4179340454199820289, 0)]
                         + [(p, 0) for p in _EXTRA_MONT])
def test_field_policies_match_oracle(emu, p, force_mont):
    """The host twin of both field policies on the structured corpus of tests/field_corpus.py (every pair of its
    values) plus random odd words, against the oracle."""
    rng = np.random.default_rng(5)
    sa, sb = fc.gl_pairs() if p == GL else fc.mont_pairs(p)
    a = [int(x) for x in sa] + [int(v) % p for v in rng.integers(0, 2**63, 4000, dtype=np.uint64) * 2 + 1]
    b = [int(y) for y in sb] + [int(v) % p for v in rng.integers(0, 2**63, 4000, dtype=np.uint64) * 2 + 1]
    a, b = np.array(a, dtype=np.uint64), np.array(b, dtype=np.uint64)
    out = np.empty_like(a)
    for op, fn in ((0, oracle.add), (1, oracle.sub), (2, oracle.mul)):
        assert emu.emu_field_op(p, op, _ptr(a), _ptr(b), _ptr(out), len(a), force_mont) == 0
        exp = np.array([fn(p, int(x), int(y)) for x, y in zip(a, b)], dtype=np.uint64)
        assert np.array_equal(out, exp), op
    assert emu.emu_field_op(p, 3, _ptr(a), _ptr(b), _ptr(out), len(a), force_mont) == 0
    assert np.array_equal(out, np.array([oracle.neg(p, int(x)) for x in a], dtype=np.uint64))


def test_goldilocks_shift_twiddles(emu):
    w16 = oracle.root_of_unity(GL, 16)
    w16i = oracle.inverse(GL, w16)
    out = np.empty(16, dtype=np.uint64)
    for a in list(fc.gl_values()) + [int(v) for v in oracle.splitmix(GL, 9, 50)]:
        emu.emu_gl_w16(a, _ptr(out))
        for e in range(8):
            assert int(out[e]) == oracle.mul(GL, a, oracle.pow_(GL, w16, e)), (a, e)
            assert int(out[8 + e]) == oracle.mul(GL, a, oracle.pow_(GL, w16i, e)), (a, e)


@pytest.mark.parametrize("S", range(192))
def test_goldilocks_host_mul_pow2_on_the_shift_corpus(S):
    """The host twin of mul_pow2<S> on the inputs the device harness gets for S, against Python integers."""
    x = np.array(fc.gl_shift_inputs(S), dtype=np.uint64)
    assert np.array_equal(fc.host_gl_shift(0, S, False, x), fc.exact("mul", GL, x, [pow(2, S, GL)] * len(x))), S


@pytest.mark.parametrize("inverse", [False, True])
@pytest.mark.parametrize("e", range(8))
def test_goldilocks_host_w16_sub_on_the_shift_corpus(e, inverse):
    """w16_sub<E, INV>(a, b) = (a − b)·ω16^±E, with a − b (or b − a, where the sign is folded into the subtraction)
    running over the shift corpus of its S."""
    a, b = fc.gl_w16_sub_operands(fc.w16_shift(e, inverse))
    w = pow(oracle.root_of_unity(GL, 16), -e if inverse else e, GL)
    assert np.array_equal(fc.host_gl_shift(1, e, inverse, a, b), fc.exact("mul", GL, fc.exact("sub", GL, a, b),
                                                                            [w] * len(a)))


def test_corpus_reaches_every_case():
    """Every case the derivations in field.cuh name is reached at least MIN_HITS times by the corpus handed to its
    op; a case fewer inputs below p reach is listed with its size in field_corpus and must be reached exactly that
    often (the corpus holds all of it).  The test primes are prime."""
    def check(counts, expected, small, what):
        for case in expected:
            need, _ = small.get(case, (None, None))
            got = counts.get(case, 0)
            if need is None:
                assert got >= fc.MIN_HITS, (what, case, got)
            else:
                assert got == need, (what, case, got, need)
    a, b = fc.gl_pairs()
    check(fc.count_cases(fc.gl_add_cases, a, b), ("sum_lt_p", "sum_in_p_2_64", "sum_carries_2_64"), {}, "gl add")
    check(fc.count_cases(fc.sub_cases, a, b), ("a_ge_b", "a_lt_b"), {}, "gl sub")
    check(fc.count_cases(fc.gl_mul_cases, a, b), fc.GL_MUL_CASES, fc.GL_MUL_SMALL, "gl mul")
    for S in range(192):
        counts = fc.count_cases(lambda x: fc.gl_shift_cases(S, x), fc.gl_shift_inputs(S))
        small = {c: v for (s, c), v in fc.GL_SHIFT_SMALL.items() if s == S}
        check(counts, fc.SHIFT_CASES[fc.gl_shift_form(S)], small, f"mul_pow2<{S}>")
    for e in range(8):   # w16_sub hands mul_pow2 the difference: the same inputs, reached through the subtraction
        for inverse in (False, True):
            S = fc.w16_shift(e, inverse)
            a, b = fc.gl_w16_sub_operands(S)
            d = fc.exact("sub", GL, b, a) if S >= 96 else fc.exact("sub", GL, a, b)
            assert set(int(v) for v in d) >= set(fc.gl_shift_inputs(S)), (e, inverse)
    for name, p in fc.MONT_PRIMES.items():
        assert fc.is_prime(p), name
        a, b = fc.mont_pairs(p)
        if p < fc.EXHAUSTIVE_BELOW:      # every pair of residues: each case holds all the inputs it can
            assert len(a) == p * p
            continue
        check(fc.count_cases(lambda x, y: fc.mont_add_cases(p, x, y), a, b), fc.mont_add_expected_cases(p), {}, name)
        check(fc.count_cases(fc.sub_cases, a, b), ("a_ge_b", "a_lt_b"), {}, name)
        check(fc.count_cases(lambda x, y: fc.redc_cases(p, x, y), a, b), fc.mont_redc_expected_cases(p), {}, name)


def test_swizzle_is_conflict_free(emu):
    for tile_log in (9, 10, 12, 14):
        for wb in range(0, tile_log - 3):
            assert emu.emu_swizzle_worst_conflict(tile_log, wb) == 1, (tile_log, wb)


@pytest.mark.parametrize("p,log_n", [(101, 1), (101, 2), (17, 1), (17, 2), (17, 3), (17, 4), (127, 1)])
def test_emulated_small_moduli_match_reference_fft(emu, p, log_n):
    g = oracle.generator(p)
    n = 1 << log_n
    rng = np.random.default_rng(log_n)
    for batch in (1, 3, 37):
        a = rng.integers(0, p, n * batch).astype(np.uint64)
        X = emu_ntt(emu, p, g, a, log_n, batch)
        for b in range(batch):
            assert np.array_equal(X[b * n:(b + 1) * n], oracle.fft(p, a[b * n:(b + 1) * n]))
        back = emu_ntt(emu, p, g, X, log_n, batch, inverse=True)
        assert np.array_equal(back, a)
        for b in range(batch):
            assert np.array_equal(back[b * n:(b + 1) * n], oracle.ifft(p, X[b * n:(b + 1) * n]))


def test_emulated_reference_kat(emu, kats):
    k = kats["polynomial"]
    X = emu_ntt(emu, 101, 2, k["a"], 2)
    assert list(X) == k["fft_a"]
    assert list(emu_ntt(emu, 101, 2, X, 2, inverse=True)) == k["a"]


@pytest.mark.parametrize("log_n", list(range(1, 15)))
@pytest.mark.parametrize("mont", [False, True])
def test_emulated_goldilocks_single_pass(emu, log_n, mont):
    n = 1 << log_n
    g = 7
    p = GL
    if mont:  # a different generator routes Goldilocks through the generic Montgomery policy
        g = oracle.pow_(GL, 7, 5)
    batch = 3 if log_n <= 12 else 1
    a = oracle.splitmix(p, 100 + log_n, n * batch)
    X = emu_ntt(emu, p, g, a, log_n, batch)
    for b in range(batch):
        assert np.array_equal(X[b * n:(b + 1) * n], oracle.ntt_fast(p, a[b * n:(b + 1) * n], g=g)), b
    assert np.array_equal(emu_ntt(emu, p, g, X, log_n, batch, inverse=True), a)


def test_emulated_adaptive_tiles_config2(emu):
    """The tile shapes run_ntt() picks for one 2^20 transform (config 2) on a 132-SM GPU: 2^12 / 2^11."""
    a = oracle.splitmix(GL, 42, 1 << 20)
    X = emu_ntt(emu, GL, 7, a, 20, tiles=(12, 11))
    assert np.array_equal(X, oracle.ntt_fast(GL, a))
    assert np.array_equal(emu_ntt(emu, GL, 7, X, 20, inverse=True, tiles=(12, 11)), a)


def test_emulated_golden_vectors(emu, gold64):
    assert list(emu_ntt(emu, GL, 7, list(range(1, 9)), 3)) == gold64["ntt8_1to8"]
    a = oracle.splitmix(GL, 42, 1024)
    assert list(emu_ntt(emu, GL, 7, a, 10)) == gold64["ntt_2_10_full"]


@pytest.mark.parametrize("tiles", [(13, 13), (14, 14), (13, 14), (14, 13), (12, 12), (12, 11), (13, 12), (11, 11)])
@pytest.mark.parametrize("log_n,batch", [(14, 2), (15, 1), (16, 2), (17, 1), (18, 1)])
def test_emulated_goldilocks_two_pass(emu, log_n, batch, tiles):
    n = 1 << log_n
    a = oracle.splitmix(GL, 42, n * batch)
    X = emu_ntt(emu, GL, 7, a, log_n, batch, tiles=tiles)
    for b in range(batch):
        assert np.array_equal(X[b * n:(b + 1) * n], oracle.ntt_fast(GL, a[b * n:(b + 1) * n]))
    assert np.array_equal(emu_ntt(emu, GL, 7, X, log_n, batch, inverse=True, tiles=tiles), a)


def test_emulated_two_pass_generic_and_fused_mul(emu, gold64):
    log_n, n = 16, 1 << 16
    a, b = oracle.splitmix(GL, 42, n), oracle.splitmix(GL, 43, n)
    g5 = oracle.pow_(GL, 7, 5)
    assert np.array_equal(emu_ntt(emu, GL, g5, a, log_n), oracle.ntt_fast(GL, a, g=g5))
    # fused point-wise multiply in the last stage, then inverse: the cyclic convolution golden
    A = emu_ntt(emu, GL, 7, a, log_n)
    AB = emu_ntt(emu, GL, 7, b, log_n, mul=A)
    c = emu_ntt(emu, GL, 7, AB, log_n, inverse=True)
    gsum = gold64["cyclic_conv_2_16_seed42_seed43"]
    assert int(c[0]) == gsum["first"] and int(c[1]) == gsum["second"] and int(c[-1]) == gsum["last"]
    assert int(np.sum(c, dtype=np.uint64)) == gsum["sum_mod_2_64"]
    assert int(np.bitwise_xor.reduce(c)) == gsum["xor"]
    # single-pass fused multiply
    a10, b10 = a[:1024].copy(), b[:1024].copy()
    A10 = emu_ntt(emu, GL, 7, a10, 10)
    exp = np.array([oracle.mul(GL, int(x), int(y)) for x, y in zip(oracle.ntt_fast(GL, b10), A10)], dtype=np.uint64)
    assert np.array_equal(emu_ntt(emu, GL, 7, b10, 10, mul=A10), exp)
    # Montgomery fused multiply in the pass-2 store, with the preferred and the adapted tile shapes
    for p, g, lg in ((PBIG, 3, 16), (BABYBEAR, 31, 18)):
        x, m = oracle.splitmix(p, 44, 1 << lg), oracle.splitmix(p, 45, 1 << lg)
        x[0], m[1] = p - 1, p - 1
        exp = oracle.vec_mul(p, oracle.ntt_fast(p, x, g=g), m)
        for tiles in ((14, 13), (12, 11)):
            assert np.array_equal(emu_ntt(emu, p, g, x, lg, mul=m, tiles=tiles), exp), (p, lg, tiles)


def emu_ntt_bounded(emu, p, g, src, dst_len, log_n, inverse=False, mul=None, tile_cap=12, tiles=(13, 13)):
    s = np.ascontiguousarray(src, dtype=np.uint64)
    d = np.full(dst_len + 3, 0xDEADBEEF, dtype=np.uint64)   # 3 guard words past the clipped output
    m = None if mul is None else np.ascontiguousarray(mul, dtype=np.uint64)
    rc = emu.emu_ntt_bounded(p, g, _ptr(s), len(s), _ptr(d), dst_len, _ptr(m), log_n, int(inverse), tile_cap, tiles[0],
                             tiles[1])
    assert rc == 0 and np.all(d[dst_len:] == 0xDEADBEEF), "wrote past dst_len"
    return d[:dst_len]


@pytest.mark.parametrize("p,g,log_n,src_len,dst_len", [
    (GL, 7, 3, 5, 8), (GL, 7, 10, 1, 1024), (GL, 7, 12, 3000, 4000), (GL, 7, 13, 4097, 8191),
    (GL, 7, 14, 8192, 16383), (GL, 7, 15, 20001, 32768), (GL, 7, 16, 32768, 65535), (GL, 7, 16, 65536, 17),
    (17, 14, 4, 7, 13), (GL, 49, 14, 5000, 9000),
    (BABYBEAR, 31, 15, 20001, 32768), (BABYBEAR, 31, 16, 65536, 40001), (BABYBEAR, 31, 17, 70000, 131071),
    (BABYBEAR, 31, 18, 131073, 262144), (PBIG, 3, 15, 32768, 20000), (PBIG, 3, 16, 30001, 65536),
    (PBIG, 3, 17, 131072, 99999), (PBIG, 3, 18, 200001, 262143),
])
@pytest.mark.parametrize("variant", [0, 1, 2])
def test_emulated_bounded_out_of_place_transform(emu, p, g, log_n, src_len, dst_len, variant):
    """poly_mul's transforms: a short operand is zero-extended inside the load phase and the output is clipped
    inside the store phase (ntt_device_bounded).  Same values as padding / slicing around the plain transform,
    nothing written past dst_len, the source untouched."""
    n = 1 << log_n
    src = oracle.splitmix(p, 900 + log_n, src_len)
    padded = np.concatenate([src, np.zeros(n - src_len, dtype=np.uint64)])
    emu.emu_set_variant(variant)   # 0: the kernel's per-mode choice of phase formulation, 1 / 2: force either
    try:
        _bounded_checks(emu, p, g, log_n, src, padded, dst_len)
    finally:
        emu.emu_set_variant(0)


def _bounded_checks(emu, p, g, log_n, src, padded, dst_len):
    n = 1 << log_n
    for inverse in (False, True):
        ref = oracle.ntt_fast(p, padded, inverse=inverse, g=g)
        keep = src.copy()
        got = emu_ntt_bounded(emu, p, g, src, dst_len, log_n, inverse=inverse)
        assert np.array_equal(got, ref[:dst_len]) and np.array_equal(src, keep), (log_n, inverse)
    # with the fused point-wise multiply (the second transform of poly_mul)
    mul = oracle.splitmix(p, 77, n)
    got = emu_ntt_bounded(emu, p, g, src, n, log_n, mul=mul)
    assert np.array_equal(got, oracle.vec_mul(p, oracle.ntt_fast(p, padded, g=g), mul))


# ---- the specialised 4096-point-per-tile kernel (ntt12_kernel.cuh) ------------------------------------------
@pytest.mark.parametrize("mode,lc", [(1, 2), (2, 1), (2, 2)])
def test_additive_layout_is_injective_and_conflict_free(emu, mode, lc):
    """word(e) of ntt12_kernel.cuh: injective on the tile, inside TILE_SLOTS, and every shared-memory access of
    every phase (tile load, three radix-16 rounds, un-bit-reversing store) is conflict-free: 8 lanes on eight
    16-byte banks for the 128-bit accesses, 16 lanes on sixteen 8-byte banks for the pass-1 store's 64-bit reads."""
    assert emu.emu_layout12_worst_conflict(mode, lc) == 1


@pytest.mark.parametrize("log_n,tiles,table", [(24, (14, 13), 1), (24, (14, 13), 0), (23, (14, 12), 1)])
def test_fast12_two_pass_transform_matches_oracle(emu, log_n, tiles, table):
    """2^24 = 4096 × 4096 with the inter-pass twiddle table (both passes through the specialised kernel) and without
    it (pass 1 generic with stepped twiddles, pass 2 specialised), and 2^23 = 4096 × 2048 (pass 1 specialised, pass 2
    generic): forward against the oracle, then the inverse back to the input."""
    a = oracle.splitmix(GL, 42, 1 << log_n)
    emu.emu_set_tw_table(table)
    try:
        before = emu.emu_fast12_tiles()
        X = emu_ntt(emu, GL, 7, a, log_n, tiles=tiles)
        assert emu.emu_fast12_tiles() > before, "the specialised path was not taken"
        assert np.array_equal(X, oracle.ntt_fast(GL, a))
        assert np.array_equal(emu_ntt(emu, GL, 7, X, log_n, inverse=True, tiles=tiles), a)
    finally:
        emu.emu_set_tw_table(0)


def test_fast12_agrees_with_generic_kernel_and_fused_multiply(emu):
    """Same 2^24 transform through the generic tile kernel (fast12 off) and the specialised one, plus the fused
    point-wise multiply of pass 2 (NTT_FLAG_MUL → the FMUL instantiation)."""
    a, b = oracle.splitmix(GL, 5, 1 << 24), oracle.splitmix(GL, 6, 1 << 24)
    emu.emu_set_tw_table(1)
    try:
        fast = emu_ntt(emu, GL, 7, a, 24, tiles=(14, 13), mul=b)
        emu.emu_set_fast12(0)
        slow = emu_ntt(emu, GL, 7, a, 24, tiles=(14, 13), mul=b)
    finally:
        emu.emu_set_fast12(1)
        emu.emu_set_tw_table(0)
    assert np.array_equal(fast, slow)
    assert np.array_equal(fast, oracle.vec_mul(GL, oracle.ntt_fast(GL, a), b))


# ---- the three-pass 2^24 transform (ntt3_kernel.cuh) --------------------------------------------------------
def test_three_pass_tile_layout_is_conflict_free(emu):
    assert emu.emu_layout3_worst_conflict() == 1


@pytest.mark.parametrize("t1_table", [0, 1])
def test_three_pass_2_24_matches_oracle_forward_fused_multiply_and_inverse(emu, t1_table):
    """2^24 = 256·256·256: pass 1 (ω_n^(k1·m) twiddle stepped, or from the n-word table), pass 2 (64 Ki-entry table),
    pass 3 (contiguous axis, natural-order output), the fused point-wise multiply of the last pass, and the inverse
    (n^-1 in the pass-2 table) — the kernel's own functions on the CPU, against the oracle."""
    a, b = oracle.splitmix(GL, 42, 1 << 24), oracle.splitmix(GL, 43, 1 << 24)
    X = a.copy()
    assert emu.emu_ntt3(_ptr(X), None, 24, 1, 0, t1_table) == 0
    ref = oracle.ntt_fast(GL, a)
    assert np.array_equal(X, ref)
    if t1_table == 0:
        Y = a.copy()
        assert emu.emu_ntt3(_ptr(Y), _ptr(b), 24, 1, 0, 0) == 0
        assert np.array_equal(Y, oracle.vec_mul(GL, ref, b))
    assert emu.emu_ntt3(_ptr(X), None, 24, 1, 1, t1_table) == 0
    assert np.array_equal(X, a)


def test_two_pass_256_tiles_2_16_batch(emu):
    """2^16 = 256·256 (BASELINE config 5's transform length) through the same tile functions, a batch of 5: forward
    against the oracle per transform, fused multiply, inverse."""
    n, batch = 1 << 16, 5
    a = oracle.splitmix(GL, 9, n * batch)
    m = oracle.splitmix(GL, 10, n * batch)
    X = a.copy()
    assert emu.emu_ntt3(_ptr(X), None, 16, batch, 0, 0) == 0
    for b in range(batch):
        assert np.array_equal(X[b * n:(b + 1) * n], oracle.ntt_fast(GL, a[b * n:(b + 1) * n])), b
    Y = a.copy()
    assert emu.emu_ntt3(_ptr(Y), _ptr(m), 16, batch, 0, 0) == 0
    assert np.array_equal(Y, oracle.vec_mul(GL, X, m))
    assert emu.emu_ntt3(_ptr(X), None, 16, batch, 1, 0) == 0
    assert np.array_equal(X, a)


@pytest.mark.parametrize("log_n", [16, 20])
def test_one_group_per_thread_flavour_of_the_tile_passes(emu, log_n):
    """Grids that do not fill the GPU run the same tile functions with 256 threads and one radix-16 group each
    (switch bit 1 of the emulator): forward against the oracle, inverse round trip."""
    n = 1 << log_n
    a = oracle.splitmix(GL, 31 + log_n, n)
    X = a.copy()
    assert emu.emu_ntt3(_ptr(X), None, log_n, 1, 0, 2) == 0
    assert np.array_equal(X, oracle.ntt_fast(GL, a))
    assert emu.emu_ntt3(_ptr(X), None, log_n, 1, 1, 2) == 0
    assert np.array_equal(X, a)


def test_2_16_cluster_formulation_in_place(emu):
    """ntt16c_kernel's data flow on the host: pass 2 of the sixteen tiles writes into the receive buffers of the
    sixteen pass-3 CTAs (distributed shared memory on the GPU), pass 3 runs out of them, in place on the operand —
    a batch of 3 against the oracle, fused multiply, inverse."""
    n, batch = 1 << 16, 3
    a = oracle.splitmix(GL, 51, n * batch)
    m = oracle.splitmix(GL, 52, n * batch)
    X = a.copy()
    assert emu.emu_ntt16_cluster(_ptr(X), None, batch, 0) == 0
    for b in range(batch):
        assert np.array_equal(X[b * n:(b + 1) * n], oracle.ntt_fast(GL, a[b * n:(b + 1) * n])), b
    Y = a.copy()
    assert emu.emu_ntt16_cluster(_ptr(Y), _ptr(m), batch, 0) == 0
    assert np.array_equal(Y, oracle.vec_mul(GL, X, m))
    assert emu.emu_ntt16_cluster(_ptr(X), None, batch, 1) == 0
    assert np.array_equal(X, a)


@pytest.mark.parametrize("log_n,batch", [(17, 2), (18, 1), (19, 2), (25, 1)])
def test_split_transforms_register_first_pass_and_interleaving_last_pass(emu, log_n, batch):
    """n = R·2^16 (2^17 … 2^19) and n = 2·2^24: a radix-R register pass with the twiddles ω_n^(k1·m), then R tile transforms
    whose last pass writes X[k1 + R·k'] as contiguous 16-word runs: forward against the oracle, fused multiply, inverse."""
    n = 1 << log_n
    a = oracle.splitmix(GL, 40 + log_n, n * batch)
    m = oracle.splitmix(GL, 50 + log_n, n * batch)
    X = a.copy()
    assert emu.emu_ntt3(_ptr(X), None, log_n, batch, 0, 1) == 0
    for b in range(batch):
        assert np.array_equal(X[b * n:(b + 1) * n], oracle.ntt_fast(GL, a[b * n:(b + 1) * n])), b
    if log_n < 25:
        Y = a.copy()
        assert emu.emu_ntt3(_ptr(Y), _ptr(m), log_n, batch, 0, 1) == 0
        assert np.array_equal(Y, oracle.vec_mul(GL, X, m))
    assert emu.emu_ntt3(_ptr(X), None, log_n, batch, 1, 1) == 0
    assert np.array_equal(X, a)


@pytest.mark.parametrize("log_n,batch", [(16, 3), (20, 2), (21, 2)])
def test_shared_multiplier_of_a_batch(emu, log_n, batch):
    """The fused point-wise multiply with ONE n-word multiplier for the whole batch (mask n - 1 on the multiplier
    index): what the distributed transform uses to put its twiddle column into the local transforms' store phase."""
    n = 1 << log_n
    a = oracle.splitmix(GL, 80 + log_n, n * batch)
    m = oracle.splitmix(GL, 90 + log_n, n)
    X = a.copy()
    assert emu.emu_ntt3_shared_mul(_ptr(X), _ptr(m), log_n, batch) == 0
    for b in range(batch):
        assert np.array_equal(X[b * n:(b + 1) * n], oracle.vec_mul(GL, oracle.ntt_fast(GL, a[b * n:(b + 1) * n]), m)), b


@pytest.mark.parametrize("log_n,t1_table", [(21, 0), (21, 1), (22, 1), (22, 0), (23, 1)])
def test_mid_sizes_first_pass_of_32_64_128_points(emu, log_n, t1_table):
    """2^21 … 2^23: the first pass is an R = 2^(log n - 16)-point transform (radix R/16, then radix 16; 16·16/R of them side by
    side in a tile), passes 2 and 3 are those of 2^24 with R in the strides: forward against the oracle, fused
    multiply, inverse; first-pass twiddles stepped (0) or from the n-word table (1)."""
    n = 1 << log_n
    a = oracle.splitmix(GL, 60 + log_n, n)
    m = oracle.splitmix(GL, 70 + log_n, n)
    X = a.copy()
    assert emu.emu_ntt3(_ptr(X), None, log_n, 1, 0, t1_table) == 0
    assert np.array_equal(X, oracle.ntt_fast(GL, a))
    Y = a.copy()
    assert emu.emu_ntt3(_ptr(Y), _ptr(m), log_n, 1, 0, t1_table) == 0
    assert np.array_equal(Y, oracle.vec_mul(GL, X, m))
    assert emu.emu_ntt3(_ptr(X), None, log_n, 1, 1, t1_table) == 0
    assert np.array_equal(X, a)


@pytest.mark.parametrize("t1_table", [0, 1])
def test_2_20_as_sixteen_interleaved_2_16_transforms_plus_radix16(emu, t1_table):
    """2^20 (BASELINE config 2) = passes A1 / A2 of the tile kernel on 16 interleaved 2^16-point transforms + the
    register-only radix-16 pass C: a batch of 2 against the oracle per transform, fused multiply, inverse; pass A2's
    twiddle stepped (0) or from the n-word table (1)."""
    n, batch = 1 << 20, 2
    a = oracle.splitmix(GL, 19, n * batch)
    m = oracle.splitmix(GL, 20, n * batch)
    X = a.copy()
    assert emu.emu_ntt3(_ptr(X), None, 20, batch, 0, t1_table) == 0
    for b in range(batch):
        assert np.array_equal(X[b * n:(b + 1) * n], oracle.ntt_fast(GL, a[b * n:(b + 1) * n])), b
    Y = a.copy()
    assert emu.emu_ntt3(_ptr(Y), _ptr(m), 20, batch, 0, t1_table) == 0
    assert np.array_equal(Y, oracle.vec_mul(GL, X, m))
    assert emu.emu_ntt3(_ptr(X), None, 20, batch, 1, t1_table) == 0
    assert np.array_equal(X, a)


def test_three_pass_bounded_source_and_destination(emu):
    """The polynomial product's use of the 2^24 transform: the source is shorter than n (zero-extended inside the first
    pass's loads), the destination buffer is shorter than n (the last pass stores dst[0, dst_len) only — the words
    after it must stay untouched)."""
    n = 1 << 24
    src_len, dst_len = (1 << 23) + 12345, n - 54321
    a = oracle.splitmix(GL, 77, src_len)
    full = np.zeros(n, dtype=np.uint64)
    full[:src_len] = a
    ref = oracle.ntt_fast(GL, full)
    guard = np.uint64(0xDEADBEEFCAFEF00D)
    dst = np.full(dst_len + 1024, guard, dtype=np.uint64)
    assert emu.emu_ntt3_bounded(_ptr(a), src_len, _ptr(dst), dst_len, None, 0) == 0
    assert np.array_equal(dst[:dst_len], ref[:dst_len])
    assert np.all(dst[dst_len:] == guard)
    back = np.full(src_len + 64, guard, dtype=np.uint64)
    assert emu.emu_ntt3_bounded(_ptr(ref), n, _ptr(back), src_len, None, 1) == 0
    assert np.array_equal(back[:src_len], a)
    assert np.all(back[src_len:] == guard)
