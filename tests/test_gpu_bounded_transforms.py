"""The zero-padded and clipped transforms behind ronk_poly_mul_u64, on the device.

Every product on the transform path runs two forward transforms that read a[0, da) and b[0, db) as if zero-extended to
n = 2^k words and one inverse that stores only c[0, L), L = da + db - 1.  The padding and the clipping happen inside the
kernels' load and store phases, in instantiations (BOUNDED) and on a dispatch that ronk_ntt_u64 never takes.  Here each
kernel family meets each edge of those bounds:

* every call is laid out in an arena of 0xFFFFFFFFFFFFFFFF words, which is no residue of any test prime: n - da such
  words lie directly behind a (and n - db behind b), so a load that ignores the bound by a word, a line or a row reads
  poison instead of whatever the allocator left there, and guard words lie in front of c and behind c[L), so a store
  past the bound is seen.  Some views start at odd word offsets: 8-byte alignment is all the ABI asks;
* the product is compared bit for bit over all L words with an exact O(L) reference: one operand has five nonzero
  terms (at 0, 1, the middle, and the last two indices), so c = Σ aᵢ·(b shifted by i), in both orientations (the second
  operand's transform carries the fused point-wise multiply).  Dense × dense goes against the oracle's transforms up
  to 2^22 points and against Horner evaluations above;
* the profile names of the launches are asserted, so the family a row claims to cover is the family that ran."""
import os

import numpy as np
import pytest

import oracle
from gpu_util import GL, MONT_PRIMES, ctx, dev, host, s64

pytestmark = pytest.mark.gpu

POISON = -1                      # 0xFFFFFFFFFFFFFFFF as the int64 torch stores
FRONT = 16                       # poison words in front of every view, before the view's own offset
OFFSETS = [(0, 0, 0), (1, 3, 5), (8, 2, 11), (7, 9, 15)]    # word offsets of (a, b, c) past FRONT, cycled over the shapes
TABLE_BUILDS = {"pow_table", "tw2d_gather", "interpass_table", "ntt3_t1", "ntt3_t2"}   # first use of a plan
FIELDS = {"gl": (GL, 7), **{name: (p, g) for name, (p, g, _) in MONT_PRIMES.items()}}


# ---- contexts and launch names ----------------------------------------------------------------------------------------
def context_with(env):
    """A context on the suite's stream created under `env` (the tuning variables are read once, at creation)."""
    import torch
    from ronkathon_b200 import Context
    ctx()
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


def launch_names(c, fn):
    """The profile names of the launches fn() makes on c, without the one-off table builds of a new plan."""
    c.sync()
    c.prof_fetch()
    c.prof_enable(True)
    try:
        fn()
        names = [n for n, _ in c.prof_fetch()]
    finally:
        c.prof_enable(False)
    return [n for n in names if n not in TABLE_BUILDS]


_TWO, _THREE = ["ntt_pass1", "ntt_pass2"], ["ntt3_pass1", "ntt3_pass2", "ntt3_pass3"]


def _inv(names):
    return ["i" + n for n in names]


def expected_launches(field, k, L, env=None):
    """(the two forward transforms' names, the accepted name lists of the inverse) of one product on the transform
    path.  A forward transform is always bounded (da, db < n); the inverse is bounded unless L = n, and then returns to
    the default kernel of its size."""
    env = env or {}
    if k <= 13:
        return ["ntt_single"] * 2, [["intt_single"]]
    ntt3 = field == "gl" and env.get("RONK_NTT3") != "0"
    fwd = _THREE if ntt3 and (k == 24 or (21 <= k <= 23 and env.get("RONK_NTT3_MID") != "0")) else _TWO
    inv = [_inv(fwd)]
    if ntt3 and L == 1 << k:
        if k == 16:
            inv = [["intt16_cluster"], _inv(_TWO)]        # the two-launch path where no 16-CTA cluster can be placed
        elif 17 <= k <= 19:
            inv = [["intt3_split", "intt3_pass2", "intt3_pass3"]]
        elif k == 20:
            inv = [["intt3_a1", "intt3_a2", "intt3_c"]]
        elif k >= 25:
            inv = [["intt3_split"] + _inv(_THREE)]
    return fwd * 2, inv


def assert_family(field, k, L, names, env=None):
    fwd, inv = expected_launches(field, k, L, env)
    assert names[:len(fwd)] == fwd and names[len(fwd):] in inv, (field, k, L, env, names)


# ---- the arena ----------------------------------------------------------------------------------------------------------
def transform_size(L):
    return 1 << max(1, (L - 1).bit_length())


class Arena:
    """One ronk_poly_mul_u64 call inside poisoned device buffers.  a and b are views with n - da (n - db) poison words
    behind them and at least FRONT in front; c is a view of L poison words with FRONT guard words in front and
    n - L + 64 behind.  over = "a" / "b": c starts where that operand does, in one buffer of n + 64 words."""

    def __init__(self, a, b, offsets=(0, 0, 0), over=None):
        import torch
        self.da, self.db = a.numel(), b.numel()
        self.L = self.da + self.db - 1
        self.n = n = transform_size(self.L)
        self.a0, self.b0, self.over = a, b, over
        oa, ob, oc = (FRONT + o for o in offsets)
        full = lambda words: torch.full((words,), POISON, dtype=torch.int64, device="cuda")
        self.A, self.B = full(oa + n + 64), full(ob + n + 64)
        self.a, self.b = self.A[oa:oa + self.da], self.B[ob:ob + self.db]
        self.a.copy_(a)
        self.b.copy_(b)
        if over is None:
            self.C = full(oc + n + 64)
            self.c = self.C[oc:oc + self.L]
        else:
            self.C = self.A if over == "a" else self.B
            start = oa if over == "a" else ob
            self.c = self.C[start:start + self.L]

    def run(self, c, p, g):
        from ronkathon_b200 import _lib
        c.call("ronk_poly_mul_u64", p, g, _lib._ptr(self.a), self.da, _lib._ptr(self.b), self.db, _lib._ptr(self.c))

    def _around(self, buf, view, what, tag):
        lo = (view.data_ptr() - buf.data_ptr()) // 8
        for name, part, base in (("in front of", buf[:lo], 0), ("behind", buf[lo + view.numel():], lo + view.numel())):
            bad = (part != POISON).nonzero()
            assert bad.numel() == 0, f"{tag}: word {int(bad[0]) + base - lo} relative to {what}[0] ({name} {what}) was written"

    def check(self, expected, tag):
        """The poison around a, b and c is intact, the operands are unchanged, and c is `expected` (host words, or a
        device tensor) word for word; the message names the first wrong index."""
        import torch
        ctx().sync()
        tag = f"{tag} da={self.da} db={self.db} L={self.L} n={self.n}"
        self._around(self.C, self.c, "c", tag)
        if self.over != "a":
            self._around(self.A, self.a, "a", tag)
            assert torch.equal(self.a, self.a0), f"{tag}: a was changed"
        if self.over != "b":
            self._around(self.B, self.b, "b", tag)
            assert torch.equal(self.b, self.b0), f"{tag}: b was changed"
        exp = expected if isinstance(expected, torch.Tensor) else dev(expected)
        assert exp.numel() == self.L
        if not torch.equal(self.c, exp):
            i = int((self.c != exp).nonzero()[0])
            got, want = int(self.c[i]) & (1 << 64) - 1, int(exp[i]) & (1 << 64) - 1
            raise AssertionError(f"{tag}: first wrong word c[{i}] = {got:#x}, expected {want:#x} "
                                 f"(i mod 16 = {i % 16}, i mod 256 = {i % 256}, L - i = {self.L - i})")


# ---- operands and exact references ----------------------------------------------------------------------------------------
def dense_operand(p, length, seed):
    """Random residues made on the device, the first and last of them p - 1 and p - 2."""
    from ronkathon_b200 import ops
    t = ops.splitmix_fill(ctx(), length, seed, p)
    t[0] = s64(p - 1)
    t[-1] = s64(p - 2)
    return t


def sparse_operand(p, length, seed):
    """(device tensor, [(index, value)]): nonzero only at 0, 1, the middle and the last two indices."""
    r = [int(v) or 1 for v in oracle.splitmix(p, seed, 2)]
    terms = dict(zip([0, 1, length // 2, length - 2, length - 1], [p - 1, r[0], 1, r[1], p - 1]))
    h = np.zeros(length, dtype=np.uint64)
    for i, v in terms.items():
        h[i] = v
    return dev(h), sorted(terms.items())


def sparse_times_dense(p, terms, sparse_len, d):
    """Σ vᵢ·(d shifted by i): O(L) per term, exact."""
    out = np.zeros(sparse_len + len(d) - 1, dtype=np.uint64)
    for i, v in terms:
        t = d if v == 1 else oracle.vec_mul(p, d, np.full(len(d), v, dtype=np.uint64))
        out[i:i + len(d)] = oracle.poly_add(p, out[i:i + len(d)], t)
    return out


def conv_oracle(p, g, a, b):
    """The product by the convolution theorem with the oracle's transforms."""
    L = len(a) + len(b) - 1
    n = transform_size(L)
    pa, pb = np.zeros(n, np.uint64), np.zeros(n, np.uint64)
    pa[:len(a)], pb[:len(b)] = a, b
    fa, fb = oracle.ntt_fast(p, pa, g=g), oracle.ntt_fast(p, pb, g=g)
    return oracle.ntt_fast(p, oracle.vec_mul(p, fa, fb), inverse=True, g=g)[:L]


def operands(p, da, db, kind, seed):
    """kind a_sparse / b_sparse / dense → (a, b, reference of the product as a function of nothing)."""
    if kind == "a_sparse":
        a, terms = sparse_operand(p, da, seed)
        b = dense_operand(p, db, seed + 1)
        return a, b, lambda: sparse_times_dense(p, terms, da, host(b))
    if kind == "b_sparse":
        a = dense_operand(p, da, seed)
        b, terms = sparse_operand(p, db, seed + 1)
        return a, b, lambda: sparse_times_dense(p, terms, db, host(a))
    return dense_operand(p, da, seed), dense_operand(p, db, seed + 1), None


def check_by_evaluation(p, arena, tag):
    """Dense × dense beyond the oracle's transforms: both end coefficients and c(x) = a(x)·b(x) at four points."""
    a, b, c = host(arena.a0), host(arena.b0), host(arena.c)
    assert int(c[0]) == oracle.mul(p, int(a[0]), int(b[0])) and int(c[-1]) == oracle.mul(p, int(a[-1]), int(b[-1])), tag
    for x in oracle.splitmix(p, 977, 4):
        x = int(x)
        assert oracle.poly_eval_horner(p, c, x) == oracle.mul(p, oracle.poly_eval_horner(p, a, x),
                                                              oracle.poly_eval_horner(p, b, x)), (tag, x)
    return dev(c)   # the arena's own checks then see the poison and the operands


# ---- the grid: kernel family × bound edge --------------------------------------------------------------------------------
def on_transform_path(k, da, db):
    """ronk_poly_mul_u64 transforms when da·db exceeds its estimate of the transforms' cost."""
    return float(da) * float(db) > 1.5 * float(1 << k) * k + 4096.0


def shortest_operand(k, L):
    da = 5
    while not on_transform_path(k, da, L + 1 - da):
        da += 1
    return da


def shapes(k):
    """name → (da, db), every one on the transform path with n/2 < L ≤ n = 2^k.  Rows refer to the two-pass view:
    pass 1 reads x[j1·N2 + j2] (row j1 of N2 words), pass 2 writes X[k1 + N1·k2] (row k2 of N1 words)."""
    n, h = 1 << k, 1 << (k - 1)
    N1, N2 = 1 << (k + 1) // 2, 1 << k // 2
    by_L = lambda da, L: (da, L + 1 - da)
    s = {
        "full": (h + h // 4 + 3, h - h // 4 - 2),                       # L = n: the inverse is unbounded
        "clip1": by_L(h + h // 4 + 3, n - 1),
        "half+1": by_L(h // 2 + 1, h + 1),                              # the largest clip, the largest zero extension
        "short_a": by_L(shortest_operand(k, n - 3), n - 3),
        "short_b": by_L(n - 2 - shortest_operand(k, n - 3), n - 3),
        "halves": (h, h),
        "halves+1": (h + 1, h),
    }
    row = (N1 // 2 - 3) * N2                                            # a mid-range row of the pass-1 view
    for d in (-1, 0, 1):
        s[f"a_row{d:+d}"] = by_L(row + d, n - 8)
    line = (h // 2 & ~15) + 48
    for d in (15, 16, 17):
        s[f"a_line{d % 16}"] = by_L(line + d, n - 5)
    if 21 <= k <= 24:                                                   # rows of the 256-point-tile passes
        for d in (-1, 1):
            s[f"a_256r{d:+d}"] = by_L(n // 4 + 5 * 256 + d, n - 6)
            s[f"a_64kr{d:+d}"] = by_L(n // 4 + 65536 + d, n - 7)
            s[f"L_64kr{d:+d}"] = by_L(n // 3, n - 65536 + d)
    for d in (-1, 1):
        s[f"L_row{d:+d}"] = by_L(n // 3 + 1, n - 3 * N1 + d)
    for d in (15, 1):
        s[f"L_line{d}"] = by_L(n // 3 + 2, n - 64 + d)
    for name, (da, db) in s.items():
        assert h < da + db - 1 <= n and min(da, db) >= 5 and on_transform_path(k, da, db), (k, name, da, db)
    return s


AT_2_24 = ["clip1", "a_row+1", "a_64kr-1", "L_row-1"]
BEYOND = {"full": "a_sparse", "clip1": "a_sparse", "a_row+1": "b_sparse"}   # k ≥ 25: one sparse orientation each
REDUCED = ["full", "clip1", "short_a", "a_row+1", "a_line15", "L_row-1"]    # the moduli with a smaller selection
DENSE_ABOVE_2_18 = {"clip1", "a_row+1", "L_row-1"}
SIZES = {
    "gl": list(range(9, 27)),
    "pbig": [9, 12, 13, 14, 15, 16, 18, 20, 22, 24],
    "babybear": [9, 12, 13, 14, 15, 16, 18, 20, 22, 24],
    "p57": [13, 16, 22],
    "koalabear": [14, 24],
    "p32": [12, 16],
    "gl_g5": [13, 18, 22],
}


def _grid():
    out = []
    for field, ks in SIZES.items():
        for k in ks:
            assert k <= dict(gl=32, **{n: s for n, (_, _, s) in MONT_PRIMES.items()})[field]
            names = list(shapes(k))
            if k >= 25:
                names = list(BEYOND)
            elif k == 24:
                names = AT_2_24
            elif field not in ("gl", "pbig", "babybear"):
                names = REDUCED
            out += [pytest.param(field, k, name, id=f"{field}-2^{k}-{name}") for name in names]
    return out


def kinds_of(k, shape):
    if k >= 25:
        return [BEYOND[shape]]
    dense = k <= 18 or (k <= 22 and shape in DENSE_ABOVE_2_18) or shape == "clip1"
    return ["a_sparse", "b_sparse"] + (["dense"] if dense else [])


@pytest.mark.parametrize("field,k,shape", _grid())
def test_bounded_product(field, k, shape):
    """One (kernel family, bound edge): the product in the arena against the exact reference, in every operand kind the
    size affords, and the profile names of the family the row stands for."""
    p, g = FIELDS[field]
    da, db = shapes(k)[shape]
    offsets = OFFSETS[list(shapes(k)).index(shape) % len(OFFSETS)]
    c = ctx()
    for kind in kinds_of(k, shape):
        tag = f"{field} 2^{k} {shape} {kind}"
        a, b, reference = operands(p, da, db, kind, 1000 * k + 7)
        arena = Arena(a, b, offsets)
        arena.run(c, p, g)
        if reference is not None:
            exp = reference()
        elif k <= 22:
            exp = conv_oracle(p, g, host(a), host(b))
        else:
            exp = check_by_evaluation(p, arena, tag)
        arena.check(exp, tag)
    names = launch_names(c, lambda: arena.run(c, p, g))      # the same call again, profiled
    assert_family(field, k, arena.L, names)
    arena.check(exp, tag + " (profiled)")


# ---- the same edges under the other tile shapes and launch modes -------------------------------------------------------------
ENVS = [{"RONK_TILE_ADAPT": "0"},    # 2^14 / 2^13 tiles at every size: the 512- and 256-thread bounded instantiations
        {"RONK_NTT3_MID": "0"},      # Goldilocks 2^21 … 2^23 on the bounded two-pass kernel
        {"RONK_NTT3": "0"},          # Goldilocks 2^24 on it as well
        {"RONK_TW_TABLE": "1"},      # pass 1 multiplies by the tabulated inter-pass twiddles
        {"RONK_PDL": "0"}]           # pass 2 launched without programmatic dependent launch


@pytest.mark.parametrize("env", ENVS, ids=["=".join(*e.items()) for e in ENVS])
def test_other_configurations_agree_bit_for_bit(env):
    """A context created under `env` returns the default context's words (themselves checked by the grid) on one clip, one
    row edge and one line edge at 2^16, 2^20, 2^22 and 2^24, with the poison and the guards intact."""
    c1 = context_with(env)
    try:
        for field in ("gl", "pbig"):
            p, g = FIELDS[field]
            for k in (16, 20, 22, 24):
                for shape in ("clip1", "a_row+1", "L_line15"):
                    da, db = shapes(k)[shape]
                    a, b = dense_operand(p, da, 50 + k), dense_operand(p, db, 51 + k)
                    ref, arena = Arena(a, b, (3, 5, 1)), Arena(a, b, (3, 5, 1))
                    ref.run(ctx(), p, g)
                    names = launch_names(c1, lambda: arena.run(c1, p, g))
                    assert_family(field, k, arena.L, names, env)
                    c1.sync()
                    arena.check(ref.c, f"{env} {field} 2^{k} {shape}")
    finally:
        c1.close()


# ---- the output over an operand ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("over", ["a", "b"])
@pytest.mark.parametrize("field,k", [("gl", 15), ("gl", 18), ("gl", 20), ("gl", 22), ("gl", 24), ("pbig", 16), ("pbig", 22)],
                         ids=lambda v: v if isinstance(v, str) else f"2^{v}")
def test_output_may_start_where_an_operand_does(field, k, over):
    """c = a or c = b on every transform family: both operands are consumed before the last launch writes c.  The operand
    under c is the dense one; the words between its end and n are poison until c covers them."""
    p, g = FIELDS[field]
    h = 1 << (k - 1)
    da, db = h + 3, h - 11
    a, b, reference = operands(p, da, db, "b_sparse" if over == "a" else "a_sparse", 300 + k)
    exp = reference()
    arena = Arena(a, b, (5, 2, 0), over=over)
    names = launch_names(ctx(), lambda: arena.run(ctx(), p, g))
    assert_family(field, k, arena.L, names)
    arena.check(exp, f"{field} 2^{k} c over {over}")


# ---- the other two product paths in the same arena --------------------------------------------------------------------------
CRT = {"f101-2^14x2^14": (101, 2, 1 << 14, 1 << 14, 0), "2^64-59-3000x2000": ((1 << 64) - 59, 2, 3000, 2000, 3),
       "2^64-59-2^19": ((1 << 64) - 59, 2, (1 << 19) + 3, (1 << 19) - 7, 3)}


@pytest.mark.parametrize("case", list(CRT))
def test_multi_modular_path_in_the_arena(case):
    """The multi-modular path (no power-of-two root in p - 1): its bounded transforms read the raw operands where p is
    below the auxiliary primes, crt_reduce reads them where it is above."""
    p, g, da, db, reductions = CRT[case]
    c = context_with({"RONK_CRT_MUL_MIN": "1"})
    try:
        for kind in ("a_sparse", "b_sparse"):
            a, b, reference = operands(p, da, db, kind, 70)
            arena = Arena(a, b, (1, 7, 3))
            names = launch_names(c, lambda: arena.run(c, p, g))
            assert names[-1] == "crt_combine" and names.count("crt_reduce") == reductions, names
            assert "poly_mul_schoolbook" not in names
            c.sync()
            exp = oracle.poly_mul(p, host(a), host(b)) if da * db <= 1 << 24 else reference()
            arena.check(exp, f"{case} {kind}")
    finally:
        c.close()


@pytest.mark.parametrize("da,db", [(1, 5000), (5000, 1), (257, 129)])
def test_schoolbook_kernel_in_the_arena(da, db):
    """g = 0: one thread per coefficient of c, no transform."""
    a, b = dev(oracle.splitmix(GL, 80, da)), dev(oracle.splitmix(GL, 81, db))
    arena = Arena(a, b, (3, 1, 9))
    names = launch_names(ctx(), lambda: arena.run(ctx(), GL, 0))
    assert names == ["poly_mul_schoolbook"]
    arena.check(oracle.poly_mul(GL, host(a), host(b)), f"schoolbook {da}x{db}")
