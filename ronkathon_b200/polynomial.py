"""Host-side mirror of `Polynomial<B: Basis, F: FiniteField, const D: usize>`
(src/polynomial/mod.rs, src/polynomial/arithmetic.rs).  Coefficients live in a numpy uint64 array
of canonical residues; every operation is a call into libronk_b200.so (CUDA kernels) — no field
arithmetic happens in Python.  `D` is `len(coefficients)`.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from ._lib import RonkPanic


class Monomial:
    """Basis marker (polynomial/mod.rs:48-55)."""


class Lagrange:
    """Basis marker (polynomial/mod.rs:57-72); nodes are ω_n^i and stay implicit (delta D6)."""


def _coeffs(field, values) -> np.ndarray:
    vals = [int(getattr(v, "value", v)) % field.ORDER for v in values]
    return np.array(vals, dtype=np.uint64)


class Polynomial:
    def __init__(self, coefficients, field, basis=Monomial):
        self.field = field
        self.basis = basis
        self.coefficients = _coeffs(field, coefficients)
        if basis is Lagrange:  # Lagrange::new asserts (ORDER-1) % n == 0 (polynomial/mod.rs:361)
            if len(self.coefficients) == 0 or (field.ORDER - 1) % len(self.coefficients) != 0:
                raise RonkPanic(1, "assertion failed: (ORDER - 1) % n == 0")

    # -- helpers -----------------------------------------------------------------------------
    @property
    def p(self):
        return self.field.ORDER

    @property
    def g(self):
        return self.field.PRIMITIVE_ELEMENT.value

    def _ctx(self):
        return _lib.default_context()

    def _like(self, arr, basis=None):
        out = Polynomial.__new__(Polynomial)
        out.field, out.basis = self.field, basis or self.basis
        out.coefficients = np.ascontiguousarray(arr, dtype=np.uint64)
        return out

    def num_terms(self):
        return len(self.coefficients)

    def __eq__(self, other):
        return (isinstance(other, Polynomial) and self.field is other.field and self.basis is other.basis
                and np.array_equal(self.coefficients, other.coefficients))

    def __repr__(self):
        return f"Polynomial<{self.basis.__name__},{self.field!r},{len(self.coefficients)}>({list(map(int, self.coefficients))})"

    # -- Monomial basis ------------------------------------------------------------------------
    def degree(self):  # polynomial/mod.rs:113-115
        nz = np.nonzero(self.coefficients)[0]
        return int(nz[-1]) if len(nz) else 0

    def leading_coefficient(self):  # polynomial/mod.rs:120-122
        nz = np.nonzero(self.coefficients)[0]
        return self.field(int(self.coefficients[nz[-1]])) if len(nz) else self.field.ZERO

    def evaluate(self, x):
        x = self.field(getattr(x, "value", x))
        out = np.empty(1, dtype=np.uint64)
        if self.basis is Monomial:  # polynomial/mod.rs:133-139
            xs = np.array([x.value], dtype=np.uint64)
            self._ctx().call("ronk_poly_eval_u64_host", self.p, _lib._ptr(self.coefficients), len(self.coefficients),
                             _lib._ptr(xs), 1, _lib._ptr(out))
            return self.field(int(out[0]))
        res = C.c_uint64()  # polynomial/mod.rs:382-415
        self._ctx().call("ronk_poly_lagrange_eval_u64_host", self.p, self.g, _lib._ptr(self.coefficients),
                         len(self.coefficients), x.value, C.byref(res))
        return self.field(res.value)

    def evaluate_many(self, xs):
        """Batched `evaluate`: one kernel with one CTA per point in the monomial basis; in the Lagrange basis the
        barycentric form on the nodes ω^i, O(n) per point (0 at a node, as `evaluate`)."""
        xs = _coeffs(self.field, xs)
        out = np.empty(len(xs), dtype=np.uint64)
        if self.basis is Monomial:
            self._ctx().call("ronk_poly_eval_u64_host", self.p, _lib._ptr(self.coefficients), len(self.coefficients),
                             _lib._ptr(xs), len(xs), _lib._ptr(out))
        else:
            self._ctx().call("ronk_poly_lagrange_eval_batch_u64_host", self.p, self.g, _lib._ptr(self.coefficients),
                             len(self.coefficients), 1, 1, _lib._ptr(xs), len(xs), _lib._ptr(out))
        return [self.field(int(v)) for v in out]

    def pow_mult(self, d2: int, coeff):  # polynomial/mod.rs:153-157
        coeff = self.field(getattr(coeff, "value", coeff))
        scaled = self * Polynomial([coeff], self.field)
        return self._like(np.concatenate([np.zeros(d2, dtype=np.uint64), scaled.coefficients]))

    def dft(self):  # polynomial/mod.rs:240-258 — any n | p-1
        assert self.basis is Monomial
        out = np.empty(len(self.coefficients), dtype=np.uint64)
        self._ctx().call("ronk_dft_u64_host", self.p, self.g, _lib._ptr(self.coefficients), len(self.coefficients),
                         _lib._ptr(out))
        return self._like(out, Lagrange)

    def idft(self):
        """Lagrange → Monomial for any n | p-1: the inverse of `dft`, a_j = n^-1 Σ_k X_k ω^(-jk).  An extension: the
        reference has no inverse for n that is not a power of two.  O(n log n) wherever ronk_ntt_any_u64 runs
        Bluestein's algorithm."""
        assert self.basis is Lagrange
        data = self.coefficients.copy()
        self._ctx().call("ronk_ntt_any_u64_host", self.p, self.g, _lib._ptr(data), len(data), 1, 1)
        return self._like(data, Monomial)

    def _ntt(self, inverse: bool):
        n = len(self.coefficients)
        if n == 0 or n & (n - 1):  # where [(); D.is_power_of_two() as usize - 1]: (mod.rs:274)
            raise RonkPanic(1, "D must be a power of two")
        data = self.coefficients.copy()
        self._ctx().call("ronk_ntt_u64_host", self.p, self.g, _lib._ptr(data), n.bit_length() - 1, 1, int(inverse))
        return data

    def fft(self):  # polynomial/mod.rs:273-290
        assert self.basis is Monomial
        return self._like(self._ntt(False), Lagrange)

    def ifft(self):  # polynomial/mod.rs:430-453
        assert self.basis is Lagrange
        return self._like(self._ntt(True), Monomial)

    # -- arithmetic (polynomial/arithmetic.rs) ---------------------------------------------------
    def _addsub(self, rhs, name):
        import torch  # device staging for the device-pointer entry points
        a = torch.from_numpy(self.coefficients.view(np.int64)).cuda()
        b = torch.from_numpy(rhs.coefficients.view(np.int64)).cuda()
        out = torch.empty_like(a)
        self._ctx().call(name, self.p, _lib._ptr(a), a.numel(), _lib._ptr(b), b.numel(), _lib._ptr(out))
        self._ctx().sync()
        return self._like(out.cpu().numpy().view(np.uint64))

    def __add__(self, rhs):  # :16-35 — result has D terms, rhs zero-extended / truncated
        return self._addsub(rhs, "ronk_poly_add_u64")

    def __sub__(self, rhs):  # :49-68
        return self._addsub(rhs, "ronk_poly_sub_u64")

    def __neg__(self):  # :78-95
        zero = self._like(np.zeros(len(self.coefficients), dtype=np.uint64))
        return zero._addsub(self, "ronk_poly_sub_u64")

    def __mul__(self, rhs):  # :97-119 — D + D2 - 1 terms, never trimmed
        out = np.empty(len(self.coefficients) + len(rhs.coefficients) - 1, dtype=np.uint64)
        self._ctx().call("ronk_poly_mul_u64_host", self.p, self.g, _lib._ptr(self.coefficients),
                         len(self.coefficients), _lib._ptr(rhs.coefficients), len(rhs.coefficients), _lib._ptr(out))
        return self._like(out)

    def quotient_and_remainder(self, rhs):  # polynomial/mod.rs:170-225
        d = len(self.coefficients)
        q, r = np.empty(d, dtype=np.uint64), np.empty(d, dtype=np.uint64)
        self._ctx().call("ronk_poly_divrem_u64_host", self.p, _lib._ptr(self.coefficients), d,
                         _lib._ptr(rhs.coefficients), len(rhs.coefficients), _lib._ptr(q), _lib._ptr(r))
        return self._like(q), self._like(r)

    def __truediv__(self, rhs):  # :121-133
        return self.quotient_and_remainder(rhs)[0]

    def __mod__(self, rhs):  # :135-146
        return self.quotient_and_remainder(rhs)[1]

    @staticmethod
    def from_array(coeffs, field, d: int):
        """From<[F; N]> (polynomial/mod.rs:503-515): zero-pad or truncate to D terms."""
        c = list(coeffs)[:d]
        return Polynomial(c + [0] * (d - len(c)), field)
