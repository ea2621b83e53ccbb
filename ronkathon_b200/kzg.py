"""Host-side mirror of ronkathon's kzg module (src/kzg/setup.rs): setup / commit / open / check.
`commit` is the group-coordinate MSM kernel in libronk_b200.so, `commit_batch` its batched form; `check` and
`check_batch` look both pairings up in a table of the reference's Tate pairing on E[17] (ronk_kzg_check_pluto_ext_batch)."""
from __future__ import annotations

import numpy as np

from . import _lib
from .curve import G1_GENERATOR, G2_GENERATOR, AffinePoint
from .field import PlutoScalarField
from .polynomial import Polynomial


def setup():
    """kzg/setup.rs:10-43: tau = 2; 7 G1 powers and 2 G2 powers."""
    tau = PlutoScalarField(2)
    g1 = [G1_GENERATOR * tau.pow(i) for i in range(7)]
    g2 = [G2_GENERATOR * tau.pow(i) for i in range(2)]
    return g1, g2


def _pack(points) -> np.ndarray:
    if isinstance(points, np.ndarray):
        return np.ascontiguousarray(points, dtype=np.uint8).reshape(-1)
    return np.frombuffer(b"".join(p.raw for p in points), dtype=np.uint8).copy()


def commit(coeffs, g1_srs) -> AffinePoint:
    """kzg/setup.rs:48-60: Σ g1_srs[i]·coeffs[i]; asserts g1_srs.len() >= coeffs.len()."""
    pts = _pack(g1_srs)
    # coefficients are PlutoScalarField values; raw ints are reduced as PlutoScalarField::new does
    # (prime/mod.rs:48-51: value % P) — never wrapped by the uint8 cast
    sc = np.array([int(getattr(c, "value", c)) % 17 for c in coeffs], dtype=np.uint8)
    out = np.empty(4, dtype=np.uint8)
    n_pts = len(pts) // 4
    # the zip stops at the shorter sequence, so only the first len(coeffs) points are shipped
    _lib.default_context().call("ronk_msm_pluto_ext_host", _lib._ptr(pts), n_pts, _lib._ptr(sc), len(sc),
                                _lib._ptr(out))
    return AffinePoint(out.tobytes())


def commit_batch(rows, g1_srs) -> list:
    """[commit(r, g1_srs) for r in rows] in one batched call (ronk_msm_pluto_ext_batch_host), the panics included.  The
    rows are zero-padded to the longest: a zero scalar adds nothing, and the longest row is the one that sets the SRS
    length check."""
    sc = [[int(getattr(c, "value", c)) % 17 for c in r] for r in rows]
    if not sc:
        return []
    n = max(len(r) for r in sc)
    block = np.zeros((len(sc), n), dtype=np.uint8)
    for i, r in enumerate(sc):
        block[i, :len(r)] = r
    pts = _pack(g1_srs)
    out = np.empty((len(sc), 4), dtype=np.uint8)
    _lib.default_context().call("ronk_msm_pluto_ext_batch_host", _lib._ptr(pts), len(pts) // 4, _lib._ptr(block), n, len(sc),
                                _lib._ptr(out))
    return [AffinePoint(w.tobytes()) for w in out]


def open_(coeffs, eval_point, g1_srs) -> AffinePoint:
    """kzg/setup.rs:63-78: poly / (x - z) by Polynomial::div, then commit the quotient."""
    poly = Polynomial(coeffs, PlutoScalarField)
    z = PlutoScalarField(getattr(eval_point, "value", eval_point))
    divisor = Polynomial([(-z).value, 1], PlutoScalarField)
    q = poly / divisor
    return commit([int(v) for v in q.coefficients], g1_srs)


def open_batch(polys, eval_point, g1_srs) -> list:
    """open_ of every polynomial at one point: the quotients by the shared divisor [-z, 1] in one batched division
    (ronk_poly_divrem_batch_u64_host), then every quotient in one commit_batch.  Returns the points
    [open_(f, eval_point, g1_srs) for f in polys].  The rows of one batched call share their length, so polynomials of
    different lengths take one division per length rather than being zero-padded to one: a quotient keeps its
    polynomial's length."""
    rows = [Polynomial(f, PlutoScalarField) for f in polys]
    z = PlutoScalarField(getattr(eval_point, "value", eval_point))
    divisor = np.array([(-z).value, 1], dtype=np.uint64)
    quotients = [None] * len(rows)
    for d in sorted({len(f.coefficients) for f in rows}):
        idx = [i for i, f in enumerate(rows) if len(f.coefficients) == d]
        a = np.ascontiguousarray(np.stack([rows[i].coefficients for i in idx]), dtype=np.uint64)
        q, r = np.empty_like(a), np.empty_like(a)
        _lib.default_context().call("ronk_poly_divrem_batch_u64_host", rows[idx[0]].p, 0, _lib._ptr(a), d, _lib._ptr(divisor), 2, 1,
                                    len(idx), _lib._ptr(q), _lib._ptr(r))
        for i, row in zip(idx, q):
            quotients[i] = row
    return commit_batch(quotients, g1_srs)


def _scalars(xs) -> np.ndarray:
    return np.array([int(getattr(x, "value", x)) % 17 for x in xs], dtype=np.uint8)


def check(p, q, point, value, g1_srs, g2_srs) -> bool:
    """kzg/setup.rs:81-103: pairing(q, g2_srs[1] - GEN·point) == pairing(p - g1_srs[0]·value, GEN).  Raises RonkPanic
    where the reference panics: an empty g1_srs, fewer than two g2_srs points, or either pairing panicking."""
    return check_batch([p], [q], [point], [value], g1_srs, g2_srs)[0]


def check_batch(commitments, proofs, points, values, g1_srs, g2_srs) -> list:
    """[check(c, q, z, v, g1_srs, g2_srs) for each row] in one call (ronk_kzg_check_pluto_ext_batch_host); raises
    RonkPanic if any row panics.  Scalars are reduced mod 17, as PlutoScalarField::new does."""
    c, q = _pack(commitments), _pack(proofs)
    z, v = _scalars(points), _scalars(values)
    n = len(z)
    if not (len(c) == len(q) == 4 * n and len(v) == n):
        raise ValueError("commitments, proofs, points and values must have one entry per row")
    g1, g2 = _pack(g1_srs), _pack(g2_srs)
    ok = np.empty(n, dtype=np.uint8)
    _lib.default_context().call("ronk_kzg_check_pluto_ext_batch_host", _lib._ptr(c), _lib._ptr(q), _lib._ptr(z), _lib._ptr(v), n,
                                _lib._ptr(g1), len(g1) // 4, _lib._ptr(g2), len(g2) // 4, _lib._ptr(ok))
    return [bool(b) for b in ok]


def commit_lagrange(evaluations, g1_srs) -> AffinePoint:
    """Commit to a polynomial given in the LAGRANGE basis over the 2^k-th roots of unity of F17 — the form in
    which the PLONK compiler emits its selector / permutation polynomials (compiler/program.rs:118-226,
    `Polynomial<Lagrange<PlutoScalarField>, PlutoScalarField, GROUP_ORDER>`).  The prover step the reference
    never wrote: Lagrange → monomial by the inverse transform (polynomial/mod.rs:430-453, on the GPU), then
    kzg::commit (kzg/setup.rs:48-60, the MSM kernel)."""
    from .polynomial import Lagrange
    poly = evaluations if isinstance(evaluations, Polynomial) else Polynomial(evaluations, PlutoScalarField, Lagrange)
    if poly.basis is not Lagrange:
        raise _lib.RonkPanic(1, "commit_lagrange expects a Lagrange-basis polynomial")
    mono = poly.ifft()
    return commit([int(v) for v in mono.coefficients], g1_srs)


def open_lagrange(evaluations, eval_point, g1_srs) -> AffinePoint:
    """kzg/setup.rs:63-78 in evaluation form: the polynomial given by its values on the n-th roots of unity of F17, opened
    at z.  The quotient (f - f(z)) / (X - z) is formed on the same nodes in one O(n) pass (ronk_poly_lagrange_open_u64,
    also where z is a node), then committed with commit_lagrange.  The same point as open_ on the monomial coefficients."""
    from .polynomial import Lagrange
    poly = evaluations if isinstance(evaluations, Polynomial) else Polynomial(evaluations, PlutoScalarField, Lagrange)
    if poly.basis is not Lagrange:
        raise _lib.RonkPanic(1, "open_lagrange expects a Lagrange-basis polynomial")
    z = PlutoScalarField(getattr(eval_point, "value", eval_point))
    n = len(poly.coefficients)
    value = np.empty(1, dtype=np.uint64)
    quotient = np.empty(n, dtype=np.uint64)
    _lib.default_context().call("ronk_poly_lagrange_open_u64_host", poly.p, poly.g, _lib._ptr(poly.coefficients), n, 1, 1,
                                z.value, _lib._ptr(value), _lib._ptr(quotient))
    return commit_lagrange(Polynomial(quotient, PlutoScalarField, Lagrange), g1_srs)


def commit_preprocessed(polys: dict, g1_srs) -> dict:
    """Commitments to a `CommonPreprocessedInput` (compiler/program.rs:59-63: ql, qr, qm, qo, qc, s1, s2, s3),
    each given as GROUP_ORDER evaluations: commit_lagrange of every column, with the columns' inverse transforms as one
    batched transform per length (one in all, as the columns share GROUP_ORDER) and their commitments in one
    commit_batch."""
    from .polynomial import Lagrange
    cols = {}
    for name, ev in polys.items():
        poly = ev if isinstance(ev, Polynomial) else Polynomial(ev, PlutoScalarField, Lagrange)
        if poly.basis is not Lagrange:
            raise _lib.RonkPanic(1, "commit_preprocessed expects Lagrange-basis polynomials")
        n = len(poly.coefficients)
        if n & (n - 1):   # where [(); D.is_power_of_two() as usize - 1]: (polynomial/mod.rs:274)
            raise _lib.RonkPanic(1, "D must be a power of two")
        cols[name] = poly
    mono = {}
    for n in sorted({len(p.coefficients) for p in cols.values()}):
        names = [k for k, p in cols.items() if len(p.coefficients) == n]
        data = np.ascontiguousarray(np.stack([cols[k].coefficients for k in names]), dtype=np.uint64)
        p0 = cols[names[0]]
        _lib.default_context().call("ronk_ntt_u64_host", p0.p, p0.g, _lib._ptr(data), n.bit_length() - 1, len(names), 1)
        mono.update(zip(names, data))
    return dict(zip(polys, commit_batch([mono[k] for k in polys], g1_srs)))

