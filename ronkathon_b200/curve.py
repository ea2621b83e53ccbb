"""Host-side mirror of `AffinePoint<PlutoExtendedCurve>` (src/curve/mod.rs:67-235,
src/curve/pluto_curve.rs:27-64).  Group operations run in libronk_b200.so's curve kernels."""
from __future__ import annotations

import numpy as np

from . import _lib
from ._lib import RonkPanic

INF_BYTES = bytes([0xFF] * 4)


class AffinePoint:
    """Point on y² = x³ + 3 over GF(101²) (x = x0 + x1·t), or Infinity."""

    __slots__ = ("raw",)

    def __init__(self, raw: bytes):
        self.raw = bytes(raw)

    @staticmethod
    def new(x, y):
        """AffinePoint::new (curve/mod.rs:78-82): asserts the point is on the curve.
        x, y: ints (base-field embedding) or (c0, c1) pairs."""
        x0, x1 = (x, 0) if isinstance(x, int) else x
        y0, y1 = (y, 0) if isinstance(y, int) else y
        p = AffinePoint(bytes([x0 % 101, x1 % 101, y0 % 101, y1 % 101]))
        p + AffinePoint.infinity()  # the add kernel validates is_on_curve; raises RonkPanic otherwise
        return p

    @staticmethod
    def infinity():
        return AffinePoint(INF_BYTES)

    @property
    def is_infinity(self):
        return self.raw == INF_BYTES

    def xy(self):  # curve/mod.rs:141-146
        if self.is_infinity:
            return (0, 0), (0, 0), True
        return (self.raw[0], self.raw[1]), (self.raw[2], self.raw[3]), False

    def _call(self, name, *bufs):
        out = np.empty(4, dtype=np.uint8)
        args = [_lib._ptr(np.frombuffer(b, dtype=np.uint8).copy()) for b in bufs]
        _lib.default_context().call(name, *args, _lib._ptr(out), 1)
        return AffinePoint(out.tobytes())

    def __add__(self, rhs):  # curve/mod.rs:178-213
        return self._call("ronk_point_add_pluto_ext_host", self.raw, rhs.raw)

    def __neg__(self):  # curve/mod.rs:225-235
        return self._call("ronk_point_neg_pluto_ext_host", self.raw)

    def __sub__(self, rhs):  # curve/mod.rs:240-244
        return self + (-rhs)

    def double(self):  # curve/mod.rs:113-128
        return self + self

    def __mul__(self, scalar):  # Mul<ScalarField> (curve/mod.rs:157-172)
        s = int(getattr(scalar, "value", scalar)) % 17
        return self._call("ronk_point_smul_pluto_ext_host", self.raw, bytes([s]))

    __rmul__ = __mul__

    def __eq__(self, other):
        return isinstance(other, AffinePoint) and self.raw == other.raw

    def __hash__(self):
        return hash(self.raw)

    def __repr__(self):
        if self.is_infinity:
            return "Infinity"
        return f"Point({self.raw[0]}+{self.raw[1]}t, {self.raw[2]}+{self.raw[3]}t)"


# curve constants (pluto_curve.rs:27-51)
G1_GENERATOR = AffinePoint(bytes([1, 0, 2, 0]))       # PlutoBaseCurve::GENERATOR embedded
G2_GENERATOR = AffinePoint(bytes([36, 0, 0, 31]))     # PlutoExtendedCurve::GENERATOR
CURVE_ORDER = 17


def sum_points(points):
    """Sum (curve/mod.rs:219-223): reduce(+) or Infinity."""
    acc = None
    for p in points:
        acc = p if acc is None else acc + p
    return AffinePoint.infinity() if acc is None else acc


def pairing(p: AffinePoint, q: AffinePoint):
    """pairing::<PlutoExtendedCurve, 17> (curve/pairing.rs:33-54): (c0, c1) of the value in GF(101²), a 17th root of
    unity.  Raises RonkPanic where the reference panics: p or q is not 17-torsion or is Infinity, or p == q."""
    out = np.empty(2, dtype=np.uint8)
    a = np.frombuffer(p.raw, dtype=np.uint8).copy()
    b = np.frombuffer(q.raw, dtype=np.uint8).copy()
    _lib.default_context().call("ronk_pairing_pluto_ext_host", _lib._ptr(a), _lib._ptr(b), 1, _lib._ptr(out))
    return int(out[0]), int(out[1])
