"""§8f "next" rows, one thin layer above the hot path (all arithmetic in libronk_b200.so):

* Reed–Solomon `Message::encode::<N>` (src/codes/reed_solomon.rs:42-52): the codeword is the
  message polynomial evaluated at the N-th roots of unity ω_N^i — i.e. `Polynomial::dft` of the
  message zero-padded to N coefficients (a plain NTT when N is a power of two).
* Reed–Solomon `Message::decode` (reed_solomon.rs:55-107): Lagrange interpolation through the first
  K coordinates (`ronk_poly_interpolate_u64_host`).
* Reed–Solomon errors-and-erasures correction (`rs_correct`): reads all N coordinates and corrects up to the
  decoding radius (`ronk_rs_decode_u64_host`).
* Shamir `split` (src/shamir/mod.rs:53-58): `Polynomial::evaluate` at x = 1..n, one batched kernel.
* Shamir `split_secret` / `combine_shares` over batches of secrets (`shamir_split`, `shamir_combine`): one batched
  multipoint evaluation at x = 1..n, and one batched interpolation through the shares' x's.
* Shamir recovery from wrong or missing shares (`shamir_recover`): errors-and-erasures Reed–Solomon decoding of every
  row at the shares' x's (`ronk_rs_decode_at_u64_host`).
"""
from __future__ import annotations

import secrets as _secrets

import numpy as np

from .polynomial import Polynomial


def rs_encode(message, n: int, field):
    """Returns [(x_i, y_i)] with x_i = ω_n^i, y_i = m(x_i)  (reed_solomon.rs:42-52).
    Panics (RonkPanic) if n ∤ p-1, like primitive_root_of_unity."""
    k = len(message)
    assert n >= k, "codeword must be at least as long as the message"
    w = field.primitive_root_of_unity(n)
    padded = Polynomial(list(message) + [0] * (n - k), field)
    ys = padded.fft() if n & (n - 1) == 0 and n > 1 else padded.dft()
    xs = Polynomial([1] + [0] * (n - 1), field)  # x_i = ω^i: evaluate X at the roots, i.e. dft of the monomial X
    xs.coefficients = np.roll(xs.coefficients, 1) if n > 1 else xs.coefficients
    xvals = xs.dft().coefficients if n > 1 else np.array([1 % field.ORDER], dtype=np.uint64)
    assert int(xvals[1 % n]) == w.value or n == 1
    return [(field(int(x)), field(int(y))) for x, y in zip(xvals, ys.coefficients)]


def rs_decode(codeword, k: int, field):
    """Message::decode (reed_solomon.rs:55-107): the message is the interpolant through the first
    k coordinates of the codeword, one O(k²) device interpolation.  codeword: [(x_i, y_i)]."""
    from . import _lib
    assert len(codeword) >= k, "codeword must be at least as long as the message"
    xs = np.array([int(getattr(x, "value", x)) for x, _ in codeword[:k]], dtype=np.uint64)
    ys = np.array([int(getattr(y, "value", y)) for _, y in codeword[:k]], dtype=np.uint64)
    out = np.empty(k, dtype=np.uint64)
    _lib.default_context().call("ronk_poly_interpolate_u64_host", field.ORDER, _lib._ptr(xs), _lib._ptr(ys), k,
                                _lib._ptr(out))
    return [field(int(v)) for v in out]


def rs_correct(codeword, k: int, field, erasures=()):
    """Errors-and-erasures decoding of one received word [(x_i, y_i)] whose x_i are ω_n^i in order (as rs_encode
    gives them): returns (message, errors), the message as k field elements and the number of errors corrected, or
    (None, -1) when no codeword lies within the decoding radius (2·errors + len(erasures) ≤ n - k).  `erasures` are
    positions whose y is unknown.  Beyond rs_decode, which trusts the first k coordinates, this reads all n and corrects
    them: one batched device decode (ronk_rs_decode_u64_host)."""
    from . import _lib
    n = len(codeword)
    assert 0 < k <= n, "need 0 < k <= n"
    p, g = field.ORDER, field.PRIMITIVE_ELEMENT.value
    xs = np.array([int(getattr(x, "value", x)) for x, _ in codeword], dtype=np.uint64)
    ys = np.array([int(getattr(y, "value", y)) for _, y in codeword], dtype=np.uint64)
    ctx = _lib.default_context()
    dom = np.zeros(n, dtype=np.uint64)           # ω_n^i: the transform of the monomial X (of 1 when n = 1)
    dom[1 % n] = 1
    ctx.call("ronk_ntt_any_u64_host", p, g, _lib._ptr(dom), n, 1, 0)
    assert np.array_equal(xs, dom), "x coordinates must be ω_n^i, i = 0 … n-1, in order"
    erased = np.zeros(n, dtype=np.uint8)
    erased[list(erasures)] = 1
    msg = np.empty(k, dtype=np.uint64)
    status = np.empty(1, dtype=np.int32)
    ctx.call("ronk_rs_decode_u64_host", p, g, _lib._ptr(ys), _lib._ptr(erased), n, k, 1, _lib._ptr(msg),
             _lib._ptr(status))
    if status[0] < 0:
        return None, -1
    return [field(int(v)) for v in msg], int(status[0])


def shamir_shares(coefficients, n: int, field):
    """Evaluations of the sharing polynomial at x = 1..n (shamir/mod.rs:53-58), one kernel launch."""
    poly = Polynomial(coefficients, field)
    return list(zip(range(1, n + 1), poly.evaluate_many(range(1, n + 1))))


def shamir_split(secrets, threshold: int, n: int, field, coefficients=None):
    """split_secret (shamir/mod.rs:33-60) of every secret: returns (xs, ys) with xs = [1, …, n] and ys a (len(secrets), n)
    array, row b the shares of secrets[b].  Row b's polynomial is secrets[b] + Σ_j coefficients[b][j-1]·X^j, j < threshold;
    without `coefficients` they are drawn from the operating system's CSPRNG (`secrets.randbelow`).  One batched
    multipoint evaluation on the device.  Panics (AssertionError) like the reference on threshold 0 or n < threshold."""
    from . import _lib
    assert threshold > 0, "threshold must be at least 1"
    assert n >= threshold, "share count must be at least the threshold"
    p = field.ORDER
    assert n < p, "the share x's 1..n must be distinct field elements"
    s = [int(getattr(v, "value", v)) % p for v in secrets]
    if coefficients is None:
        coefficients = [[_secrets.randbelow(p) for _ in range(threshold - 1)] for _ in s]
    assert len(coefficients) == len(s) and all(len(c) == threshold - 1 for c in coefficients), \
        "coefficients is len(secrets) rows of threshold - 1"
    rows = np.array([[v] + [int(getattr(c, "value", c)) % p for c in cs] for v, cs in zip(s, coefficients)],
                    dtype=np.uint64).reshape(len(s), threshold)
    xs = np.arange(1, n + 1, dtype=np.uint64)
    ys = np.empty((len(s), n), dtype=np.uint64)
    if s:
        _lib.default_context().call("ronk_poly_multieval_batch_u64_host", p, field.PRIMITIVE_ELEMENT.value,
                                    _lib._ptr(rows), threshold, len(s), _lib._ptr(xs), n, _lib._ptr(ys))
    return xs, ys


def shamir_combine(shares_xs, shares_ys, field):
    """combine_shares (shamir/mod.rs:76-97) of every row: shares_xs (k,) are the x's every secret's shares share,
    shares_ys is (batch, k); returns the batch secrets as field elements.  The secret is coefficient 0 of the interpolant
    through the shares, the reference's Lagrange sum at 0, also for more shares than the threshold.  One batched
    interpolation on the device; a repeated x panics (RonkPanic) as the reference's inverse does."""
    from . import _lib
    p = field.ORDER
    xs = np.array([int(getattr(x, "value", x)) % p for x in shares_xs], dtype=np.uint64)
    k = len(xs)
    assert k > 0, "at least one share is required"
    ys = np.array([[int(getattr(y, "value", y)) % p for y in row] for row in shares_ys], dtype=np.uint64).reshape(-1, k)
    out = np.empty_like(ys)
    if len(ys):
        _lib.default_context().call("ronk_poly_interpolate_batch_u64_host", p, field.PRIMITIVE_ELEMENT.value,
                                    _lib._ptr(xs), _lib._ptr(ys), k, len(ys), _lib._ptr(out))
    return [field(int(v)) for v in out[:, 0]]


def shamir_recover(shares_xs, shares_ys, threshold: int, field, missing=None):
    """combine_shares that survives dishonest and absent shareholders: shares_xs (n,) are the distinct x's every
    secret's shares share, shares_ys is (batch, n), and `missing` (None, or a (batch, n) mask) marks shares known to be
    absent, whose y's are never read.  Every row is Reed–Solomon decoded at the x's, with message length `threshold`:
    with e wrong and ε missing shares, a row with 2e + ε ≤ n - threshold gives its secret exactly.  Returns
    (secrets, errors): a secret is a field element, or None for a row that cannot be recovered (then errors is -1);
    errors[b] counts the wrong shares found in row b.  No row is ever given a secret whose polynomial differs from its
    shares in more than (n - threshold - ε)/2 of them.  One batched device decode (ronk_rs_decode_at_u64_host); a
    repeated x panics (RonkPanic)."""
    from . import _lib
    p = field.ORDER
    xs = np.array([int(getattr(x, "value", x)) % p for x in shares_xs], dtype=np.uint64)
    n = len(xs)
    assert 0 < threshold <= n, "need 0 < threshold <= share count"
    ys = np.array([[int(getattr(y, "value", y)) % p for y in row] for row in shares_ys], dtype=np.uint64).reshape(-1, n)
    batch = len(ys)
    erased = None
    if missing is not None:
        erased = np.ascontiguousarray(np.asarray(missing, dtype=bool).reshape(batch, n), dtype=np.uint8)
    msg = np.empty((batch, threshold), dtype=np.uint64)
    status = np.empty(batch, dtype=np.int32)
    if batch:
        _lib.default_context().call("ronk_rs_decode_at_u64_host", p, field.PRIMITIVE_ELEMENT.value, _lib._ptr(xs),
                                    _lib._ptr(ys), _lib._ptr(erased), n, threshold, batch, _lib._ptr(msg),
                                    _lib._ptr(status))
    secrets = [field(int(msg[b, 0])) if status[b] >= 0 else None for b in range(batch)]
    return secrets, [int(s) for s in status]
