"""Device-resident operator API (torch tensors hold the HBM buffers; libronk_b200.so does the work).

This is the path bench.py times: buffers stay on the GPU, calls are asynchronous on the
context's stream.  Tensors are int64 views of uint64 canonical residues (torch has no uint64
arithmetic; nothing here does arithmetic in torch).
"""
from __future__ import annotations

import numpy as np

from . import _lib
from ._lib import GOLDILOCKS, Context


def _check_u64(t):
    import torch
    assert t.is_cuda and t.dtype == torch.int64 and t.is_contiguous(), "need a contiguous CUDA int64 (uint64 view) tensor"


def to_device(a: np.ndarray, device="cuda"):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64)).to(device)


def to_host(t) -> np.ndarray:
    return t.cpu().numpy().view(np.uint64)


def ntt_(ctx: Context, data, log_n: int, batch: int = 1, inverse: bool = False, p: int = GOLDILOCKS, g: int = 7):
    """In-place Polynomial::fft / ifft over `batch` contiguous transforms."""
    _check_u64(data)
    assert data.numel() == (batch << log_n)
    ctx.call("ronk_ntt_u64", p, g, _lib._ptr(data), log_n, batch, int(inverse))
    return data


def ntt_any_(ctx: Context, data, n: int, batch: int = 1, inverse: bool = False, p: int = GOLDILOCKS, g: int = 7):
    """In-place transforms of any length n | p - 1 (Polynomial::dft and its inverse) over `batch` contiguous rows:
    the power-of-two transform, Bluestein's algorithm where its convolution fits, else the O(n²) dft kernels."""
    _check_u64(data)
    assert data.numel() == batch * n
    ctx.call("ronk_ntt_any_u64", p, g, _lib._ptr(data), n, batch, int(inverse))
    return data


def ntt_coset_(ctx: Context, data, log_n: int, shift: int, batch: int = 1, inverse: bool = False, p: int = GOLDILOCKS,
               g: int = 7):
    """In-place transforms on the coset shift·H_n over `batch` contiguous rows: forward X[k] = Σ_j a_j (shift·ω^k)^j,
    inverse its inverse.  shift = 1 is ntt_."""
    _check_u64(data)
    assert data.numel() == (batch << log_n)
    ctx.call("ronk_ntt_coset_u64", p, g, _lib._ptr(data), log_n, batch, shift, int(inverse))
    return data


def lde(ctx: Context, coeffs, log_n: int, shift: int, p: int = GOLDILOCKS, g: int = 7):
    """Low-degree extension: the coefficients (d,) — or rows (batch, d) — evaluated on shift·H_N, N = 2^log_n ≥ d.
    Returns a new (N,) — or (batch, N) — tensor."""
    import torch
    _check_u64(coeffs)
    assert coeffs.dim() in (1, 2), "coeffs is (d,) or (batch, d)"
    batch, d = (1, coeffs.shape[0]) if coeffs.dim() == 1 else coeffs.shape
    out = torch.empty(coeffs.shape[:-1] + (1 << log_n,), dtype=torch.int64, device=coeffs.device)
    ctx.call("ronk_poly_lde_u64", p, g, _lib._ptr(coeffs), d, log_n, shift, batch, _lib._ptr(out))
    return out


def ntt_mul_(ctx: Context, data, mul, log_n: int, batch: int = 1, p: int = GOLDILOCKS, g: int = 7):
    """data ← NTT(data) ⊙ mul, the point-wise product fused into the last stage."""
    _check_u64(data); _check_u64(mul)
    ctx.call("ronk_ntt_mul_u64", p, g, _lib._ptr(data), _lib._ptr(mul), log_n, batch)
    return data


def poly_mul(ctx: Context, a, b, p: int = GOLDILOCKS, g: int = 7):
    """Polynomial::mul — returns a new tensor with len(a)+len(b)-1 coefficients."""
    import torch
    _check_u64(a); _check_u64(b)
    out = torch.empty(a.numel() + b.numel() - 1, dtype=torch.int64, device=a.device)
    ctx.call("ronk_poly_mul_u64", p, g, _lib._ptr(a), a.numel(), _lib._ptr(b), b.numel(), _lib._ptr(out))
    return out


def poly_mul_batch(ctx: Context, a, b, p: int = GOLDILOCKS, g: int = 7):
    """Polynomial::mul of every row pair: a is (batch, da); b is (batch, db), or (db,) for one b shared by every row.
    Returns a new (batch, da + db - 1) tensor, row r = a[r]·b[r] (or a[r]·b), each row the words poly_mul gives."""
    import torch
    _check_u64(a); _check_u64(b)
    assert a.dim() == 2 and b.dim() in (1, 2), "a is (batch, da); b is (batch, db) or (db,)"
    batch, da = a.shape
    shared = b.dim() == 1
    db = b.shape[-1]
    assert shared or b.shape[0] == batch
    out = torch.empty((batch, da + db - 1), dtype=torch.int64, device=a.device)
    ctx.call("ronk_poly_mul_batch_u64", p, g, _lib._ptr(a), da, _lib._ptr(b), db, int(shared), batch, _lib._ptr(out))
    return out


def poly_divrem(ctx: Context, a, b, p: int = GOLDILOCKS, g: int = 7):
    """Polynomial::quotient_and_remainder — returns new tensors (q, r), each with len(a) coefficients (zero-padded
    like the reference's arrays).  Synchronous; raises RonkPanic where the reference panics."""
    import torch
    _check_u64(a); _check_u64(b)
    q = torch.empty_like(a)
    r = torch.empty_like(a)
    ctx.call("ronk_poly_divrem_u64", p, g, _lib._ptr(a), a.numel(), _lib._ptr(b), b.numel(), _lib._ptr(q), _lib._ptr(r))
    return q, r


def poly_divrem_batch(ctx: Context, a, b, p: int = GOLDILOCKS, g: int = 7):
    """Polynomial::quotient_and_remainder of every row: a is (batch, da); b is (batch, db), or (db,) for one divisor
    shared by every row.  Returns new (q, r) tensors of shape (batch, da), each row the words poly_divrem gives for it.
    Synchronous; raises RonkPanic where the reference panics on any row."""
    import torch
    _check_u64(a); _check_u64(b)
    assert a.dim() == 2 and b.dim() in (1, 2), "a is (batch, da); b is (batch, db) or (db,)"
    batch, da = a.shape
    shared = b.dim() == 1
    assert shared or b.shape[0] == batch
    q = torch.empty_like(a)
    r = torch.empty_like(a)
    ctx.call("ronk_poly_divrem_batch_u64", p, g, _lib._ptr(a), da, _lib._ptr(b), b.shape[-1], int(shared), batch, _lib._ptr(q),
             _lib._ptr(r))
    return q, r


def poly_eval(ctx: Context, coeffs, xs, p: int = GOLDILOCKS):
    import torch
    _check_u64(coeffs); _check_u64(xs)
    out = torch.empty_like(xs)
    ctx.call("ronk_poly_eval_u64", p, _lib._ptr(coeffs), coeffs.numel(), _lib._ptr(xs), xs.numel(), _lib._ptr(out))
    return out


def _rows(evals, n: int):
    """(n,) or (batch, n) evaluations → (batch, leading shape)."""
    _check_u64(evals)
    assert evals.dim() in (1, 2) and evals.shape[-1] == n, "evals is (n,) or (batch, n)"
    return (1 if evals.dim() == 1 else evals.shape[0]), tuple(evals.shape[:-1])


def lagrange_eval(ctx: Context, evals, xs, n: int, shift: int = 1, p: int = GOLDILOCKS, g: int = 7):
    """Lagrange-basis rows on the coset shift·H_n (evals (n,) or (batch, n), row b holding f_b(shift·ω^j)) evaluated at
    the m points xs, by the barycentric formula in O(n) per point: a new (m,) or (batch, m) tensor.  At a node the value
    is 0, as the reference's Lagrange evaluate gives.  Asynchronous."""
    import torch
    batch, lead = _rows(evals, n)
    _check_u64(xs)
    out = torch.empty(lead + (xs.numel(),), dtype=torch.int64, device=evals.device)
    ctx.call("ronk_poly_lagrange_eval_u64", p, g, _lib._ptr(evals), n, batch, shift, _lib._ptr(xs), xs.numel(),
             _lib._ptr(out))
    return out


def lagrange_open(ctx: Context, evals, z: int, n: int, shift: int = 1, p: int = GOLDILOCKS, g: int = 7):
    """Opens Lagrange-basis rows on shift·H_n at z: returns new tensors (values, quotient), values[b] = f_b(z) ((,) or
    (batch,)) and quotient the evaluations of (f_b - f_b(z)) / (X - z) on the same nodes (the shape of evals).
    Asynchronous."""
    import torch
    batch, lead = _rows(evals, n)
    values = torch.empty(lead if lead else (1,), dtype=torch.int64, device=evals.device)
    quotient = torch.empty_like(evals)
    ctx.call("ronk_poly_lagrange_open_u64", p, g, _lib._ptr(evals), n, batch, shift, z, _lib._ptr(values),
             _lib._ptr(quotient))
    return (values if lead else values[0]), quotient


def poly_from_roots(ctx: Context, xs, p: int = GOLDILOCKS, g: int = 7):
    """Π (X - xs[i]) — returns a new tensor of len(xs) + 1 coefficients (subproduct tree above the crossover)."""
    import torch
    _check_u64(xs)
    out = torch.empty(xs.numel() + 1, dtype=torch.int64, device=xs.device)
    ctx.call("ronk_poly_from_roots_u64", p, g, _lib._ptr(xs), xs.numel(), _lib._ptr(out))
    return out


def poly_multieval(ctx: Context, coeffs, xs, p: int = GOLDILOCKS, g: int = 7):
    """evaluate at every xs[i] — the same words as poly_eval, on a subproduct tree above the crossover."""
    import torch
    _check_u64(coeffs); _check_u64(xs)
    out = torch.empty_like(xs)
    ctx.call("ronk_poly_multieval_u64", p, g, _lib._ptr(coeffs), coeffs.numel(), _lib._ptr(xs), xs.numel(), _lib._ptr(out))
    return out


def poly_interpolate(ctx: Context, xs, ys, p: int = GOLDILOCKS, g: int = 7):
    """The interpolant through (xs[i], ys[i]) — len(xs) coefficients.  Synchronous; raises RonkPanic for a repeated x."""
    import torch
    _check_u64(xs); _check_u64(ys)
    assert xs.numel() == ys.numel()
    out = torch.empty_like(xs)
    ctx.call("ronk_poly_interpolate_u64", p, g, _lib._ptr(xs), _lib._ptr(ys), xs.numel(), _lib._ptr(out))
    return out


def poly_multieval_batch(ctx: Context, coeffs, xs, p: int = GOLDILOCKS, g: int = 7):
    """evaluate every row of coeffs (batch, d) at every xs[i]: a new (batch, m) tensor, row b the words poly_multieval
    gives for coeffs[b].  One subproduct tree over xs serves every row.  Asynchronous."""
    import torch
    _check_u64(coeffs); _check_u64(xs)
    assert coeffs.dim() == 2, "coeffs is (batch, d)"
    batch, d = coeffs.shape
    out = torch.empty((batch, xs.numel()), dtype=torch.int64, device=xs.device)
    ctx.call("ronk_poly_multieval_batch_u64", p, g, _lib._ptr(coeffs), d, batch, _lib._ptr(xs), xs.numel(), _lib._ptr(out))
    return out


def poly_interpolate_batch(ctx: Context, xs, ys, p: int = GOLDILOCKS, g: int = 7):
    """The interpolant through (xs[i], ys[b, i]) for every row of ys (batch, k): a new (batch, k) tensor, row b the words
    poly_interpolate gives for ys[b].  One subproduct tree over xs serves every row.  Synchronous; raises RonkPanic for
    a repeated x."""
    import torch
    _check_u64(xs); _check_u64(ys)
    assert ys.dim() == 2 and ys.shape[1] == xs.numel(), "ys is (batch, len(xs))"
    out = torch.empty_like(ys)
    ctx.call("ronk_poly_interpolate_batch_u64", p, g, _lib._ptr(xs), _lib._ptr(ys), xs.numel(), ys.shape[0], _lib._ptr(out))
    return out


def rs_encode(ctx: Context, msg, n: int, batch: int = 1, p: int = GOLDILOCKS, g: int = 7):
    """Reed–Solomon Message::encode of `batch` messages (msg: batch × k, row-major): a new batch × n tensor of
    codewords, position i holding the message polynomial at ω_n^i."""
    import torch
    _check_u64(msg)
    assert msg.numel() % batch == 0
    out = torch.empty(batch * n, dtype=torch.int64, device=msg.device)
    ctx.call("ronk_rs_encode_u64", p, g, _lib._ptr(msg), msg.numel() // batch if batch else 0, n, batch, _lib._ptr(out))
    return out


def rs_decode(ctx: Context, received, k: int, erased=None, batch: int = 1, p: int = GOLDILOCKS, g: int = 7):
    """Errors-and-erasures decoding of `batch` received words (batch × n): returns new tensors (messages, batch × k;
    status, int32 per row: the errors corrected, or -1 with a zero message for a row outside the decoding radius).
    erased: None or a uint8/bool tensor of batch × n, nonzero at erased positions.  Asynchronous."""
    import torch
    _check_u64(received)
    assert received.numel() % batch == 0 if batch else received.numel() == 0
    n = received.numel() // batch if batch else 0
    if erased is not None:
        erased = erased.to(torch.uint8).contiguous()
        assert erased.is_cuda and erased.numel() == received.numel()
    msg = torch.empty(batch * k, dtype=torch.int64, device=received.device)
    status = torch.empty(batch, dtype=torch.int32, device=received.device)
    ctx.call("ronk_rs_decode_u64", p, g, _lib._ptr(received), _lib._ptr(erased), n, k, batch, _lib._ptr(msg),
             _lib._ptr(status))
    return msg, status


def rs_decode_at(ctx: Context, xs, received, k: int, erased=None, batch: int = 1, p: int = GOLDILOCKS, g: int = 7):
    """rs_decode for received words whose positions share any n distinct points xs (n words, canonical): returns new
    tensors (messages, batch × k; status, int32 per row: the errors corrected, or -1 with a zero message for a row
    outside the decoding radius).  erased: None or a uint8/bool tensor of batch × n, nonzero at erased positions, whose
    received values are never read.  Synchronous; raises RonkPanic for a repeated point."""
    import torch
    _check_u64(xs); _check_u64(received)
    n = xs.numel()
    assert received.numel() == batch * n, "received is batch × len(xs)"
    if erased is not None:
        erased = erased.to(torch.uint8).contiguous()
        assert erased.is_cuda and erased.numel() == received.numel()
    msg = torch.empty(batch * k, dtype=torch.int64, device=received.device)
    status = torch.empty(batch, dtype=torch.int32, device=received.device)
    ctx.call("ronk_rs_decode_at_u64", p, g, _lib._ptr(xs), _lib._ptr(received), _lib._ptr(erased), n, k, batch,
             _lib._ptr(msg), _lib._ptr(status))
    return msg, status


def field_binop(ctx: Context, op: str, a, b, p: int = GOLDILOCKS):
    import torch
    _check_u64(a); _check_u64(b)
    out = torch.empty_like(a)
    ctx.call({"add": "ronk_field_add_u64", "sub": "ronk_field_sub_u64", "mul": "ronk_field_mul_u64",
              "div": "ronk_field_div_u64"}[op], p, _lib._ptr(a), _lib._ptr(b), _lib._ptr(out), a.numel())
    return out


def splitmix_fill(ctx: Context, n: int, seed: int, p: int = GOLDILOCKS, device="cuda"):
    import torch
    out = torch.empty(n, dtype=torch.int64, device=device)
    ctx.call("ronk_splitmix_fill_u64", p, seed, _lib._ptr(out), n)
    return out


def msm(ctx: Context, points, scalars) -> bytes:
    """kzg::commit on device-resident packed points (uint8 [n,4]) and scalars (uint8 [n])."""
    import torch
    assert points.is_cuda and points.dtype == torch.uint8 and scalars.dtype == torch.uint8
    out = np.empty(4, dtype=np.uint8)
    ctx.call("ronk_msm_pluto_ext", _lib._ptr(points), points.numel() // 4, _lib._ptr(scalars), scalars.numel(),
             _lib._ptr(out))
    return out.tobytes()


def msm_batch(ctx: Context, points, scalars):
    """kzg::commit of every row of scalars (uint8 [batch, n]) against the device-resident packed points (uint8 [n', 4],
    n' ≥ n): a new uint8 [batch, 4] device tensor, row r the point msm gives for scalars[r].  Synchronous; raises
    RonkPanic where msm does on any row."""
    import torch
    assert points.is_cuda and points.dtype == torch.uint8 and points.is_contiguous()
    assert scalars.is_cuda and scalars.dtype == torch.uint8 and scalars.dim() == 2 and scalars.is_contiguous(), \
        "scalars is a contiguous uint8 (batch, n) tensor"
    batch, n = scalars.shape
    out = torch.empty((batch, 4), dtype=torch.uint8, device=scalars.device)
    ctx.call("ronk_msm_pluto_ext_batch", _lib._ptr(points), points.numel() // 4, _lib._ptr(scalars), n, batch, _lib._ptr(out))
    return out


def pairing(ctx: Context, P, Q):
    """The reference's Tate pairing (curve/pairing.rs:33-54) of the device-resident packed points P[i], Q[i] (uint8 [n, 4]):
    a new uint8 [n, 2] device tensor of (c0, c1).  Synchronous; raises RonkPanic where the reference panics on any pair."""
    import torch
    for t in (P, Q):
        assert t.is_cuda and t.dtype == torch.uint8 and t.is_contiguous()
    n = P.numel() // 4
    assert Q.numel() == 4 * n
    out = torch.empty((n, 2), dtype=torch.uint8, device=P.device)
    ctx.call("ronk_pairing_pluto_ext", _lib._ptr(P), _lib._ptr(Q), n, _lib._ptr(out))
    return out


def kzg_check(ctx: Context, C, Pi, z, v, g1_srs, g2_srs):
    """kzg::check (kzg/setup.rs:81-103) of every row on device tensors: commitments C and proofs Pi (uint8 [n, 4]),
    points z and values v (uint8 [n], F17 residues), the SRS points g1_srs and g2_srs (uint8 [k, 4]).  A new uint8 [n]
    device tensor, 1 where the row verifies.  Synchronous; raises RonkPanic where the reference panics on any row."""
    import torch
    for t in (C, Pi, z, v, g1_srs, g2_srs):
        assert t.is_cuda and t.dtype == torch.uint8 and t.is_contiguous()
    n = z.numel()
    assert C.numel() == Pi.numel() == 4 * n and v.numel() == n
    ok = torch.empty(n, dtype=torch.uint8, device=z.device)
    ctx.call("ronk_kzg_check_pluto_ext_batch", _lib._ptr(C), _lib._ptr(Pi), _lib._ptr(z), _lib._ptr(v), n, _lib._ptr(g1_srs),
             g1_srs.numel() // 4, _lib._ptr(g2_srs), g2_srs.numel() // 4, _lib._ptr(ok))
    return ok


def poseidon_permute_(ctx: Context, states, cfg, p: int | None = None):
    """The reference's Poseidon permutation (hashes/poseidon/mod.rs:137-149) of every row of states, a contiguous
    [batch, width] device tensor, in place, in one launch.  cfg: a hashes.PoseidonConfig; p defaults to its field's
    modulus (Goldilocks for plain-int constants).  Asynchronous on the context's stream."""
    _check_u64(states)
    p = cfg.modulus(p)
    assert states.dim() == 2 and states.shape[1] == cfg.width, "states is a [batch, width] tensor"
    ctx.call("ronk_poseidon_permute_u64", *cfg.args(ctx, p), _lib._ptr(states), states.shape[0])
    return states


def poseidon_hash(ctx: Context, rows, cfg, p: int | None = None):
    """Poseidon::hash (mod.rs:137-149) of every row of rows ([batch, k] device tensor, k ≤ width): zero-padded to width,
    permuted, word 1.  A new [batch] tensor.  The padding and the column are torch operations on the current stream,
    which the context is expected to share, as for every tensor this module allocates."""
    import torch
    _check_u64(rows)
    assert rows.dim() == 2, "rows is a [batch, k] tensor"
    if rows.shape[1] > cfg.width:
        raise _lib.RonkPanic(_lib.EINVAL, "state longer than the hash width (poseidon/mod.rs:138 underflows)")
    states = torch.zeros((rows.shape[0], cfg.width), dtype=torch.int64, device=rows.device)
    states[:, :rows.shape[1]] = rows
    poseidon_permute_(ctx, states, cfg, p)
    return states[:, 1].contiguous()


def poseidon_sponge(ctx: Context, rows, n_out: int, rate: int, cfg, p: int | None = None):
    """One fresh PoseidonSponge (hashes/poseidon/sponge.rs) per row of rows ([batch, len] device tensor): absorb the row,
    start squeezing, squeeze n_out words.  A new [batch, n_out] tensor; asynchronous on the context's stream."""
    import torch
    _check_u64(rows)
    assert rows.dim() == 2, "rows is a [batch, len] tensor"
    p = cfg.modulus(p)
    out = torch.empty((rows.shape[0], n_out), dtype=torch.int64, device=rows.device)
    ctx.call("ronk_poseidon_sponge_u64", *cfg.args(ctx, p), rate, _lib._ptr(rows), rows.shape[1], rows.shape[0],
             _lib._ptr(out), n_out)
    return out


def _check_u8(t):
    import torch
    assert t.is_cuda and t.dtype == torch.uint8 and t.is_contiguous(), "need a contiguous CUDA uint8 tensor"


def merkle_levels(n: int):
    """(sizes, offsets) of the levels of a SHA-256 Merkle tree of n ≥ 1 leaves, leaf level first, as the node buffer of
    merkle_build lays them out: level l holds ⌈n / 2^l⌉ nodes from node offsets[l] on, l = 0 … L, L = ⌈log2 n⌉."""
    sizes = [n]
    while sizes[-1] > 1:
        sizes.append((sizes[-1] + 1) // 2)
    offsets = [sum(sizes[:l]) for l in range(len(sizes))]
    return sizes, offsets


def _messages(data, offsets):
    _check_u8(data)
    _check_u64(offsets)
    assert offsets.dim() == 1 and offsets.numel() >= 1, "offsets holds n + 1 entries"
    return offsets.numel() - 1


def sha256(ctx: Context, data, offsets):
    """SHA-256 (hashes/sha.rs:88-201) of each message data[offsets[i]:offsets[i+1]] of a uint8 device tensor; offsets is
    an int64 device tensor of n + 1 entries.  A new [n, 32] uint8 tensor; one launch, then one synchronisation to check
    the offsets (RonkPanic when they decrease or pass the data)."""
    import torch
    n = _messages(data, offsets)
    out = torch.empty((n, 32), dtype=torch.uint8, device=data.device)
    ctx.call("ronk_sha256", _lib._ptr(data) if data.numel() else None, data.numel(), _lib._ptr(offsets), n, _lib._ptr(out))
    return out


def merkle_build(ctx: Context, data, offsets):
    """MerkleTree::new (tree/merkle.rs:31-60) over the messages of data and offsets (as sha256 takes them): (nodes, level
    offsets).  nodes is a new [Σ sizes, 32] uint8 tensor holding every level, leaf level first; level l starts at row
    level_offsets[l], and the root is the last row.  n = 0 gives an empty buffer and no levels."""
    import torch
    n = _messages(data, offsets)
    if n == 0:
        return torch.empty((0, 32), dtype=torch.uint8, device=data.device), []
    sizes, level_offsets = merkle_levels(n)
    nodes = torch.empty((sum(sizes), 32), dtype=torch.uint8, device=data.device)
    ctx.call("ronk_merkle_build_sha256", _lib._ptr(data) if data.numel() else None, data.numel(), _lib._ptr(offsets), n,
             _lib._ptr(nodes))
    return nodes, level_offsets


def merkle_proofs(ctx: Context, nodes, n: int, indices):
    """get_proof (merkle.rs:66-81) of each leaf index (int64 device tensor [m]) against the tree of n leaves that
    merkle_build wrote into nodes: (siblings [m, L, 32] uint8, sides [m, L] uint8, 0 = Left and 1 = Right).  An index at
    which the reference panics raises RonkPanic."""
    import torch
    _check_u8(nodes)
    _check_u64(indices)
    depth = len(merkle_levels(n)[0]) - 1 if n else 0
    m = indices.numel()
    sib = torch.empty((m, depth, 32), dtype=torch.uint8, device=nodes.device)
    sides = torch.empty((m, depth), dtype=torch.uint8, device=nodes.device)
    ctx.call("ronk_merkle_proofs_sha256", _lib._ptr(nodes), n, _lib._ptr(indices), m, _lib._ptr(sib), _lib._ptr(sides))
    return sib, sides


def merkle_verify(ctx: Context, root, data, offsets, siblings, sides):
    """prove (merkle.rs:84-98) of each message of data and offsets with its proof (siblings [m, depth, 32], sides
    [m, depth] uint8 device tensors) against root (32-byte uint8 device tensor): a new [m] bool tensor."""
    import torch
    m = _messages(data, offsets)
    _check_u8(root)
    _check_u8(siblings)
    _check_u8(sides)
    assert root.numel() == 32, "root is 32 bytes"
    assert sides.dim() == 2 and sides.shape[0] == m and siblings.shape == (m, sides.shape[1], 32), \
        "siblings [m, depth, 32] and sides [m, depth]"
    depth = sides.shape[1]
    ok = torch.empty(m, dtype=torch.uint8, device=data.device)
    ctx.call("ronk_merkle_verify_sha256", _lib._ptr(root), _lib._ptr(data) if data.numel() else None, data.numel(),
             _lib._ptr(offsets), m, _lib._ptr(siblings) if siblings.numel() else None,
             _lib._ptr(sides) if sides.numel() else None, depth, _lib._ptr(ok))
    return ok.bool()


def msm_buckets(ctx: Context, points, scalars) -> bytes:
    out = np.empty(68, dtype=np.uint8)
    ctx.call("ronk_msm_pluto_ext_buckets", _lib._ptr(points), points.numel() // 4, _lib._ptr(scalars),
             scalars.numel(), _lib._ptr(out))
    return out.tobytes()


def msm_combine(ctx: Context, bucket_sets: bytes) -> bytes:
    arr = np.frombuffer(bucket_sets, dtype=np.uint8).copy()
    out = np.empty(4, dtype=np.uint8)
    ctx.call("ronk_msm_combine_buckets_host", _lib._ptr(arr), len(arr) // 68, _lib._ptr(out))
    return out.tobytes()
