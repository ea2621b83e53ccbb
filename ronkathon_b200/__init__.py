"""ronkathon_b200 — H100-native (sm_90a) finite-field polynomial engine: the drop-in for
pluto/ronkathon's PrimeField / Polynomial / kzg::commit hot path.

The compute lives in `libronk_b200.so` (hand-written CUDA behind the C ABI in
include/ronk_b200.h).  This package is the host-side mirror of the reference's surface:

    field.PrimeField(P), PlutoBaseField, PlutoScalarField, GoldilocksField
    polynomial.Polynomial (Monomial / Lagrange bases: evaluate, dft, fft, ifft, + - * / %)
    curve.AffinePoint, kzg.setup / commit / open_
    ops.*  — device-resident operator API on torch tensors (what bench.py times)
    dist.* — multi-GPU sharding (batch ranges, one-all-to-all distributed transform, MSM all-gather)
    codes.* — next rows: Reed–Solomon encode, Shamir-style multi-point evaluation
    hashes.PoseidonConfig / Poseidon / PoseidonSponge — the reference's Poseidon over any prime field
    hashes.Sha256, tree.MerkleTree — the reference's SHA-256 and its Merkle tree

There is no CPU fallback: importing works anywhere, but creating a Context needs an H100.
"""
from ._lib import GOLDILOCKS, Context, RonkError, RonkPanic, default_context, set_default_context  # noqa: F401
from .curve import AffinePoint, G1_GENERATOR, G2_GENERATOR  # noqa: F401
from .field import GoldilocksField, PlutoBaseField, PlutoScalarField, PrimeField  # noqa: F401
from .polynomial import Lagrange, Monomial, Polynomial  # noqa: F401
from . import codes, dist, hashes, kzg, ops, tree  # noqa: F401
