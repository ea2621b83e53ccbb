"""Host-side mirror of ronkathon's `tree::merkle` (src/tree/merkle.rs): `MerkleTree`, `Proof` and `LeftOrRight`, with
SHA-256 as the reference hashes.

Every digest runs in libronk_b200.so on the default context: the tree is built by `ronk_merkle_build_sha256_host`,
proofs are gathered by `ronk_merkle_proofs_sha256_host` and checked by `ronk_merkle_verify_sha256_host`.  The reference's
panics raise `RonkPanic`.  `ops.merkle_build`, `ops.merkle_proofs` and `ops.merkle_verify` are the batched device paths.
"""
from __future__ import annotations

import enum

import numpy as np

from . import _lib
from ._lib import RonkPanic
from .ops import merkle_levels


class LeftOrRight(enum.IntEnum):
    """The side of a proof's sibling (merkle.rs:14-21); the values are the side bytes of the C entries."""
    Left = 0
    Right = 1


class Proof(list):
    """Proof (merkle.rs:25-26): a list of (sibling digest, LeftOrRight), leaf level first."""


def _bytes(leaf) -> bytes:
    return leaf.encode() if isinstance(leaf, str) else bytes(leaf)


def _batch(messages):
    """(data, offsets) of the messages as the C entries take them."""
    data = np.frombuffer(b"".join(messages), dtype=np.uint8)
    offsets = np.zeros(len(messages) + 1, dtype=np.uint64)
    np.cumsum([len(m) for m in messages], out=offsets[1:])
    return data, offsets


def _ptr(a):
    return _lib._ptr(a) if a.size else None


class MerkleTree:
    """MerkleTree::new (merkle.rs:31-60) of leaves given as str (hashed as their UTF-8 bytes, as `as_bytes()`) or bytes.
    `hashes` holds the levels root first, as the reference stores them; a tree of no leaves has one empty level."""

    def __init__(self, leaves):
        self.leaves = list(leaves)
        n = len(self.leaves)
        self._n = n
        if n == 0:
            self._nodes = np.zeros(0, dtype=np.uint8)
            self.hashes = [[]]
            return
        data, offsets = _batch([_bytes(v) for v in self.leaves])
        sizes, offs = merkle_levels(n)
        self._nodes = np.empty(sum(sizes) * 32, dtype=np.uint8)
        _lib.default_context().call("ronk_merkle_build_sha256_host", _ptr(data), data.size, _lib._ptr(offsets), n,
                                    _lib._ptr(self._nodes))
        raw = self._nodes.tobytes()
        self.hashes = [[raw[32 * (offs[l] + i):32 * (offs[l] + i + 1)] for i in range(sizes[l])]
                       for l in reversed(range(len(sizes)))]

    def root_hash(self) -> bytes:
        """root_hash (merkle.rs:63): the single node of the top level; a tree of no leaves panics."""
        if not self.hashes[0]:
            raise RonkPanic(_lib.EINVAL, "index out of bounds: the tree has no leaves (merkle.rs:63)")
        return self.hashes[0][0]

    def get_proof(self, leaf_index: int) -> Proof:
        """get_proof (merkle.rs:66-81): the sibling and its side at every level below the root.  Panics where a sibling
        index lies past its level, which the path of every unpaired last node reaches."""
        depth = len(self.hashes) - 1
        if depth == 0:
            return Proof()
        idx = np.array([leaf_index], dtype=np.uint64)
        sib = np.empty(32 * depth, dtype=np.uint8)
        sides = np.empty(depth, dtype=np.uint8)
        _lib.default_context().call("ronk_merkle_proofs_sha256_host", _lib._ptr(self._nodes), self._n, _lib._ptr(idx), 1,
                                    _lib._ptr(sib), _lib._ptr(sides))
        raw = sib.tobytes()
        return Proof((raw[32 * l:32 * (l + 1)], LeftOrRight(int(sides[l]))) for l in range(depth))

    def prove(self, value, proof) -> bool:
        """prove (merkle.rs:84-98): folds the digest of value through the proof and compares it with the root."""
        root = np.frombuffer(self.root_hash(), dtype=np.uint8)
        data, offsets = _batch([_bytes(value)])
        steps = list(proof)
        sib = np.frombuffer(b"".join(bytes(s) for s, _ in steps), dtype=np.uint8)
        if sib.size != 32 * len(steps):
            raise ValueError("every sibling is a 32-byte digest")
        sides = np.array([int(LeftOrRight(side)) for _, side in steps], dtype=np.uint8)
        ok = np.zeros(1, dtype=np.uint8)
        _lib.default_context().call("ronk_merkle_verify_sha256_host", _lib._ptr(root), _ptr(data), data.size,
                                    _lib._ptr(offsets), 1, _ptr(sib), _ptr(sides), len(steps), _lib._ptr(ok))
        return bool(ok[0])
