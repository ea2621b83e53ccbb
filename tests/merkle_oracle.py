"""TEST INFRASTRUCTURE: src/tree/merkle.rs restated literally on top of Python's hashlib SHA-256, an implementation
independent of the library's kernels.  Nothing under ronkathon_b200/ imports it.

Levels are stored root first, as the reference's `hashes`.  Each panic of the reference raises `Panic`."""
from __future__ import annotations

import hashlib


class Panic(Exception):
    """Where the reference panics (an index out of bounds)."""


def digest(m: bytes) -> bytes:
    return hashlib.sha256(m).digest()


def _as_bytes(v) -> bytes:
    return v.encode() if isinstance(v, str) else bytes(v)


class Tree:
    def __init__(self, leaves):
        """MerkleTree::new (merkle.rs:31-60), odd last node paired with itself."""
        self.leaves = list(leaves)
        hashes = []
        leaf_hashes = [digest(_as_bytes(v)) for v in self.leaves]
        branch = list(leaf_hashes)
        hashes.append(leaf_hashes)
        while len(branch) > 1:
            new = [digest(branch[i] + branch[i + 1]) for i in range(0, len(branch) - 1, 2)]
            if len(branch) % 2 == 1:
                new.append(digest(branch[-1] + branch[-1]))
            hashes.append(new)
            branch = new
        hashes.reverse()
        self.hashes = hashes

    def root_hash(self) -> bytes:
        if not self.hashes[0]:
            raise Panic("hashes[0][0] of an empty level (merkle.rs:63)")
        return self.hashes[0][0]

    def get_proof(self, leaf_index: int):
        """get_proof (merkle.rs:66-81): [(sibling, 'Left' | 'Right')], leaf level first."""
        proof = []
        index = leaf_index
        for level in reversed(self.hashes[1:]):
            side, sib = ("Right", index + 1) if index % 2 == 0 else ("Left", index - 1)
            if sib >= len(level):
                raise Panic(f"index {sib} out of bounds for a level of {len(level)} (merkle.rs:77)")
            proof.append((level[sib], side))
            index //= 2
        return proof

    def prove(self, value, proof) -> bool:
        """prove (merkle.rs:84-98)."""
        h = digest(_as_bytes(value))
        for sib, side in proof:
            h = digest(sib + h) if side == "Left" else digest(h + sib)
        return h == self.root_hash()

    def nodes(self) -> bytes:
        """Every level leaf level first, each contiguous: the node buffer of ronk_merkle_build_sha256."""
        return b"".join(b"".join(level) for level in reversed(self.hashes))
