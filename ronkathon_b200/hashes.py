"""Host-side mirror of ronkathon's `hashes::poseidon` (src/hashes/poseidon/{mod,sponge}.rs): `PoseidonConfig`,
`Poseidon::hash` and `PoseidonSponge` with its Init → Absorbing → Squeezing typestate, over any prime field; and of
`hashes::sha::Sha256` (src/hashes/sha.rs), whose digests run in libronk_b200.so (`ronk_sha256`).

Every permutation runs in libronk_b200.so (`ronk_poseidon_permute_u64`).  The single-object classes keep their state on
the host and permute a batch of one state per call, which is literal and slow; `ops.poseidon_permute_`,
`ops.poseidon_hash` and `ops.poseidon_sponge` are the batched device paths, as `ops.sha256` is for SHA-256.  The other
hashes of `src/hashes` (SHA-512, SHA-3, GHASH) are not mirrored.
"""
from __future__ import annotations

import weakref

import numpy as np

from . import _lib
from ._lib import GOLDILOCKS, RonkPanic


def _value(x) -> int:
    return int(getattr(x, "value", x))


def _field_of(items):
    """The PrimeField class of the first field element among items, or None when all are plain ints."""
    for x in items:
        if hasattr(x, "ORDER"):
            return type(x)
    return None


class PoseidonConfig:
    """PoseidonConfig::new (mod.rs:39-56), with the reference's argument order.  rc and mds hold ints or field elements;
    `field` is their PrimeField class, found from the elements when not given.  A config without a field serves any p
    through the ops functions, which reduce its constants mod p as F::from does."""

    def __init__(self, width: int, alpha: int, num_p: int, num_f: int, rc, mds, field=None):
        if width <= 1:
            raise RonkPanic(_lib.EINVAL, "hash width should be greater than 1 (poseidon/mod.rs:47)")
        if len(mds) != width:
            raise RonkPanic(_lib.EINVAL, "mds matrix should be as long as width (poseidon/mod.rs:48)")
        if len(rc) != (num_p + num_f) * width:
            raise RonkPanic(_lib.EINVAL, "round constants should be equal to number of full and partial rounds "
                                         "(poseidon/mod.rs:49-53)")
        rows = [list(r) for r in mds]
        if any(len(r) != width for r in rows):
            raise ValueError("every MDS row must hold width elements")
        self.width, self.alpha, self.num_p, self.num_f = int(width), int(alpha), int(num_p), int(num_f)
        self.field = field or _field_of(list(rc) + [x for r in rows for x in r])
        self._rc = [_value(v) for v in rc]
        self._mds = [[_value(v) for v in r] for r in rows]
        self._tables = {}                          # p → (rc, mds) reduced mod p
        self._device = weakref.WeakKeyDictionary()  # Context → {p: (rc, mds) device tensors}

    def modulus(self, p: int | None = None) -> int:
        """The p a call runs over: p, else the constants' field, else Goldilocks."""
        if p is None:
            return self.field.ORDER if self.field is not None else GOLDILOCKS
        if self.field is not None and p != self.field.ORDER:
            raise ValueError(f"the constants are elements of {self.field!r}, not of F_{p}")
        return int(p)

    def tables(self, p: int):
        """(rc uint64 [(num_f + num_p)·width], mds uint64 [width, width]) reduced mod p."""
        if p not in self._tables:
            rc = np.array([v % p for v in self._rc], dtype=np.uint64)
            mds = np.array([[v % p for v in r] for r in self._mds], dtype=np.uint64).reshape(self.width, self.width)
            self._tables[p] = (rc, mds)
        return self._tables[p]

    def device_tables(self, ctx, p: int):
        """The constants on ctx's device, uploaded once per (context, p)."""
        import torch
        per_ctx = self._device.setdefault(ctx, {})
        if p not in per_ctx:
            rc, mds = self.tables(p)
            dev = torch.device("cuda", ctx.device)
            t = tuple(torch.from_numpy(a.reshape(-1).view(np.int64).copy()).to(dev) for a in (rc, mds))
            torch.cuda.synchronize(dev)     # the copies ran on torch's stream; the context's stream may be another
            per_ctx[p] = t
        return per_ctx[p]

    def args(self, ctx, p: int):
        """The configuration arguments of the C entries: (p, width, alpha, num_f, num_p, rc, mds)."""
        rc, mds = self.device_tables(ctx, p)
        return (p, self.width, self.alpha, self.num_f, self.num_p, _lib._ptr(rc), _lib._ptr(mds))


def _permute_one(cfg: PoseidonConfig, state: list[int]) -> list[int]:
    """One permutation of a host state through ronk_poseidon_permute_u64 on the default context."""
    from . import ops
    ctx = _lib.default_context()
    p = cfg.modulus()
    s = ops.to_device(np.array(state, dtype=np.uint64), device=f"cuda:{ctx.device}")
    ops.poseidon_permute_(ctx, s.view(1, cfg.width), cfg, p)
    ctx.sync()
    return [int(v) for v in ops.to_host(s)]


class Poseidon:
    """Poseidon (mod.rs:24-150): `Poseidon(width, alpha, num_p, num_f, rc, mds).hash(state)`."""

    def __init__(self, width: int, alpha: int, num_p: int, num_f: int, rc, mds, field=None):
        self.config = PoseidonConfig(width, alpha, num_p, num_f, rc, mds, field)
        if self.config.field is None:
            raise TypeError("give the field: the constants are plain ints")
        self.state = [self.config.field.ZERO] * width

    def _run(self, state: list[int]):
        self.state = [self.config.field(v) for v in _permute_one(self.config, state)]

    def hash(self, state):
        """Poseidon::hash (mod.rs:137-149): zero-pads state to width, permutes it and returns element 1.  A state longer
        than width panics, as the reference's `width - state.len()` underflows."""
        state = list(state)
        if len(state) > self.config.width:
            raise RonkPanic(_lib.EINVAL, "state longer than the hash width (poseidon/mod.rs:138 underflows)")
        p = self.config.field.ORDER
        self._run([_value(v) % p for v in state] + [0] * (self.config.width - len(state)))
        return self.state[1]


class SpongeStateError(RuntimeError):
    """A sponge call its typestate does not offer: the reference's `Err` from `absorb` on a squeezing sponge and from
    `squeeze` on an absorbing one (sponge.rs:280-294), and the calls its typestates lack (a compile error there)."""


class PoseidonSponge:
    """PoseidonSponge (sponge.rs:71-294): `PoseidonSponge(width, alpha, num_p, num_f, rate, rc, mds)`, then
    start_absorbing() → absorb(...)* → start_squeezing() → squeeze(n)*.  The state lives on the host; each permutation
    is one device call."""

    def __init__(self, width: int, alpha: int, num_p: int, num_f: int, rate: int, rc, mds, field=None):
        self.poseidon = Poseidon(width, alpha, num_p, num_f, rc, mds, field)
        if not 0 < rate <= width:
            raise RonkPanic(_lib.EINVAL, "rate must be in [1, width]: the reference underflows width - rate or never "
                                         "finishes absorbing")
        self.rate, self.capacity = rate, width - rate
        self.absorb_index = self.squeeze_index = 0
        self.sponge_state = "init"
        self._s = [0] * width

    def _require(self, state: str, what: str):
        if self.sponge_state != state:
            raise SpongeStateError(f"{what} needs a sponge in the {state} state; this one is {self.sponge_state}")

    def permute(self):
        self._s = _permute_one(self.poseidon.config, self._s)
        self.poseidon.state = [self.poseidon.config.field(v) for v in self._s]
        self.absorb_index = 0

    def start_absorbing(self):
        self._require("init", "start_absorbing")
        self.sponge_state = "absorbing"
        return self

    def _add(self, at: int, values):
        """state[at + i] += values[i], through the device's field addition."""
        if not values:
            return
        a = np.array(self._s[at:at + len(values)], dtype=np.uint64)
        b = np.array(values, dtype=np.uint64)
        out = np.empty(len(values), dtype=np.uint64)
        _lib.default_context().call("ronk_field_binop_u64_host", 0, self.poseidon.config.field.ORDER, _lib._ptr(a),
                                    _lib._ptr(b), _lib._ptr(out), len(values))
        self._s[at:at + len(values)] = [int(v) for v in out]

    def absorb(self, elements):
        """absorb (sponge.rs:142-194): permutes after each full rate-chunk."""
        if self.sponge_state == "squeezing":
            raise SpongeStateError("sponge is in squeezing state")
        self._require("absorbing", "absorb")
        p = self.poseidon.config.field.ORDER
        rest = [_value(v) % p for v in elements]
        if self.absorb_index + len(rest) <= self.rate:
            self._add(self.capacity + self.absorb_index, rest)
            self.absorb_index += len(rest)
            return self
        if self.absorb_index != 0:
            take = self.rate - self.absorb_index
            self._add(self.capacity + self.absorb_index, rest[:take])
            rest = rest[take:]
            self.permute()
        full = len(rest) // self.rate * self.rate
        for c in range(0, full, self.rate):
            self._add(self.capacity + self.absorb_index, rest[c:c + self.rate])
            self.permute()
        if full < len(rest):
            self._add(self.capacity, rest[full:])
            self.absorb_index = len(rest) - full
        return self

    def start_squeezing(self):
        """start_squeezing (sponge.rs:198-213): permutes when a chunk is partly absorbed."""
        self._require("absorbing", "start_squeezing")
        if self.absorb_index != 0:
            self.permute()
        self.sponge_state = "squeezing"
        return self

    def squeeze(self, n: int):
        """squeeze (sponge.rs:244-274): n elements from state[capacity + squeeze_index ..], permuting at each rate."""
        if self.sponge_state == "absorbing":
            raise SpongeStateError("sponge is in squeeze state")
        self._require("squeezing", "squeeze")
        F = self.poseidon.config.field
        out = []
        while True:
            left = n - len(out)
            start = self.capacity + self.squeeze_index
            if self.squeeze_index + left <= self.rate:
                out += self._s[start:start + left]
                self.squeeze_index += left
                return [F(v) for v in out]
            size = min(left, self.rate - self.squeeze_index)
            out += self._s[start:start + size]
            self.squeeze_index += size
            if self.squeeze_index == self.rate:
                self.permute()
                self.squeeze_index = 0


class Sha256:
    """Sha256 (sha.rs:203-232): `Sha256().digest(input)` is the 32-byte SHA-256 of the bytes, computed on the device as a
    batch of one message (`ronk_sha256_host` on the default context)."""

    def digest(self, data) -> bytes:
        m = np.frombuffer(bytes(data), dtype=np.uint8)
        offsets = np.array([0, m.size], dtype=np.uint64)
        out = np.empty(32, dtype=np.uint8)
        _lib.default_context().call("ronk_sha256_host", _lib._ptr(m) if m.size else None, m.size, _lib._ptr(offsets), 1,
                                    _lib._ptr(out))
        return out.tobytes()
