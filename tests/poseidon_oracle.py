"""ctypes front-end for tests/poseidon_oracle.c: the reference's Poseidon permutation and sponge restated in C.

TEST INFRASTRUCTURE ONLY.  The library is compiled once per process into a temporary directory, so the tests need no
write access to the tree."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
P64, SZ, U64 = C.POINTER(C.c_uint64), C.c_size_t, C.c_uint64
PSZ = C.POINTER(C.c_size_t)
_lib = None


class OraclePanic(Exception):
    """Raised where the reference would panic."""


def lib():
    global _lib
    if _lib is None:
        so = os.path.join(tempfile.mkdtemp(prefix="ronk_poseidon_oracle_"), "libposeidon_oracle.so")
        subprocess.check_call(["gcc", "-O2", "-std=gnu11", "-fPIC", "-shared", "-Wall", "-o", so,
                               os.path.join(HERE, "poseidon_oracle.c")])
        _lib = C.CDLL(so)
        _lib.orc_pos_permute.argtypes = [U64, SZ, U64, SZ, SZ, P64, P64, P64, SZ]
        _lib.orc_pos_sponge.argtypes = [U64, SZ, U64, SZ, SZ, P64, P64, SZ, P64, PSZ, SZ, PSZ, SZ, P64]
        _lib.orc_pos_sponge.restype = C.c_int
    return _lib


def _u64(x) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(x, dtype=np.uint64).reshape(-1))


def _p(a, t=P64):
    return a.ctypes.data_as(t)


class Config:
    """PoseidonConfig::new (poseidon/mod.rs:39-56): the three asserts, then constants reduced mod p (F::from)."""

    def __init__(self, p, width, alpha, num_p, num_f, rc, mds):
        if width <= 1:
            raise OraclePanic("hash width should be greater than 1")
        if len(mds) != width:
            raise OraclePanic("mds matrix should be as long as width")
        if len(rc) != (num_p + num_f) * width:
            raise OraclePanic("round constants should be equal to number of full and partial rounds")
        self.p, self.width, self.alpha, self.num_p, self.num_f = p, width, alpha, num_p, num_f
        self.rc = _u64([int(v) % p for v in rc])
        self.mds = _u64([int(v) % p for row in mds for v in row])
        assert self.mds.size == width * width, "every MDS row holds width words"


def permute(cfg: Config, states) -> np.ndarray:
    """Poseidon::hash's rounds on every row of states (uint64 [batch, width]); a new array."""
    s = np.array(states, dtype=np.uint64).reshape(-1, cfg.width).copy()
    lib().orc_pos_permute(cfg.p, cfg.width, cfg.alpha, cfg.num_f, cfg.num_p, _p(cfg.rc), _p(cfg.mds), _p(s), s.shape[0])
    return s


def hash_(cfg: Config, state) -> int:
    """Poseidon::hash (mod.rs:137-149): zero-pad to width (a longer state panics), permute, word 1."""
    if len(state) > cfg.width:
        raise OraclePanic("state longer than width")
    return int(permute(cfg, list(state) + [0] * (cfg.width - len(state)))[0, 1])


def sponge(cfg: Config, rate: int, absorbs, squeezes) -> list[int]:
    """A fresh sponge: absorb each list of `absorbs` in turn, start squeezing, squeeze each count of `squeezes`; the
    squeezed words concatenated."""
    data = _u64([int(v) for a in absorbs for v in a])
    abs_ = np.array([len(a) for a in absorbs] or [0], dtype=np.uintp)
    sq = np.array(list(squeezes) or [0], dtype=np.uintp)
    out = np.zeros(max(int(sq.sum()), 1), dtype=np.uint64)
    if lib().orc_pos_sponge(cfg.p, cfg.width, cfg.alpha, cfg.num_f, cfg.num_p, _p(cfg.rc), _p(cfg.mds), rate,
                            _p(data) if data.size else None, _p(abs_, PSZ), len(absorbs), _p(sq, PSZ), len(squeezes),
                            _p(out)):
        raise OraclePanic("rate must be in [1, width]")
    return [int(v) for v in out[:int(sq.sum())]]


def sponge_rows(cfg: Config, rate: int, rows, n_out: int) -> np.ndarray:
    """One sponge per row of rows (uint64 [batch, len]): one absorb of the row, one squeeze of n_out words."""
    rows = np.asarray(rows, dtype=np.uint64)
    return np.array([sponge(cfg, rate, [list(r)], [n_out]) for r in rows], dtype=np.uint64).reshape(len(rows), n_out)
