"""ctypes front-end for tests/pairing_oracle.c: the reference's Tate pairing and kzg::check restated in C.

TEST INFRASTRUCTURE ONLY.  The library is compiled once per process into a temporary directory, so the tests need no
write access to the tree."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
PU8, SZ = C.POINTER(C.c_uint8), C.c_size_t
_lib = None


class OraclePanic(Exception):
    """Raised where the reference would panic."""


def lib():
    global _lib
    if _lib is None:
        so = os.path.join(tempfile.mkdtemp(prefix="ronk_pairing_oracle_"), "libpairing_oracle.so")
        subprocess.check_call(["gcc", "-O2", "-std=gnu11", "-fPIC", "-shared", "-Wall", "-o", so,
                               os.path.join(HERE, "pairing_oracle.c")])
        _lib = C.CDLL(so)
        _lib.orc_pairing.argtypes = [PU8, PU8, PU8]
        _lib.orc_pairing.restype = C.c_int
        _lib.orc_kzg_check.argtypes = [PU8, PU8, C.c_uint, C.c_uint, PU8, SZ, PU8, SZ, PU8]
        _lib.orc_kzg_check.restype = C.c_int
        _lib.orc_point_order.argtypes = [PU8]
        _lib.orc_point_order.restype = C.c_uint
        _lib.orc_pairing_many.argtypes = [PU8, PU8, SZ, PU8, PU8]
        _lib.orc_kzg_check_many.argtypes = [PU8, PU8, PU8, PU8, SZ, PU8, SZ, PU8, SZ, PU8, PU8]
    return _lib


def _u8(x) -> np.ndarray:
    if isinstance(x, (bytes, bytearray)):
        return np.frombuffer(bytes(x), dtype=np.uint8).copy()
    if isinstance(x, np.ndarray):
        return np.ascontiguousarray(x, dtype=np.uint8).reshape(-1)
    return np.frombuffer(b"".join(bytes(p) for p in x), dtype=np.uint8).copy()


def _p(a):
    return a.ctypes.data_as(PU8)


def pairing(p, q):
    """(c0, c1) of pairing(p, q) for packed points; OraclePanic where the reference panics."""
    a, b, out = _u8(p), _u8(q), np.empty(2, np.uint8)
    if lib().orc_pairing(_p(a), _p(b), _p(out)):
        raise OraclePanic("pairing panics")
    return int(out[0]), int(out[1])


def point_order(p) -> int:
    """Order of a packed curve point (1 for Infinity); 0 for bytes off the curve."""
    return int(lib().orc_point_order(_p(_u8(p))))


def pairing_many(P, Q):
    """Row-wise pairing of packed points uint8 [n, 4]: (values uint8 [n, 2], panics bool [n])."""
    a, b = _u8(P), _u8(Q)
    n = a.size // 4
    out, panic = np.zeros((n, 2), np.uint8), np.empty(n, np.uint8)
    lib().orc_pairing_many(_p(a), _p(b), n, _p(out), _p(panic))
    return out, panic.astype(bool)


def kzg_check(c, q, z, v, g1_srs, g2_srs) -> bool:
    """kzg::check(c, q, z, v, g1_srs, g2_srs); OraclePanic where the reference panics."""
    g1, g2 = _u8(g1_srs), _u8(g2_srs)
    a, b, ok = _u8(c), _u8(q), np.empty(1, np.uint8)
    if lib().orc_kzg_check(_p(a), _p(b), z, v, _p(g1), g1.size // 4, _p(g2), g2.size // 4, _p(ok)):
        raise OraclePanic("kzg::check panics")
    return bool(ok[0])


def kzg_check_many(C_, Q, z, v, g1_srs, g2_srs):
    """Row-wise kzg::check: (ok bool [n], panics bool [n])."""
    a, b = _u8(C_), _u8(Q)
    z, v = np.ascontiguousarray(z, np.uint8), np.ascontiguousarray(v, np.uint8)
    g1, g2 = _u8(g1_srs), _u8(g2_srs)
    n = z.size
    ok, panic = np.zeros(n, np.uint8), np.empty(n, np.uint8)
    lib().orc_kzg_check_many(_p(a), _p(b), _p(z), _p(v), n, _p(g1), g1.size // 4, _p(g2), g2.size // 4, _p(ok), _p(panic))
    return ok.astype(bool), panic.astype(bool)
