"""CPU tier: the SHA-256 and Merkle routines of ronk_sha256 / ronk_merkle_build_sha256 (ronkathon_b200/csrc/sha256.cuh,
compiled for the host by tests/emu/sha256_emu.cpp, a test fixture, never part of the product) against Python's
hashlib: every message length 0 … 300 at each of the 4 start alignments, the node path with its constant padding block,
and the in-CTA level reduction on spans whose level end is odd or even."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np
import pytest

import merkle_oracle as mo

HERE = os.path.dirname(os.path.abspath(__file__))
PU8, P64 = C.POINTER(C.c_uint8), C.POINTER(C.c_uint64)


@pytest.fixture(scope="module")
def emu():
    so = os.path.join(tempfile.mkdtemp(prefix="ronk_sha256_emu_"), "libsha256_emu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", so,
                           os.path.join(HERE, "emu", "sha256_emu.cpp")])
    lib = C.CDLL(so)
    lib.emu_sha_k.restype = lib.emu_sha_kw_pad64.restype = C.c_uint32
    lib.emu_sha_k.argtypes = lib.emu_sha_kw_pad64.argtypes = [C.c_int]
    lib.emu_sha256.argtypes = [PU8, P64, C.c_uint64, PU8]
    lib.emu_sha_node.argtypes = [PU8, PU8, PU8]
    lib.emu_merkle_span.argtypes = [PU8, C.c_uint32, C.c_uint32, PU8]
    lib.emu_merkle_span.restype = C.c_uint64
    return lib


def _u8(a):
    return a.ctypes.data_as(PU8)


def _aligned(nbytes, rng):
    """Random bytes in a buffer whose element 0 is 16-byte aligned."""
    raw = rng.integers(0, 256, nbytes + 16, dtype=np.uint8)
    skip = (-raw.ctypes.data) % 16
    return raw[skip:skip + nbytes]


def test_every_length_at_every_alignment(emu):
    rng = np.random.default_rng(1)
    lengths = np.arange(0, 301, dtype=np.uint64)
    for align in range(4):
        # messages back to back, the first at `align`, each then at the alignment its predecessors leave
        buf = _aligned(int(align + lengths.sum()) + 8, rng)
        off = np.concatenate([[align], align + np.cumsum(lengths)]).astype(np.uint64)
        out = np.zeros(32 * len(lengths), np.uint8)
        emu.emu_sha256(_u8(buf), off.ctypes.data_as(P64), len(lengths), _u8(out))
        for i, n in enumerate(lengths):
            msg = buf[int(off[i]):int(off[i + 1])].tobytes()
            assert out[32 * i:32 * i + 32].tobytes() == hashlib.sha256(msg).digest(), (align, int(n))
        # and each length alone at exactly this alignment
        for n in (0, 1, 3, 4, 55, 56, 63, 64, 65, 119, 120, 300):
            single = np.array([align, align + n], np.uint64)
            emu.emu_sha256(_u8(buf), single.ctypes.data_as(P64), 1, _u8(out))
            assert out[:32].tobytes() == hashlib.sha256(buf[align:align + n].tobytes()).digest(), (align, n)


def test_padding_block_constants_follow_from_k(emu):
    k = [emu.emu_sha_k(i) for i in range(64)]
    w = [0x80000000] + [0] * 14 + [512]
    rot = lambda x, n: ((x >> n) | (x << (32 - n))) & 0xFFFFFFFF  # noqa: E731
    for i in range(16, 64):
        s0 = rot(w[i - 15], 7) ^ rot(w[i - 15], 18) ^ (w[i - 15] >> 3)
        s1 = rot(w[i - 2], 17) ^ rot(w[i - 2], 19) ^ (w[i - 2] >> 10)
        w.append((s1 + w[i - 7] + s0 + w[i - 16]) & 0xFFFFFFFF)
    assert [emu.emu_sha_kw_pad64(i) for i in range(64)] == [(k[i] + w[i]) & 0xFFFFFFFF for i in range(64)]


def test_node_path_on_random_pairs(emu):
    rng = np.random.default_rng(2)
    out = np.zeros(32, np.uint8)
    for _ in range(500):
        l, r = rng.integers(0, 256, 32, dtype=np.uint8), rng.integers(0, 256, 32, dtype=np.uint8)
        emu.emu_sha_node(_u8(l), _u8(r), _u8(out))
        assert out.tobytes() == hashlib.sha256(l.tobytes() + r.tobytes()).digest()
    z = np.zeros(32, np.uint8)
    emu.emu_sha_node(_u8(z), _u8(z), _u8(out))
    assert out.tobytes() == hashlib.sha256(bytes(64)).digest()


@pytest.mark.parametrize("cnt", [1, 2, 3, 5, 6, 7, 64, 255, 256, 257, 300, 511, 512])
def test_span_reduction_odd_and_even_ends(emu, cnt):
    rng = np.random.default_rng(cnt)
    leaves = [rng.integers(0, 256, 32, dtype=np.uint8).tobytes() for _ in range(cnt)]
    # the oracle's levels above these digests, 9 of them as a span of the last CTA reduces: a level of one node, the
    # level's odd end, is paired with itself
    levels, cur = [], leaves
    for _ in range(9):
        nxt = [mo.digest(cur[i] + cur[i + 1]) for i in range(0, len(cur) - 1, 2)]
        if len(cur) % 2:
            nxt.append(mo.digest(cur[-1] + cur[-1]))
        levels.append(nxt)
        cur = nxt
    for nlev in sorted({0, 1, (cnt - 1).bit_length(), 9}):
        out = np.zeros(32 * 1024, np.uint8)
        lv = np.frombuffer(b"".join(leaves), np.uint8).copy()
        written = emu.emu_merkle_span(_u8(lv), cnt, nlev, _u8(out))
        want = b"".join(b"".join(level) for level in levels[:nlev])
        assert written * 32 == len(want) and out[:len(want)].tobytes() == want, (cnt, nlev)
