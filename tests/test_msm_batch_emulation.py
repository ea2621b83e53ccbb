"""CPU-tier check of the per-point and per-scalar tests of the batched commit (ronk_msm_pluto_ext_batch): coord_term and
scalar4_over of ronkathon_b200/csrc/msm_curve.cuh compiled for the host (tests/emu/msm_batch_emu.cpp, a test fixture,
never part of the product), against the group tables and the oracle."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle

HERE = os.path.dirname(os.path.abspath(__file__))
PU8, PU32 = C.POINTER(C.c_uint8), C.POINTER(C.c_uint32)
MSM_BINS, EXP = 20402, 102


@pytest.fixture(scope="module")
def emu():
    src = os.path.join(HERE, "emu", "msm_batch_emu.cpp")
    so = os.path.join(HERE, "emu", "libmsm_batch_emu.so")
    hdrs = [os.path.join(HERE, "..", "ronkathon_b200", "csrc", h) for h in ("msm_curve.cuh", "field.cuh")]
    newest = max(os.path.getmtime(x) for x in [src] + hdrs)
    if not os.path.exists(so) or os.path.getmtime(so) < newest:
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", so, src])
    lib = C.CDLL(so)
    lib.emu_group_tables.argtypes = [PU32, PU32]
    lib.emu_group_tables.restype = C.c_int
    lib.emu_coord_terms.argtypes = [PU32, PU32, C.c_uint64, PU8, PU8, PU8]
    lib.emu_scalar4_over.argtypes = [PU32, C.c_uint64, PU8]
    return lib


@pytest.fixture(scope="module")
def tables(emu):
    bintab = np.empty(MSM_BINS + 2, dtype=np.uint32)
    pttab = np.empty(EXP * EXP, dtype=np.uint32)
    assert emu.emu_group_tables(bintab.ctypes.data_as(PU32), pttab.ctypes.data_as(PU32)) == 1
    return bintab, pttab


def _terms(emu, bintab, words):
    words = np.ascontiguousarray(words, dtype=np.uint32)
    on, a, b = (np.empty(len(words), dtype=np.uint8) for _ in range(3))
    emu.emu_coord_terms(bintab.ctypes.data_as(PU32), words.ctypes.data_as(PU32), len(words), on.ctypes.data_as(PU8),
                        a.ctypes.data_as(PU8), b.ctypes.data_as(PU8))
    return on, a, b


def _over(emu, words):
    words = np.ascontiguousarray(words, dtype=np.uint32)
    out = np.empty(len(words), dtype=np.uint8)
    emu.emu_scalar4_over(words.ctypes.data_as(PU32), len(words), out.ctypes.data_as(PU8))
    return out.astype(bool)


def test_scalar_check_every_byte_at_every_position(emu):
    """A word is flagged exactly when one of its four scalars is ≥ 17: every byte value at each position, beside F17
    residues, beside other bytes ≥ 17 and beside bytes ≥ 128 (whose carry reaches the bytes above them)."""
    rng = np.random.default_rng(31)
    v = np.arange(256, dtype=np.uint32)
    for pos in range(4):
        for fill in (0, 16, 17, 127, 128, 255, None):
            others = rng.integers(0, 17, (256, 4)).astype(np.uint32) if fill is None else np.full((256, 4), fill, np.uint32)
            others[:, pos] = v
            words = others[:, 0] | others[:, 1] << 8 | others[:, 2] << 16 | others[:, 3] << 24
            want = (others >= 17).any(axis=1)
            assert np.array_equal(_over(emu, words), want), (pos, fill)
    # every word of four F17 residues passes
    r = np.arange(17, dtype=np.uint32)
    q = np.stack(np.meshgrid(r, r, r, r, indexing="ij"), axis=-1).reshape(-1, 4)
    assert not _over(emu, q[:, 0] | q[:, 1] << 8 | q[:, 2] << 16 | q[:, 3] << 24).any()
    words = rng.integers(0, 1 << 32, 100_000, dtype=np.uint64).astype(np.uint32)
    want = np.stack([(words >> (8 * k)) & 0xFF for k in range(4)], axis=1).max(axis=1) >= 17
    assert np.array_equal(_over(emu, words), want)


def test_coord_terms_match_the_group_tables_on_the_whole_group(emu, tables):
    """Every point a·G1 + b·G2 of E(F_101²) gets its own (a, b) back; Infinity is not a term (coordinates 0, and the
    kernels do not flag it)."""
    bintab, pttab = tables
    on, a, b = _terms(emu, bintab, pttab)
    k = np.arange(EXP * EXP)
    assert not on[0] and a[0] == 0 and b[0] == 0 and int(pttab[0]) == 0xFFFFFFFF
    assert on[1:].all()
    assert np.array_equal(a[1:], (k[1:] // EXP).astype(np.uint8)) and np.array_equal(b[1:], (k[1:] % EXP).astype(np.uint8))


def test_coord_terms_reject_what_the_reference_rejects(emu, tables):
    """A word is a term exactly when its coordinates are canonical and it lies on y² = x³ + 3 (curve/mod.rs:130-139):
    curve points with one coordinate byte changed, non-canonical bytes (101, 127, 128, 255) in every position, and random
    words."""
    bintab, pttab = tables
    rng = np.random.default_rng(32)
    pts = pttab[1 + rng.integers(0, EXP * EXP - 1, 3000)]
    cand = []
    for i, w in enumerate(pts):
        pos = i % 4
        cand.append(int(w) ^ (int(rng.integers(1, 128)) << (8 * pos)))                  # one coordinate changed
        bad = (101, 127, 128, 255)[i % 4]
        cand.append((int(w) & ~(0xFF << (8 * pos))) | (bad << (8 * pos)))               # non-canonical
    cand += [int(x) for x in rng.integers(0, 1 << 32, 3000, dtype=np.uint64)]
    cand += [int(x) | (int(y) << 8) | (int(z) << 16) | (int(t) << 24) for x, y, z, t in rng.integers(0, 101, (3000, 4))]
    cand = np.array(cand, dtype=np.uint64).astype(np.uint32)
    on, a, b = _terms(emu, bintab, cand)
    for w, ok, ca, cb in zip(cand, on, a, b):
        P = int(w).to_bytes(4, "little")
        want = P != b"\xff" * 4 and all(c < 101 for c in P) and oracle.on_curve(P)
        assert bool(ok) == want, P
        if ok:
            assert int(pttab[EXP * int(ca) + int(cb)]) == int(w)
        else:
            assert ca == 0 and cb == 0
