"""CPU tier: the pairing table and the per-row check of ronk_pairing_pluto_ext / ronk_kzg_check_pluto_ext_batch
(ronkathon_b200/csrc/pairing.cuh, compiled for the host by tests/emu/pairing_emu.cpp, a test fixture, never part of the
product) against the C restatement of the reference in tests/pairing_oracle.c: every entry of the 289 × 289 table, the
reference's Tate values, and the check's group-coordinate points B = g2 − z·GEN and C′ = C − v·g1 over the whole group."""
import ctypes as C
import json
import os
import subprocess
import tempfile

import numpy as np
import pytest

import oracle
import pairing_oracle as po

HERE = os.path.dirname(os.path.abspath(__file__))
PU8, PU16, PU32 = C.POINTER(C.c_uint8), C.POINTER(C.c_uint16), C.POINTER(C.c_uint32)
MSM_BINS, EXP, E17, PANIC = 20402, 102, 289, 0xFF
GEN = bytes([36, 0, 0, 31])


def _p(a, t=PU8):
    return a.ctypes.data_as(t)


def _w(b):
    return int.from_bytes(bytes(b), "little")


@pytest.fixture(scope="module")
def emu():
    so = os.path.join(tempfile.mkdtemp(prefix="ronk_pairing_emu_"), "libpairing_emu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", so,
                           os.path.join(HERE, "emu", "pairing_emu.cpp")])
    lib = C.CDLL(so)
    lib.emu_group_tables.argtypes = [PU32, PU32]
    lib.emu_group_tables.restype = C.c_int
    lib.emu_pairing_table.argtypes = [PU32, PU16, PU8]
    lib.emu_tate.argtypes = [C.c_uint32, C.c_uint32, PU8]
    lib.emu_tate.restype = C.c_int
    lib.emu_sub_smul.argtypes = [PU32, PU32, C.c_uint32, C.c_uint32, C.c_uint32, PU32]
    lib.emu_sub_smul.restype = C.c_int
    lib.emu_kzg_check.argtypes = [PU32, PU8, PU32, PU32, PU8, PU8, C.c_uint64, C.c_uint32, C.c_uint32, PU8, PU8]
    return lib


@pytest.fixture(scope="module")
def tables(emu):
    bintab = np.empty(MSM_BINS + 2, dtype=np.uint32)
    pttab = np.empty(EXP * EXP, dtype=np.uint32)
    assert emu.emu_group_tables(_p(bintab, PU32), _p(pttab, PU32)) == 1
    mu = np.empty(17, dtype=np.uint16)
    T = np.empty(E17 * E17, dtype=np.uint8)
    emu.emu_pairing_table(_p(pttab, PU32), _p(mu, PU16), _p(T))
    return bintab, pttab, mu, T


def _e17_points(pttab):
    """Packed points of E[17] in table order: index 17·(a/6) + b/6 holds a·G1 + b·G2."""
    return np.array([pttab[EXP * 6 * (i // 17) + 6 * (i % 17)] for i in range(E17)], dtype=np.uint32)


def _bytes(words):
    return np.ascontiguousarray(words, dtype=np.uint32).view(np.uint8).reshape(-1, 4)


def test_table_matches_the_oracle_on_every_pair(tables):
    _, pttab, mu, T = tables
    pts = _e17_points(pttab)
    P = np.repeat(pts, E17)
    Q = np.tile(pts, E17)
    vals, panic = po.pairing_many(_bytes(P), _bytes(Q))
    assert np.array_equal(T == PANIC, panic)
    got = mu[T[~panic]]
    want = vals[~panic, 0].astype(np.uint16) | (vals[~panic, 1].astype(np.uint16) << 8)
    assert np.array_equal(got, want)


def test_sentinels_sit_on_infinity_and_the_diagonal(tables):
    _, pttab, _, T = tables
    pts = _e17_points(pttab)
    assert pts[0] == 0xFFFFFFFF and len(set(pts.tolist())) == E17
    T2 = T.reshape(E17, E17)
    expect = np.zeros((E17, E17), dtype=bool)
    expect[0, :] = expect[:, 0] = True
    expect[np.arange(E17), np.arange(E17)] = True
    assert np.array_equal(T2 == PANIC, expect)
    assert int((T2[1:, 1:] == PANIC).sum()) == 288


def test_seventeen_values_the_roots_of_unity(tables):
    _, _, mu, T = tables
    assert sorted(set(T[T != PANIC].tolist())) == list(range(17))
    assert len(set(mu.tolist())) == 17
    for m in mu.tolist():
        x = (m & 0xFF, m >> 8)
        acc = (1, 0)
        for _ in range(17):
            acc = oracle.gf_mul(acc, x)
        assert acc == (1, 0)


def test_tate_kats(emu):
    with open(os.path.join(HERE, "golden", "pairing_kats.json")) as f:
        kats = json.load(f)["tate"]
    for t in kats:
        out = np.empty(2, dtype=np.uint8)
        assert emu.emu_tate(_w(t["p"]), _w(t["q"]), _p(out)) == 1
        assert tuple(out.tolist()) == tuple(t["expected"])


def _oracle_sub_smul(p, s, q):
    return oracle.point_add(p, oracle.point_neg(oracle.point_smul(q, s)))


def test_check_forms_over_the_whole_group(emu, tables):
    """C′ = C − v·g1_srs[0] for every curve point C and every v, and B = g2_srs[1] − z·GEN for every z, against the
    oracle's affine arithmetic (Mul<ScalarField> by repeated addition)."""
    bintab, pttab, _, _ = tables
    g1, g2 = oracle.setup()
    out = np.empty(1, dtype=np.uint32)
    for w in pttab.tolist():
        c = w.to_bytes(4, "little")
        for v in range(17):
            assert emu.emu_sub_smul(_p(bintab, PU32), _p(pttab, PU32), w, v, _w(g1[0]), _p(out, PU32)) == 1
            assert int(out[0]).to_bytes(4, "little") == _oracle_sub_smul(c, v, g1[0]), (c, v)
    for z in range(17):
        assert emu.emu_sub_smul(_p(bintab, PU32), _p(pttab, PU32), _w(g2[1]), z, _w(GEN), _p(out, PU32)) == 1
        assert int(out[0]).to_bytes(4, "little") == _oracle_sub_smul(g2[1], z, GEN), z


def _emu_check(emu, tables, c, q, z, v, g1, g2):
    bintab, _, _, T = tables
    c, q = np.ascontiguousarray(c, np.uint32), np.ascontiguousarray(q, np.uint32)
    z, v = np.ascontiguousarray(z, np.uint8), np.ascontiguousarray(v, np.uint8)
    ok, bad = np.empty(len(z), np.uint8), np.empty(len(z), np.uint8)
    emu.emu_kzg_check(_p(bintab, PU32), _p(T), _p(c, PU32), _p(q, PU32), _p(z), _p(v), len(z), _w(g1), _w(g2), _p(ok), _p(bad))
    return ok.astype(bool), bad.astype(bool)


def test_check_rows_against_the_oracle(emu, tables):
    """Every commitment of the whole group (E[17] and beyond) × every value with one valid proof, and random rows over
    the whole group with random proofs and points: the rows the kernel flags are exactly the rows the reference panics
    on, and every other row gives the reference's bool."""
    _, pttab, _, _ = tables
    g1, g2 = oracle.setup()
    coeffs, z0 = [7, 16, 1, 11, 1], 3
    proof = _w(oracle.open_(coeffs, z0, g1))
    C_ = np.repeat(pttab, 17)
    V = np.tile(np.arange(17, dtype=np.uint8), len(pttab))
    n = len(C_)
    Q = np.full(n, proof, np.uint32)
    Z = np.full(n, z0, np.uint8)
    ok, bad = _emu_check(emu, tables, C_, Q, Z, V, g1[0], g2[1])
    want, panic = po.kzg_check_many(_bytes(C_), _bytes(Q), Z, V, g1, g2)
    assert np.array_equal(bad, panic)
    assert np.array_equal(ok[~panic], want[~panic])
    assert ok[~panic].sum() >= 289 and (~ok[~panic]).sum() > 0
    rng = np.random.default_rng(5)
    m = 1 << 15
    C_, Q = pttab[rng.integers(0, len(pttab), m)], pttab[rng.integers(0, len(pttab), m)]
    e17 = _e17_points(pttab)
    Q[: m // 2] = e17[rng.integers(0, E17, m // 2)]                 # half the proofs in E[17]
    Z, V = rng.integers(0, 17, m).astype(np.uint8), rng.integers(0, 17, m).astype(np.uint8)
    ok, bad = _emu_check(emu, tables, C_, Q, Z, V, g1[0], g2[1])
    want, panic = po.kzg_check_many(_bytes(C_), _bytes(Q), Z, V, g1, g2)
    assert np.array_equal(bad, panic)
    assert np.array_equal(ok[~panic], want[~panic])
    assert (~panic).sum() > 100
