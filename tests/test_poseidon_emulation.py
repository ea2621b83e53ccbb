"""CPU tier: the row routine of ronk_poseidon_permute_u64 / ronk_poseidon_sponge_u64 (ronkathon_b200/csrc/poseidon.cuh,
compiled for the host by tests/emu/poseidon_emu.cpp, a test fixture, never part of the product) against the C
restatement of the reference in tests/poseidon_oracle.c: every width 2 … 16 on the Montgomery policy at primes from 17
to 2^64 − 59 (the subtractive REDC above 2^63) and on the Goldilocks policy, S-box exponents 0, 1, 2, 3, 5, 7 and
p − 2, odd, even and zero full-round counts, no partial rounds and no rounds at all."""
import ctypes as C
import json
import os
import subprocess
import tempfile

import numpy as np
import pytest

import poseidon_oracle as po

HERE = os.path.dirname(os.path.abspath(__file__))
GL = 0xFFFFFFFF00000001
PRIMES = [17, 101, 127, GL, (1 << 61) - 1, (1 << 64) - 59]
P64 = C.POINTER(C.c_uint64)


@pytest.fixture(scope="module")
def emu():
    so = os.path.join(tempfile.mkdtemp(prefix="ronk_poseidon_emu_"), "libposeidon_emu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", so,
                           os.path.join(HERE, "emu", "poseidon_emu.cpp")])
    lib = C.CDLL(so)
    lib.emu_poseidon_rows.argtypes = [C.c_int, C.c_uint64, C.c_uint32, C.c_uint64, C.c_uint32, C.c_uint32, P64, P64,
                                      C.c_uint32, P64, C.c_uint64, P64, C.c_uint64, C.c_uint64]
    lib.emu_poseidon_rows.restype = C.c_int
    return lib


def _p(a):
    return a.ctypes.data_as(P64)


def _rand(rng, p, n):
    return rng.integers(0, 2**64, size=n, dtype=np.uint64, endpoint=False) % np.uint64(p)


def _cfg(rng, p, width, alpha, num_f, num_p):
    rc = _rand(rng, p, (num_f + num_p) * width)
    mds = _rand(rng, p, width * width).reshape(width, width)
    return po.Config(p, width, alpha, num_p, num_f, rc.tolist(), mds.tolist())


def _emu_permute(emu, gold, cfg, states):
    s = np.ascontiguousarray(states, dtype=np.uint64).copy()
    w = cfg.width
    assert emu.emu_poseidon_rows(int(gold), cfg.p, w, cfg.alpha, cfg.num_f, cfg.num_p, _p(cfg.rc), _p(cfg.mds), w, _p(s), w,
                                 _p(s), w, s.shape[0]) == 0
    return s


def _emu_sponge(emu, gold, cfg, rate, rows, n_out):
    rows = np.ascontiguousarray(rows, dtype=np.uint64)
    out = np.zeros((rows.shape[0], max(n_out, 1)), dtype=np.uint64)
    assert emu.emu_poseidon_rows(int(gold), cfg.p, cfg.width, cfg.alpha, cfg.num_f, cfg.num_p, _p(cfg.rc), _p(cfg.mds), rate,
                                 _p(rows), rows.shape[1], _p(out), n_out, rows.shape[0]) == 0
    return out[:, :n_out]


def _policies(p):
    return (False, True) if p == GL else (False,)


@pytest.mark.parametrize("p", PRIMES)
def test_every_width_permutation(emu, p):
    rng = np.random.default_rng(p % 9973)
    for width in range(2, 17):
        cfg = _cfg(rng, p, width, 5 if p != 17 else 3, 8, 11)
        states = _rand(rng, p, 4 * width).reshape(4, width)
        want = po.permute(cfg, states)
        for gold in _policies(p):
            assert np.array_equal(_emu_permute(emu, gold, cfg, states), want), (p, width, gold)


@pytest.mark.parametrize("p", PRIMES)
def test_every_width_sponge(emu, p):
    rng = np.random.default_rng(p % 7919)
    for width in range(2, 17):
        cfg = _cfg(rng, p, width, 7, 4, 3)
        for rate in sorted({1, width // 2 or 1, width}):
            for length, n_out in ((0, 3), (rate, rate), (2 * rate + 1, 2 * rate), (3, 1)):
                rows = _rand(rng, p, 3 * length).reshape(3, length)
                want = po.sponge_rows(cfg, rate, rows, n_out)
                for gold in _policies(p):
                    got = _emu_sponge(emu, gold, cfg, rate, rows, n_out)
                    assert np.array_equal(got, want), (p, width, rate, length, n_out, gold)


@pytest.mark.parametrize("p", PRIMES)
def test_alpha_and_round_classes(emu, p):
    rng = np.random.default_rng(p % 6007)
    for alpha in (0, 1, 2, 3, 5, 7, p - 2):
        for num_f, num_p in ((8, 11), (7, 3), (3, 0), (0, 5), (0, 0), (1, 1)):
            for width in (2, 3, 16):
                cfg = _cfg(rng, p, width, alpha, num_f, num_p)
                states = _rand(rng, p, 3 * width).reshape(3, width)
                states[0] = 0                                  # 0^0 = 1 where alpha = 0
                want = po.permute(cfg, states)
                for gold in _policies(p):
                    assert np.array_equal(_emu_permute(emu, gold, cfg, states), want), (p, alpha, num_f, num_p, width, gold)


def test_zero_rounds_is_identity(emu):
    rng = np.random.default_rng(3)
    cfg = _cfg(rng, 101, 5, 3, 0, 0)
    states = _rand(rng, 101, 10).reshape(2, 5)
    assert np.array_equal(_emu_permute(emu, False, cfg, states), states)


def test_reference_kat(emu):
    with open(os.path.join(HERE, "golden", "poseidon_kats.json")) as f:
        k = json.load(f)
    cfg = po.Config(101, k["width"], k["alpha"], k["num_p"], k["num_f"], k["rc16"], k["mds16"])
    assert int(_emu_permute(emu, False, cfg, np.zeros((1, 16), np.uint64))[0, 1]) == k["hash_zero"]["expected"]
