"""CPU tier: the Poseidon oracle (tests/poseidon_oracle.c) against the reference's own known answer and sponge case
shapes (tests/golden/poseidon_kats.json), and the property the batched device sponge rests on: any split of the
absorbed words into absorb calls, and of the squeezed count into squeeze calls, gives the words of one absorb and one
squeeze.  Also PoseidonConfig's three asserts, in the oracle and in ronkathon_b200.hashes (which needs no GPU for them)."""
import json
import os

import numpy as np
import pytest

import poseidon_oracle as po

HERE = os.path.dirname(os.path.abspath(__file__))
GL = 0xFFFFFFFF00000001


@pytest.fixture(scope="module")
def kats():
    with open(os.path.join(HERE, "golden", "poseidon_kats.json")) as f:
        return json.load(f)


def _cfg(k, p=None):
    return po.Config(p or k["field"], k["width"], k["alpha"], k["num_p"], k["num_f"], k["rc16"], k["mds16"])


def test_hash_of_zero_state(kats):
    assert len(kats["rc16"]) == (kats["num_f"] + kats["num_p"]) * kats["width"] == 304
    hz = kats["hash_zero"]
    assert po.hash_(_cfg(kats), hz["state"]) == hz["expected"] == 20
    assert po.hash_(_cfg(kats), []) == 20     # zero-padding gives the same state
    with pytest.raises(po.OraclePanic):
        po.hash_(_cfg(kats), [0] * 17)


def _random_split(rng, n):
    """n as a list of call sizes, empty calls included."""
    cuts = sorted(rng.integers(0, n + 1, size=int(rng.integers(0, 6))).tolist())
    parts = np.diff([0] + cuts + [n]).tolist()
    return parts + [0] * int(rng.integers(0, 2))


@pytest.mark.parametrize("p", [101, GL])
def test_split_absorbs_and_squeezes_equal_one_call(kats, p):
    rng = np.random.default_rng(p % 1000)
    cfg = _cfg(kats, p)
    for case in kats["sponge_cases"]:
        n_in = case["absorb_size"] * case.get("absorb_time", 1)
        n_out = case["squeeze_size"] * case.get("squeeze_time", 1)
        words = [int(v) % p for v in rng.integers(0, 2**63, size=n_in)]
        one = po.sponge(cfg, kats["rate"], [words], [n_out])
        # the reference's own shapes: absorb_time calls of absorb_size words, squeeze_time calls of squeeze_size
        chunks = [words[i * case["absorb_size"]:(i + 1) * case["absorb_size"]] for i in range(case.get("absorb_time", 1))]
        assert po.sponge(cfg, kats["rate"], chunks, [case["squeeze_size"]] * case.get("squeeze_time", 1)) == one
        for _ in range(5):
            a, s = _random_split(rng, n_in), _random_split(rng, n_out)
            at = np.cumsum([0] + a)
            assert po.sponge(cfg, kats["rate"], [words[at[i]:at[i + 1]] for i in range(len(a))], s) == one, (case, a, s)


@pytest.mark.parametrize("p", [101, GL])
def test_random_splits_at_every_rate(kats, p):
    rng = np.random.default_rng(7)
    cfg = _cfg(kats, p)
    for rate in (1, 5, 6, 15, 16):
        for n_in in (0, 1, rate - 1, rate, rate + 1, 2 * rate, 3 * rate + 2):
            n_out = int(rng.integers(0, 3 * rate + 2))
            words = [int(v) % p for v in rng.integers(0, 2**63, size=n_in)]
            one = po.sponge(cfg, rate, [words], [n_out])
            a, s = _random_split(rng, n_in), _random_split(rng, n_out)
            at = np.cumsum([0] + a)
            assert po.sponge(cfg, rate, [words[at[i]:at[i + 1]] for i in range(len(a))], s) == one


def test_empty_absorb_squeezes_zeros(kats):
    cfg = _cfg(kats)
    assert po.sponge(cfg, kats["rate"], [[]], [3]) == [0, 0, 0]
    assert po.sponge(cfg, kats["rate"], [], [1, 0, 2]) == [0, 0, 0]


def test_rate_edges(kats):
    cfg = _cfg(kats)
    for bad in (0, 17):
        with pytest.raises(po.OraclePanic):
            po.sponge(cfg, bad, [[1]], [1])


def test_config_asserts(kats):
    k = kats
    with pytest.raises(po.OraclePanic):   # invalid_poseidon_config_width
        po.Config(101, 1, k["alpha"], k["num_p"], k["num_f"], [], [])
    with pytest.raises(po.OraclePanic):   # invalid_poseidon_config_mds
        po.Config(101, k["width"], k["alpha"], k["num_p"], k["num_f"], [], [])
    with pytest.raises(po.OraclePanic):   # invalid_poseidon_config_ark
        po.Config(101, k["width"], k["alpha"], k["num_p"], k["num_f"], [], k["mds16"])


def test_hashes_module_config_asserts(kats):
    from ronkathon_b200 import RonkPanic
    from ronkathon_b200.hashes import PoseidonConfig
    from ronkathon_b200.field import PlutoBaseField
    k = kats
    with pytest.raises(RonkPanic):
        PoseidonConfig(1, k["alpha"], k["num_p"], k["num_f"], [], [], field=PlutoBaseField)
    with pytest.raises(RonkPanic):
        PoseidonConfig(k["width"], k["alpha"], k["num_p"], k["num_f"], [], [], field=PlutoBaseField)
    with pytest.raises(RonkPanic):
        PoseidonConfig(k["width"], k["alpha"], k["num_p"], k["num_f"], [], k["mds16"], field=PlutoBaseField)
    cfg = PoseidonConfig(k["width"], k["alpha"], k["num_p"], k["num_f"], [v + 101 for v in k["rc16"]], k["mds16"],
                         field=PlutoBaseField)
    rc, mds = cfg.tables(101)
    assert rc.tolist() == [v % 101 for v in k["rc16"]] and mds.shape == (16, 16)   # F::from reduces mod p
