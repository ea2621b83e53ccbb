"""CPU tier: the pairing oracle (tests/pairing_oracle.c) against the reference's own pairing and kzg::check cases
(tests/golden/pairing_kats.json), with commitments and proofs from the CPU oracle's commit / open."""
import json
import os

import pytest

import oracle
import pairing_oracle as po

HERE = os.path.dirname(os.path.abspath(__file__))
INF = b"\xff" * 4


@pytest.fixture(scope="module")
def kats():
    with open(os.path.join(HERE, "golden", "pairing_kats.json")) as f:
        return json.load(f)


def test_tate_kats(kats):
    for t in kats["tate"]:
        assert po.pairing(bytes(t["p"]), bytes(t["q"])) == tuple(t["expected"])


def _row(case):
    g1, g2 = oracle.setup()
    c = case["coeffs"]
    z = case["point"]
    commitment = oracle.commit(c, g1[:len(c)])
    proof = oracle.open_(c, z, g1) if case["proof"] == "open" else INF
    value = {"eval": oracle.poly_eval(17, c, z), "point": z}.get(case["value"], case["value"])
    return commitment, proof, z, value, g1, g2


def test_check_cases(kats):
    assert len(kats["check"]) == 9
    for case in kats["check"]:
        row = _row(case)
        if case["expected"] == "panic":
            with pytest.raises(po.OraclePanic):
                po.kzg_check(*row)
        else:
            assert po.kzg_check(*row) is case["expected"], case


def test_pairing_params(kats):
    pp = kats["pairing_params"]
    commitment, proof, *_ = _row({"coeffs": pp["coeffs"], "point": pp["point"], "proof": "open", "value": "eval"})
    assert commitment == INF and proof == bytes(pp["q"])
    # the commitment is Infinity, yet p − g1·value is not, and the check passes
    assert po.kzg_check(*_row({"coeffs": pp["coeffs"], "point": pp["point"], "proof": "open", "value": "eval"}))


def test_srs_panics():
    """expect("has g1 srs") and g2_srs[1] (kzg/setup.rs:89-92)."""
    c, q, z, v, g1, g2 = _row({"coeffs": [3, 2, 1], "point": 5, "proof": "open", "value": "eval"})
    with pytest.raises(po.OraclePanic):
        po.kzg_check(c, q, z, v, [], g2)
    with pytest.raises(po.OraclePanic):
        po.kzg_check(c, q, z, v, g1, g2[:1])
    assert po.kzg_check(c, q, z, v, g1[:1], g2)


def test_pairing_panics_on_infinity_equal_and_non_torsion():
    g1, g2 = oracle.setup()
    with pytest.raises(po.OraclePanic):
        po.pairing(INF, g2[0])
    with pytest.raises(po.OraclePanic):
        po.pairing(g1[0], INF)
    with pytest.raises(po.OraclePanic):
        po.pairing(g1[0], g1[0])                      # P == Q: the zeros counter ends nonzero
    assert po.point_order(g1[0]) == po.point_order(g2[0]) == 17
    assert po.pairing(g1[0], g2[0]) != po.pairing(g1[0], g2[1])
    # a point of order 34 = 2·17: on the curve, not 17-torsion
    p34 = oracle.point_add(g1[0], next(bytes([x, 0, 0, 0]) for x in range(101) if oracle.on_curve(bytes([x, 0, 0, 0]))))
    assert po.point_order(p34) == 34
    with pytest.raises(po.OraclePanic):
        po.pairing(p34, g2[0])
    with pytest.raises(po.OraclePanic):
        po.pairing(g2[0], p34)
