"""CPU tier: the hashlib restatement of src/tree/merkle.rs (tests/merkle_oracle.py) reproduces the reference's own
tests and known answers (tests/golden/sha_merkle_kats.json), and its get_proof panics exactly where the reference's
does.  Also: nothing under ronkathon_b200/ hashes on the host (no hashlib import, no CPU fallback)."""
import hashlib
import json
import os

import pytest

import merkle_oracle as mo

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def kats():
    with open(os.path.join(HERE, "golden", "sha_merkle_kats.json")) as f:
        return json.load(f)


def test_sha256_known_answers(kats):
    assert len(kats["sha256"]) == 4
    for case in kats["sha256"]:
        assert mo.digest(case["input"].encode()).hex() == case["digest"], case["src"]


def test_level_counts(kats):
    for name in ("even_leaf_tree", "odd_leaf_tree"):
        t = kats["merkle_tests"][name]
        tree = mo.Tree(t["trees"][0])
        assert len(tree.hashes) == t["levels"], t["src"]
        assert [len(level) for level in tree.hashes] == t["level_sizes_root_first"], t["src"]


def test_different_values_give_different_roots(kats):
    t = kats["merkle_tests"]["test_different_value"]
    roots = [mo.Tree(leaves).root_hash() for leaves in t["trees"]]
    assert len(roots) == 3 and len(set(roots)) == 3, t["src"]


def test_valid_and_invalid_proofs(kats):
    t = kats["merkle_tests"]["valid_proof"]
    tree = mo.Tree(t["trees"][0])
    assert not t["should_panic"] and tree.prove(t["value"], tree.get_proof(t["index"])), t["src"]
    t = kats["merkle_tests"]["invalid_proof_wrong_element"]
    tree = mo.Tree(t["trees"][0])
    assert t["should_panic"] and not tree.prove(t["value"], tree.get_proof(t["index"])), t["src"]
    t = kats["merkle_tests"]["invalid_proof_wrong_sibling"]
    tree = mo.Tree(t["trees"][0])
    proof = tree.get_proof(t["index"])
    proof[t["zeroed_sibling"]] = (bytes(32), proof[t["zeroed_sibling"]][1])
    assert t["should_panic"] and not tree.prove(t["value"], proof), t["src"]


def _panics(n):
    """The indices below 2n + 2 at which the oracle's get_proof panics."""
    tree = mo.Tree([str(i) for i in range(n)])
    bad = set()
    for i in range(2 * n + 2):
        try:
            tree.get_proof(i)
        except mo.Panic:
            bad.add(i)
    return bad


def test_get_proof_panic_rule():
    assert 3 not in _panics(3)
    assert {4, 5} <= _panics(5) and not ({0, 1, 2, 3} & _panics(5))
    assert {4, 5} <= _panics(6) and not ({0, 1, 2, 3} & _panics(6))
    for n in (0, 1):
        tree = mo.Tree([str(i) for i in range(n)])
        assert all(tree.get_proof(i) == [] for i in (0, 1, 7))
    # the rule stated by index: some level l with ((i >> l) ^ 1) past that level's ⌈n / 2^l⌉ nodes
    for n in range(2, 40):
        depth = (n - 1).bit_length()
        rule = {i for i in range(2 * n + 2)
                if any(((i >> l) ^ 1) >= -(-n >> l) for l in range(depth))}
        assert _panics(n) == rule, n


def test_empty_tree_edges():
    tree = mo.Tree([])
    assert tree.hashes == [[]]
    with pytest.raises(mo.Panic):
        tree.root_hash()
    with pytest.raises(mo.Panic):
        tree.prove("a", [])
    one = mo.Tree(["a"])
    assert one.root_hash() == hashlib.sha256(b"a").digest() and one.prove("a", []) and not one.prove("b", [])


def test_package_has_no_host_hashing():
    pkg = os.path.join(ROOT, "ronkathon_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                text = open(os.path.join(dirpath, f)).read()
                assert "hashlib" not in text, f
