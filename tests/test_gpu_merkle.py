"""ronk_merkle_build_sha256, ronk_merkle_proofs_sha256, ronk_merkle_verify_sha256 and their _host twins (tree.MerkleTree,
ops.merkle_build / merkle_proofs / merkle_verify): the reference's Merkle tree (src/tree/merkle.rs) against its
hashlib restatement in tests/merkle_oracle.py.

Whole node buffers for n = 1 … 70 and around every span edge up to 2^20 leaves, leaves of mixed length, the launch
count of a build, every proof of small trees with the reference's panics, verification of valid and tampered proofs,
refusals in the header's order with nothing written, poisoned slack, the _host twins, a gated non-blocking stream, and
the Python MerkleTree on the reference's own trees."""
import json
import os

import numpy as np
import pytest

import merkle_oracle as mo
from gpu_util import ctx

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
EINVAL, EUNSUPPORTED = 1, 5
POISON = 0xA5
SIDE = {"Left": 0, "Right": 1}


def _p(x):
    from ronkathon_b200 import _lib
    return _lib._ptr(x)


def _rc(c, name, *args):
    from ronkathon_b200 import _lib
    c.sync()
    before = c.launches
    rc = getattr(_lib.lib(), name)(c._h, *args)
    c.sync()
    return rc, c.launches - before


def _u8(b: bytes):
    import torch
    if not b:
        return torch.empty(0, dtype=torch.uint8, device="cuda")
    return torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda()


def _i64(a):
    from ronkathon_b200 import ops
    return ops.to_device(np.asarray(a, dtype=np.uint64))


def _batch(msgs):
    offs = np.zeros(len(msgs) + 1, np.uint64)
    offs[1:] = np.cumsum([len(m) for m in msgs])
    return _u8(b"".join(msgs)), _i64(offs)


def _total(n):
    from ronkathon_b200.ops import merkle_levels
    return sum(merkle_levels(n)[0])


def _depth(n):
    return (n - 1).bit_length() if n > 1 else 0


def _launches_of_build(n):
    L = _depth(n)
    return 1 + -(-max(L - 9, 0) // 9)


def _build(c, msgs):
    """(node buffer as bytes, launches) through ronk_merkle_build_sha256."""
    import torch
    data, offs = _batch(msgs)
    nodes = torch.empty(32 * _total(len(msgs)), dtype=torch.uint8, device="cuda")
    code, launches = _rc(c, "ronk_merkle_build_sha256", _p(data) if data.numel() else None, data.numel(), _p(offs),
                         len(msgs), _p(nodes))
    assert code == 0, c.check(code)
    return nodes, launches


def _leaves(rng, n, max_len=40):
    return [rng.integers(0, 256, int(k), dtype=np.uint8).tobytes() for k in rng.integers(0, max_len + 1, n)]


def _proofs(c, nodes, n, idx):
    import torch
    L, m = _depth(n), len(idx)
    sib = torch.empty((max(m * L, 1), 32), dtype=torch.uint8, device="cuda")
    sides = torch.empty(max(m * L, 1), dtype=torch.uint8, device="cuda")
    ind = _i64(idx)
    code, launches = _rc(c, "ronk_merkle_proofs_sha256", _p(nodes), n, _p(ind), m, _p(sib), _p(sides))
    return code, launches, sib.cpu().numpy()[:m * L].reshape(m, L, 32), sides.cpu().numpy()[:m * L].reshape(m, L)


def _oracle_proof(tree, i):
    return [(s, SIDE[d]) for s, d in tree.get_proof(i)]


def _as_proof(sib, sides):
    return [(sib[l].tobytes(), int(sides[l])) for l in range(len(sides))]


def _verify(c, root, msgs, sib, sides):
    """ok bytes through ronk_merkle_verify_sha256; sib [m, depth, 32], sides [m, depth] (numpy)."""
    import torch
    m, depth = sides.shape
    data, offs = _batch(msgs)
    s = _u8(np.ascontiguousarray(sib).tobytes())
    d = _u8(np.ascontiguousarray(sides).tobytes())
    ok = torch.full((m,), POISON, dtype=torch.uint8, device="cuda")
    code, launches = _rc(c, "ronk_merkle_verify_sha256", _p(_u8(root)), _p(data) if data.numel() else None, data.numel(),
                         _p(offs), m, _p(s) if s.numel() else None, _p(d) if d.numel() else None, depth, _p(ok))
    return code, launches, ok.cpu().numpy()


# ---- builds ----------------------------------------------------------------------------------------------------------

def test_every_small_tree_whole_buffer():
    c = ctx()
    rng = np.random.default_rng(1)
    for n in range(1, 71):
        msgs = _leaves(rng, n)
        nodes, launches = _build(c, msgs)
        assert launches == 1 and nodes.cpu().numpy().tobytes() == mo.Tree(msgs).nodes(), n


@pytest.mark.parametrize("n", [511, 512, 513, 1023, 1025, 1535, 1537, 2 ** 18 - 1, 2 ** 18 + 1, 2 ** 18 + 3, 2 ** 20])
def test_span_edges_and_large_trees(n):
    c = ctx()
    rng = np.random.default_rng(n)
    if n <= 2048:
        msgs = _leaves(rng, n, 100)
    else:
        blob = rng.integers(0, 256, 32 * n, dtype=np.uint8).tobytes()
        msgs = [blob[32 * i:32 * i + 32] for i in range(n)]
    nodes, launches = _build(c, msgs)
    assert launches == _launches_of_build(n)
    assert nodes.cpu().numpy().tobytes() == mo.Tree(msgs).nodes(), n


def test_launch_count_per_build():
    c = ctx()
    for n, want in ((1, 1), (2, 1), (512, 1), (513, 2), (2 ** 18, 2), (2 ** 18 + 1, 3), (2 ** 20, 3)):
        assert _launches_of_build(n) == want
        msgs = [i.to_bytes(4, "little") for i in range(n)]
        _, launches = _build(c, msgs)
        assert launches == want, n


def test_ops_merkle_build_levels():
    from ronkathon_b200 import ops
    c = ctx()
    msgs = [b"leaf %d" % i for i in range(1000)]
    data, offs = _batch(msgs)
    nodes, level_offsets = ops.merkle_build(c, data, offs)
    tree = mo.Tree(msgs)
    h = nodes.cpu().numpy()
    assert nodes.shape == (_total(1000), 32) and len(level_offsets) == len(tree.hashes)
    for l, level in enumerate(reversed(tree.hashes)):
        assert [h[level_offsets[l] + i].tobytes() for i in range(len(level))] == level, l
    assert h[-1].tobytes() == tree.root_hash()
    empty, lv = ops.merkle_build(c, _u8(b""), _i64([0]))
    assert empty.shape == (0, 32) and lv == []


# ---- proofs ----------------------------------------------------------------------------------------------------------

def test_every_proof_of_small_trees_and_the_panics():
    c = ctx()
    rng = np.random.default_rng(2)
    for n in range(2, 34):
        msgs = _leaves(rng, n, 10)
        tree = mo.Tree(msgs)
        nodes, _ = _build(c, msgs)
        good, bad = [], []
        for i in range(2 * n + 2):
            try:
                tree.get_proof(i)
                good.append(i)
            except mo.Panic:
                bad.append(i)
        code, launches, sib, sides = _proofs(c, nodes, n, good)
        assert (code, launches) == (0, 1), n
        for j, i in enumerate(good):
            assert _as_proof(sib[j], sides[j]) == _oracle_proof(tree, i), (n, i)
        for i in bad:
            assert _proofs(c, nodes, n, [0, i, 1])[:2] == (EINVAL, 1), (n, i)


def test_reference_panic_edges():
    c = ctx()
    for n, i, want in ((3, 3, 0), (5, 4, EINVAL), (5, 5, EINVAL), (6, 5, EINVAL), (6, 3, 0), (5, 3, 0)):
        msgs = [b"%d" % k for k in range(n)]
        nodes, _ = _build(c, msgs)
        code, _, sib, sides = _proofs(c, nodes, n, [i])
        assert code == want, (n, i)
        if want == 0:
            assert _as_proof(sib[0], sides[0]) == _oracle_proof(mo.Tree(msgs), i)


def test_trees_of_one_leaf_give_empty_proofs():
    c = ctx()
    nodes, _ = _build(c, [b"only"])
    code, launches, sib, sides = _proofs(c, nodes, 1, [0, 1, 99])
    assert (code, launches) == (0, 0) and sib.shape == (3, 0, 32) and sides.shape == (3, 0)
    assert _rc(c, "ronk_merkle_proofs_sha256", None, 0, _p(_i64([5])), 1, None, None) == (0, 0)


# ---- verification ----------------------------------------------------------------------------------------------------

def test_verify_valid_and_tampered_proofs():
    c = ctx()
    rng = np.random.default_rng(3)
    for n in (2, 3, 5, 8, 13, 100, 600):
        msgs = [b"%d:" % i + x for i, x in enumerate(_leaves(rng, n, 50))]   # distinct, so no sibling equals its twin
        tree = mo.Tree(msgs)
        nodes, _ = _build(c, msgs)
        idx = [i for i in range(n) if _safe(tree, i)]
        _, _, sib, sides = _proofs(c, nodes, n, idx)
        root = tree.root_hash()
        items = [msgs[i] for i in idx]
        code, launches, ok = _verify(c, root, items, sib, sides)
        assert (code, launches) == (0, 1) and ok.tolist() == [1] * len(idx), n
        m = len(idx)
        flipped = sib.copy()
        flipped[np.arange(m), np.arange(m) % sib.shape[1], np.arange(m) % 32] ^= 1
        swapped = sides.copy()
        swapped[:, -1] ^= 1
        wrong_leaf = [x + b"!" for x in items]
        wrong_root = bytes([root[0] ^ 0x80]) + root[1:]
        assert _verify(c, root, items, flipped, sides)[2].tolist() == [0] * m
        assert _verify(c, root, items, sib, swapped)[2].tolist() == [0] * m
        assert _verify(c, root, wrong_leaf, sib, sides)[2].tolist() == [0] * m
        assert _verify(c, wrong_root, items, sib, sides)[2].tolist() == [0] * m


def _safe(tree, i):
    try:
        tree.get_proof(i)
        return True
    except mo.Panic:
        return False


def test_verify_depth_zero_and_flags():
    c = ctx()
    root = mo.digest(b"a")
    none = np.zeros((3, 0, 32), np.uint8), np.zeros((3, 0), np.uint8)
    code, launches, ok = _verify(c, root, [b"a", b"b", b"a"], *none)
    assert (code, launches) == (0, 1) and ok.tolist() == [1, 0, 1]
    # a side byte other than 0 or 1 is flagged by the device
    tree = mo.Tree([b"x", b"y"])
    sib = np.frombuffer(tree.hashes[1][1], np.uint8).reshape(1, 1, 32)
    assert _verify(c, tree.root_hash(), [b"x"], sib, np.array([[1]], np.uint8))[:2] == (0, 1)
    assert _verify(c, tree.root_hash(), [b"x"], sib, np.array([[2]], np.uint8))[:2] == (EINVAL, 1)


def test_ops_proofs_and_verify():
    import torch
    from ronkathon_b200 import ops
    c = ctx()
    msgs = [b"item %d" % i for i in range(700)]
    data, offs = _batch(msgs)
    nodes, _ = ops.merkle_build(c, data, offs)
    idx = list(range(0, 512, 7))   # from leaf 512 on every path meets an unpaired node, where get_proof panics
    sib, sides = ops.merkle_proofs(c, nodes, 700, _i64(idx))
    assert sib.shape == (len(idx), 10, 32) and sides.shape == (len(idx), 10)
    tree = mo.Tree(msgs)
    s, d = sib.cpu().numpy(), sides.cpu().numpy()
    assert all(_as_proof(s[j], d[j]) == _oracle_proof(tree, i) for j, i in enumerate(idx))
    items, ioffs = _batch([msgs[i] for i in idx])
    ok = ops.merkle_verify(c, nodes[-1].contiguous(), items, ioffs, sib, sides)
    assert ok.dtype == torch.bool and ok.all().item()


# ---- slack, refusals, host twins, streams ----------------------------------------------------------------------------

def test_slack_around_every_output_stays_poisoned():
    import torch
    c = ctx()
    msgs = [b"s%d" % i for i in range(37)]
    tree = mo.Tree(msgs)
    data, offs = _batch(msgs)
    T, slack = _total(37), 23
    buf = torch.full((32 * T + 2 * slack,), POISON, dtype=torch.uint8, device="cuda")
    nodes = buf[slack:slack + 32 * T]   # not 16-byte aligned: the byte-wise store path
    assert _rc(c, "ronk_merkle_build_sha256", _p(data), data.numel(), _p(offs), 37, _p(nodes))[0] == 0
    h = buf.cpu().numpy()
    assert (h[:slack] == POISON).all() and (h[-slack:] == POISON).all() and h[slack:-slack].tobytes() == tree.nodes()
    L, m = 6, 3
    sb = torch.full((32 * m * L + 2 * slack,), POISON, dtype=torch.uint8, device="cuda")
    sd = torch.full((m * L + 2 * slack,), POISON, dtype=torch.uint8, device="cuda")
    idx = [0, 17, 31]
    assert _rc(c, "ronk_merkle_proofs_sha256", _p(nodes), 37, _p(_i64(idx)), m, _p(sb[slack:slack + 32 * m * L]),
               _p(sd[slack:slack + m * L])) == (0, 1)
    hs, hd = sb.cpu().numpy(), sd.cpu().numpy()
    for x in (hs, hd):
        assert (x[:slack] == POISON).all() and (x[-slack:] == POISON).all()
    s, d = hs[slack:-slack].reshape(m, L, 32), hd[slack:-slack].reshape(m, L)
    assert all(_as_proof(s[j], d[j]) == _oracle_proof(tree, i) for j, i in enumerate(idx))
    ok = torch.full((m + 2 * slack,), POISON, dtype=torch.uint8, device="cuda")
    items, ioffs = _batch([msgs[i] for i in idx])
    assert _rc(c, "ronk_merkle_verify_sha256", _p(_u8(tree.root_hash())), _p(items), items.numel(), _p(ioffs), m,
               _p(_u8(s.tobytes())), _p(_u8(d.tobytes())), L, _p(ok[slack:slack + m])) == (0, 1)
    ho = ok.cpu().numpy()
    assert (ho[:slack] == POISON).all() and (ho[-slack:] == POISON).all() and ho[slack:-slack].tolist() == [1] * m


def test_refusals_in_order_write_nothing():
    import torch
    c = ctx()
    msgs = [b"a", b"bb", b"ccc", b"dddd", b"e"]
    data, offs = _batch(msgs)
    nodes = torch.full((32 * _total(5),), POISON, dtype=torch.uint8, device="cuda")
    mis = torch.zeros(8, dtype=torch.int64, device="cuda").view(torch.uint8)[4:52]
    P = lambda x: _p(x) if x is not None else None  # noqa: E731

    def build(d=data, dl=11, o=offs, n=5, out=nodes):
        return _rc(c, "ronk_merkle_build_sha256", P(d), dl, P(o), n, P(out))

    cases = [
        ("null data", build(d=None), EINVAL),
        ("null offsets", build(o=None), EINVAL),
        ("null nodes before n ≥ 2^32", build(out=None, n=1 << 32), EINVAL),
        ("misaligned offsets", build(o=mis), EINVAL),
        ("n ≥ 2^32", build(n=1 << 32), EUNSUPPORTED),
        ("data_len above 2^40", build(dl=(1 << 40) + 1), EUNSUPPORTED),
        ("nodes overlap data", build(out=data), EINVAL),
        ("nodes overlap offsets", build(out=offs), EINVAL),
    ]
    for name, got, want in cases:
        assert got == (want, 0), name
    assert (nodes.cpu().numpy() == POISON).all()
    assert build(d=None, dl=0, o=None, n=0, out=None) == (0, 0)
    assert build(o=_i64([0, 1, 3, 2, 10, 11])) == (EINVAL, 1)         # decreasing offsets, flagged on the device
    assert build(o=_i64([0, 1, 3, 6, 10, 12])) == (EINVAL, 1)         # past data_len

    assert build() == (0, 1)
    idx = _i64([0, 1, 2])
    sib = torch.full((3 * 3 * 32,), POISON, dtype=torch.uint8, device="cuda")
    sides = torch.full((9,), POISON, dtype=torch.uint8, device="cuda")

    def proofs(nd=nodes, n=5, ix=idx, m=3, s=sib, d=sides):
        return _rc(c, "ronk_merkle_proofs_sha256", P(nd), n, P(ix), m, P(s), P(d))

    cases = [
        ("null nodes", proofs(nd=None), EINVAL),
        ("null indices", proofs(ix=None), EINVAL),
        ("null siblings", proofs(s=None), EINVAL),
        ("null sides", proofs(d=None), EINVAL),
        ("misaligned indices", proofs(ix=mis), EINVAL),
        ("m ≥ 2^32", proofs(m=1 << 32), EUNSUPPORTED),
        ("n ≥ 2^32", proofs(n=1 << 32), EUNSUPPORTED),
        ("siblings overlap nodes", proofs(s=nodes), EINVAL),
        ("sides overlap indices", proofs(d=idx), EINVAL),
        ("sides overlap siblings", proofs(d=sib), EINVAL),
    ]
    for name, got, want in cases:
        assert got == (want, 0), name
    assert (sib.cpu().numpy() == POISON).all() and (sides.cpu().numpy() == POISON).all()

    root = nodes[-32:].clone()
    ok = torch.full((5,), POISON, dtype=torch.uint8, device="cuda")
    vs = torch.zeros(5 * 3 * 32, dtype=torch.uint8, device="cuda")
    vd = torch.zeros(5 * 3, dtype=torch.uint8, device="cuda")

    def verify(r=root, d=data, dl=11, o=offs, m=5, s=vs, sd=vd, depth=3, out=ok):
        return _rc(c, "ronk_merkle_verify_sha256", P(r), P(d), dl, P(o), m, P(s), P(sd), depth, P(out))

    cases = [
        ("null data", verify(d=None), EINVAL),
        ("null offsets", verify(o=None), EINVAL),
        ("null ok", verify(out=None), EINVAL),
        ("null root", verify(r=None), EINVAL),
        ("null siblings", verify(s=None), EINVAL),
        ("null sides before depth > 32", verify(sd=None, depth=33), EINVAL),
        ("m ≥ 2^32", verify(m=1 << 32), EUNSUPPORTED),
        ("depth > 32", verify(depth=33), EUNSUPPORTED),
        ("ok overlaps root", verify(out=root), EINVAL),
        ("ok overlaps sides", verify(out=vd), EINVAL),
        ("ok overlaps data", verify(out=data), EINVAL),
    ]
    for name, got, want in cases:
        assert got == (want, 0), name
    assert (ok.cpu().numpy() == POISON).all()
    assert verify(s=None, sd=None, depth=0) == (0, 1)     # depth 0 reads neither


def test_host_twins():
    c = ctx()
    rng = np.random.default_rng(5)
    msgs = _leaves(rng, 45, 30)
    tree = mo.Tree(msgs)
    blob = np.frombuffer(b"".join(msgs) or b"\0", np.uint8).copy()
    offs = np.concatenate([[0], np.cumsum([len(m) for m in msgs])]).astype(np.uint64)
    nodes = np.zeros(32 * _total(45), np.uint8)
    assert _rc(c, "ronk_merkle_build_sha256_host", _p(blob), int(offs[-1]), _p(offs), 45, _p(nodes)) == (0, 1)
    assert nodes.tobytes() == tree.nodes()
    idx = np.array([i for i in range(45) if _safe(tree, i)], np.uint64)
    m, L = idx.size, 6
    sib, sides = np.zeros((m, L, 32), np.uint8), np.zeros((m, L), np.uint8)
    assert _rc(c, "ronk_merkle_proofs_sha256_host", _p(nodes), 45, _p(idx), m, _p(sib), _p(sides)) == (0, 1)
    assert all(_as_proof(sib[j], sides[j]) == _oracle_proof(tree, int(i)) for j, i in enumerate(idx))
    items = [msgs[int(i)] for i in idx]
    iblob = np.frombuffer(b"".join(items) or b"\0", np.uint8).copy()
    ioffs = np.concatenate([[0], np.cumsum([len(x) for x in items])]).astype(np.uint64)
    root = np.frombuffer(tree.root_hash(), np.uint8).copy()
    ok = np.zeros(m, np.uint8)
    assert _rc(c, "ronk_merkle_verify_sha256_host", _p(root), _p(iblob), int(ioffs[-1]), _p(ioffs), m, _p(sib), _p(sides), L,
               _p(ok)) == (0, 1)
    assert ok.tolist() == [1] * m
    # bad offsets and side bytes are refused on the host before anything is staged or launched, with nothing written
    bad = offs.copy()
    bad[3], bad[4] = bad[4] + 1, bad[3]
    nodes[:] = POISON
    assert _rc(c, "ronk_merkle_build_sha256_host", _p(blob), int(offs[-1]), _p(bad), 45, _p(nodes)) == (EINVAL, 0)
    assert (nodes == POISON).all()
    bad_sides = sides.copy()
    bad_sides[-1, -1] = 7
    ok[:] = POISON
    assert _rc(c, "ronk_merkle_verify_sha256_host", _p(root), _p(iblob), int(ioffs[-1]), _p(ioffs), m, _p(sib),
               _p(bad_sides), L, _p(ok)) == (EINVAL, 0)
    assert (ok == POISON).all()
    # a panicking index: the device flags it, and the host outputs stay unwritten
    sib[:] = POISON
    five = np.array([4], np.uint64)
    t5 = np.zeros(32 * _total(5), np.uint8)
    f = np.frombuffer(b"abcde", np.uint8).copy()
    assert _rc(c, "ronk_merkle_build_sha256_host", _p(f), 5, _p(np.arange(6, dtype=np.uint64)), 5, _p(t5)) == (0, 1)
    assert _rc(c, "ronk_merkle_proofs_sha256_host", _p(t5), 5, _p(five), 1, _p(sib), _p(sides))[0] == EINVAL
    assert (sib == POISON).all()


def test_gated_non_blocking_stream():
    import torch
    from ronkathon_b200 import Context, ops
    msgs = [b"g%d" % i for i in range(5000)]
    data, offs = _batch(msgs)
    s = torch.cuda.Stream()
    c = Context(0, s.cuda_stream)
    try:
        g = torch.zeros_like(data)
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            torch.cuda._sleep(100_000_000)
            g.copy_(data)
            nodes, _ = ops.merkle_build(c, g, offs)
        s.synchronize()
        assert nodes.cpu().numpy().tobytes() == mo.Tree(msgs).nodes()
    finally:
        c.close()


# ---- the Python MerkleTree -------------------------------------------------------------------------------------------

def test_python_tree_on_the_reference_trees():
    from ronkathon_b200 import RonkPanic
    from ronkathon_b200.tree import LeftOrRight, MerkleTree
    ctx()
    with open(os.path.join(HERE, "golden", "sha_merkle_kats.json")) as f:
        tests = json.load(f)["merkle_tests"]
    for name, t in tests.items():
        for leaves in t["trees"]:
            tree, want = MerkleTree(leaves), mo.Tree(leaves)
            assert tree.hashes == want.hashes and tree.root_hash() == want.root_hash(), name
            assert tree.leaves == leaves
    t = tests["odd_leaf_tree"]
    assert [len(level) for level in MerkleTree(t["trees"][0]).hashes] == t["level_sizes_root_first"]
    roots = {MerkleTree(leaves).root_hash() for leaves in tests["test_different_value"]["trees"]}
    assert len(roots) == 3
    t = tests["valid_proof"]
    tree = MerkleTree(t["trees"][0])
    proof = tree.get_proof(t["index"])
    assert [(s, LeftOrRight[d]) for s, d in mo.Tree(t["trees"][0]).get_proof(t["index"])] == list(proof)
    assert tree.prove(t["value"], proof)
    assert not tree.prove(tests["invalid_proof_wrong_element"]["value"], proof)
    z = tests["invalid_proof_wrong_sibling"]["zeroed_sibling"]
    proof[z] = (bytes(32), proof[z][1])
    assert not tree.prove("b", proof)
    five = MerkleTree(["a", "b", "c", "d", "e"])
    with pytest.raises(RonkPanic):
        five.get_proof(4)
    assert five.prove("c", five.get_proof(2)) and MerkleTree([b"a", "b", "c"]).get_proof(3)
    empty = MerkleTree([])
    assert empty.hashes == [[]] and empty.get_proof(0) == []
    with pytest.raises(RonkPanic):
        empty.root_hash()
    with pytest.raises(RonkPanic):
        empty.prove("a", [])
    one = MerkleTree(["a"])
    assert one.get_proof(5) == [] and one.prove("a", []) and not one.prove("b", [])
