"""ronk_pairing_pluto_ext and ronk_kzg_check_pluto_ext_batch (curve.pairing, kzg.check / check_batch, ops.pairing,
ops.kzg_check): the reference's Tate pairing on E[17] and kzg::check, as lookups in a table of the literal Miller loop.

Every pair of E[17] and every commitment of E[17] under every value are checked against the C restatement of the
reference (tests/pairing_oracle.c); each class of input the reference panics on must come back as RONK_EINVAL."""
import functools
import json
import os

import numpy as np
import pytest

import oracle
import pairing_oracle as po
from gpu_util import ctx

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
EINVAL, EUNSUPPORTED = 1, 5
INF = b"\xff" * 4
GEN = bytes([36, 0, 0, 31])
POISON = 0xA5
_e17 = None


def _add(p, q):
    return oracle.point_add(p, q)


def _smul(p, s):
    acc = INF
    for _ in range(s):
        acc = _add(acc, p)
    return acc


def e17():
    """The 289 points of E[17] (Infinity first): i·G1 + j·GEN."""
    global _e17
    if _e17 is None:
        g1 = oracle.setup()[0][0]
        pts = {_add(_smul(g1, i), _smul(GEN, j)) for i in range(17) for j in range(17)}
        _e17 = sorted(pts, key=lambda b: (b != INF, b))
        assert len(_e17) == 289
    return _e17


@functools.lru_cache(maxsize=None)
def _points_of_order(k):
    """An on-curve point of order k (k | 102), as (102/k)·R for a point R of order 102."""
    for x0 in range(101):
        for y0 in range(101):
            for y1 in range(101):
                r = bytes([x0, 1, y0, y1])
                if oracle.on_curve(r) and po.point_order(r) == 102:
                    p = _smul(r, 102 // k)
                    assert po.point_order(p) == k
                    return p
    raise AssertionError("no point of order 102")


def _dev(rows):
    import torch
    a = np.frombuffer(b"".join(bytes(r) for r in rows), dtype=np.uint8).copy()
    return torch.from_numpy(a).cuda()


def _u8(vals):
    import torch
    return torch.from_numpy(np.ascontiguousarray(vals, dtype=np.uint8)).cuda()


def _srs():
    g1, g2 = oracle.setup()
    return g1, g2, _dev(g1), _dev(g2)


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


# ---- pairing entry ---------------------------------------------------------------------------------------------------
def test_pairing_every_pair_of_e17():
    from ronkathon_b200 import ops
    pts = e17()
    P = [p for p in pts for _ in pts]
    Q = [q for _ in pts for q in pts]
    want, panic = po.pairing_many(P, Q)
    assert panic.sum() == 289 + 288 + 288 and len(set(map(tuple, want[~panic].tolist()))) == 17
    keep = np.flatnonzero(~panic)
    got = ops.pairing(ctx(), _dev([P[i] for i in keep]), _dev([Q[i] for i in keep])).cpu().numpy()
    assert np.array_equal(got, want[keep])


def test_pairing_kats_through_curve():
    from ronkathon_b200 import curve
    with open(os.path.join(HERE, "golden", "pairing_kats.json")) as f:
        kats = json.load(f)["tate"]
    ctx()
    for t in kats:
        assert curve.pairing(curve.AffinePoint(bytes(t["p"])), curve.AffinePoint(bytes(t["q"]))) == tuple(t["expected"])


def _bad_pairs():
    pts = e17()
    p, q = pts[1], pts[40]
    bad = [(INF, q), (p, INF), (p, p), (q, q)]
    for k in (2, 3, 6, 34, 51, 102):
        r = _points_of_order(k)
        bad += [(r, q), (p, r)]
    off = bytes([1, 0, 3, 0])                             # (1, 3): 9 ≠ 1 + 3
    assert not oracle.on_curve(off)
    noncanon = bytes([p[0] + 101, p[1], p[2], p[3]])      # the same x0 mod 101, not canonical
    bad += [(off, q), (p, off), (noncanon, q), (p, noncanon), (bytes([0xFF, 0xFF, 0xFF, 0xFE]), q)]
    return bad


def test_pairing_panic_classes_are_einval():
    from ronkathon_b200 import ops
    from ronkathon_b200._lib import RonkPanic
    c = ctx()
    pts = e17()
    for a, b in _bad_pairs():
        with pytest.raises(po.OraclePanic):
            po.pairing(a, b)
        with pytest.raises(RonkPanic):
            ops.pairing(c, _dev([pts[5], a, pts[7]]), _dev([pts[9], b, pts[11]]))


# ---- kzg::check: the reference's cases -------------------------------------------------------------------------------
def test_reference_cases_through_kzg_check():
    from ronkathon_b200 import kzg
    from ronkathon_b200._lib import RonkPanic
    from ronkathon_b200.curve import AffinePoint
    with open(os.path.join(HERE, "golden", "pairing_kats.json")) as f:
        cases = json.load(f)["check"]
    ctx()
    g1, g2 = kzg.setup()
    for case in cases:
        cf, z = case["coeffs"], case["point"]
        p = kzg.commit(cf, g1)
        q = kzg.open_(cf, z, g1) if case["proof"] == "open" else AffinePoint.infinity()
        v = {"eval": oracle.poly_eval(17, cf, z), "point": z}.get(case["value"], case["value"])
        if case["expected"] == "panic":
            with pytest.raises(RonkPanic):
                kzg.check(p, q, z, v, g1, g2)
        else:
            assert kzg.check(p, q, z, v, g1, g2) is case["expected"], case


# ---- batched check ---------------------------------------------------------------------------------------------------
def test_commit_and_open_batches_all_verify():
    from ronkathon_b200 import kzg
    ctx()
    g1, g2 = kzg.setup()
    rng = np.random.default_rng(71)
    C, Q, Z, V = [], [], [], []
    for z in (0, 1, 5, 16):
        polys = [rng.integers(0, 17, int(rng.integers(1, 8))).tolist() for _ in range(40)]
        C += kzg.commit_batch(polys, g1)
        Q += kzg.open_batch(polys, z, g1)
        Z += [z] * len(polys)
        V += [oracle.poly_eval(17, f, z) for f in polys]
    want, panic = po.kzg_check_many([c.raw for c in C], [q.raw for q in Q], Z, V, [p.raw for p in g1], [p.raw for p in g2])
    # a zero quotient (a constant polynomial) is the Infinity proof: the reference panics on those rows
    keep = [i for i in range(len(Z)) if not panic[i]]
    assert len(keep) > 100 and want[keep].all()
    got = kzg.check_batch([C[i] for i in keep], [Q[i] for i in keep], [Z[i] for i in keep], [V[i] for i in keep], g1, g2)
    assert all(got)


def _valid_rows(m, seed):
    """m openings of random polynomials, oracle-made, that the oracle's check accepts (a quotient q with q(τ) = 0 has the
    Infinity proof, on which the reference panics)."""
    g1, g2 = oracle.setup()
    rng = np.random.default_rng(seed)
    rows = []
    while len(rows) < m:
        f = rng.integers(0, 17, int(rng.integers(2, 8))).tolist()
        z = int(rng.integers(0, 17))
        row = (oracle.commit(f, g1[:len(f)]), oracle.open_(f, z, g1), z, oracle.poly_eval(17, f, z))
        try:
            if po.kzg_check(*row, g1, g2):
                rows.append(row)
        except po.OraclePanic:
            pass
    return rows


def _defined(C, Q, Z, V):
    """The rows among (C, Q, Z, V) on which the oracle's check does not panic (a changed value can make C′ Infinity or
    GEN)."""
    g1, g2 = oracle.setup()
    _, panic = po.kzg_check_many(C, Q, Z, V, g1, g2)
    keep = np.flatnonzero(~panic)
    return [C[i] for i in keep], [Q[i] for i in keep], [Z[i] for i in keep], [V[i] for i in keep]


def _check(c, C, Q, Z, V, g1d=None, g2d=None):
    from ronkathon_b200 import ops
    _, _, G1, G2 = _srs()
    return ops.kzg_check(c, _dev(C), _dev(Q), _u8(Z), _u8(V), G1 if g1d is None else g1d, G2 if g2d is None else g2d).cpu().numpy()


def test_tampered_rows_give_the_oracle_bools():
    g1, g2, _, _ = _srs()
    rng = np.random.default_rng(72)
    rows = _valid_rows(300, 73)
    pts = e17()
    C, Q, Z, V = map(list, zip(*rows))
    for i in range(len(rows)):
        kind = i % 4
        if kind == 1:
            V[i] = (V[i] + int(rng.integers(1, 17))) % 17
        elif kind == 2:
            Z[i] = (Z[i] + int(rng.integers(1, 17))) % 17
        elif kind == 3:
            Q[i] = pts[int(rng.integers(1, 289))]
    want, panic = po.kzg_check_many(C, Q, Z, V, g1, g2)
    keep = np.flatnonzero(~panic)
    assert len(keep) > 250 and want[keep].sum() > 60 and (~want[keep]).sum() > 60
    got = _check(ctx(), [C[i] for i in keep], [Q[i] for i in keep], [Z[i] for i in keep], [V[i] for i in keep])
    assert np.array_equal(got.astype(bool), want[keep])


def _grid_rows():
    """One valid proof and point; every commitment of E[17] × every value, split into the rows whose rhs is defined and
    the rows whose rhs panics (C′ = C − v·g1 is Infinity or GEN)."""
    g1, g2 = oracle.setup()
    f, z = [7, 16, 1, 11, 1], 3
    q = oracle.open_(f, z, g1)
    C = [c for c in e17() for _ in range(17)]
    V = [v for _ in e17() for v in range(17)]
    want, panic = po.kzg_check_many(C, [q] * len(C), [z] * len(C), V, g1, g2)
    return C, q, z, V, want, panic


def test_every_commitment_of_e17_under_every_value():
    C, q, z, V, want, panic = _grid_rows()
    assert panic.sum() == 2 * 17           # C′ = Infinity and C′ = GEN, once per value
    keep = np.flatnonzero(~panic)
    got = _check(ctx(), [C[i] for i in keep], [q] * len(keep), [z] * len(keep), [V[i] for i in keep])
    assert np.array_equal(got.astype(bool), want[keep])
    assert want[keep].sum() >= 17


def test_panicking_rows_one_per_call():
    from ronkathon_b200._lib import RonkPanic
    c = ctx()
    g1, g2 = oracle.setup()
    (Cv, Qv, Zv, Vv), = _valid_rows(1, 74)
    assert _check(c, [Cv], [Qv], [Zv], [Vv])[0] == 1
    bad = []
    for v in (0, 1, 9, 16):
        bad.append((_smul(g1[0], v), Qv, Zv, v))                         # C′ = Infinity
        bad.append((_add(GEN, _smul(g1[0], v)), Qv, Zv, v))              # C′ = GEN: e(GEN, GEN) panics
    for k in (2, 3, 34, 102):
        bad.append((_add(Cv, _points_of_order(k)), Qv, Zv, Vv))          # C off E[17]
        bad.append((Cv, _add(Qv, _points_of_order(k)), Zv, Vv))          # proof off E[17]
    bad.append((Cv, INF, Zv, Vv))                                        # fake proof
    bad.append((Cv, Qv, 17, Vv))
    bad.append((Cv, Qv, Zv, 200))
    bad.append((bytes([1, 0, 3, 0]), Qv, Zv, Vv))                        # off the curve
    for row in bad:
        with pytest.raises(po.OraclePanic):
            po.kzg_check(*row, g1, g2)
        with pytest.raises(RonkPanic):
            _check(c, [Cv, row[0], Cv], [Qv, row[1], Qv], [Zv, row[2], Zv], [Vv, row[3], Vv])
    # B = g2 − z·GEN off E[17] or Infinity, through a non-standard g2_srs[1]
    for g2b in (_points_of_order(51), _smul(GEN, Zv)):
        with pytest.raises(RonkPanic):
            _check(c, [Cv], [Qv], [Zv], [Vv], g2d=_dev([g2[0], g2b]))
    with pytest.raises(RonkPanic):                                       # g1_srs[0] off the curve
        _check(c, [Cv], [Qv], [Zv], [Vv], g1d=_dev([bytes([1, 0, 3, 0])]))


def test_rows_past_one_cta_and_one_grid():
    """Tiles of the E[17] grid rows to 1024·4·132·2 + 7 rows: past one CTA and past one full grid stride."""
    C, q, z, V, want, panic = _grid_rows()
    keep = np.flatnonzero(~panic)
    n = 1024 * 4 * 132 * 2 + 7
    idx = np.resize(keep, n)
    rng = np.random.default_rng(75)
    rng.shuffle(idx)
    Cb = np.frombuffer(b"".join(C), np.uint8).reshape(-1, 4)[idx]
    got = _check(ctx(), Cb, [q] * n, np.full(n, z), np.asarray(V, np.uint8)[idx])
    assert np.array_equal(got.astype(bool), want[idx])


def test_host_twin_gives_the_device_bytes():
    from ronkathon_b200 import kzg
    from ronkathon_b200.curve import AffinePoint
    c = ctx()
    g1, g2 = kzg.setup()
    rows = _valid_rows(50, 76)
    C, Q, Z, V = map(list, zip(*rows))
    V[::3] = [(v + 1) % 17 for v in V[::3]]
    C, Q, Z, V = _defined(C, Q, Z, V)
    dev = _check(c, C, Q, Z, V).astype(bool).tolist()
    host = kzg.check_batch([AffinePoint(x) for x in C], [AffinePoint(x) for x in Q], Z, V, g1 + g1, g2)
    assert host == dev and any(host) and not all(host)


def test_gated_non_blocking_stream():
    import torch
    from ronkathon_b200 import Context, ops
    rows = _valid_rows(64, 77)
    C, Q, Z, V = map(list, zip(*rows))
    V[::2] = [(v + 3) % 17 for v in V[::2]]
    C, Q, Z, V = _defined(C, Q, Z, V)
    want = _check(ctx(), C, Q, Z, V)
    _, _, G1, G2 = _srs()
    Cd, Qd, Zd, Vd = _dev(C), _dev(Q), _u8(Z), _u8(V)
    s = torch.cuda.Stream()
    c = Context(0, s.cuda_stream)
    try:
        with torch.cuda.stream(s):
            ops.kzg_check(c, Cd, Qd, Zd, Vd, G1, G2)     # warm: tables
        s.synchronize()
        Vg = torch.flip(Vd, dims=[0]).contiguous()       # scalars < 17 but the wrong rows' until the gate opens
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            torch.cuda._sleep(100_000_000)
            Vg.copy_(Vd)
            got = ops.kzg_check(c, Cd, Qd, Zd, Vg, G1, G2)
        s.synchronize()
        assert np.array_equal(got.cpu().numpy(), want)
    finally:
        c.close()


def test_launch_count_does_not_depend_on_n():
    import torch
    c = ctx()
    C, q, z, V, want, panic = _grid_rows()
    keep = np.flatnonzero(~panic)
    _, _, G1, G2 = _srs()
    Call = np.frombuffer(b"".join(C), np.uint8).reshape(-1, 4)
    _check(c, [C[keep[0]]], [q], [z], [V[keep[0]]])    # the tables are built on a context's first call
    counts = []
    for n in (1, 100, 5000, 1 << 20):
        idx = np.resize(keep, n)
        Cd = torch.from_numpy(Call[idx].copy()).cuda()
        Qd, Zd, Vd = _dev([q] * n), _u8(np.full(n, z)), _u8(np.asarray(V, np.uint8)[idx])
        ok = torch.empty(n, dtype=torch.uint8, device="cuda")
        rc, launches = _rc(c, "ronk_kzg_check_pluto_ext_batch", _p(Cd), _p(Qd), _p(Zd), _p(Vd), n, _p(G1), 7, _p(G2), 2, _p(ok))
        assert rc == 0
        counts.append(launches)
        P, Qp = _dev([e17()[1]] * n), _dev([e17()[2]] * n)
        out = torch.empty(2 * n, dtype=torch.uint8, device="cuda")
        rc, launches = _rc(c, "ronk_pairing_pluto_ext", _p(P), _p(Qp), n, _p(out))
        assert rc == 0
        counts.append(launches)
    assert counts == [1] * len(counts)


# ---- errors ----------------------------------------------------------------------------------------------------------
def test_refusals_leave_a_poisoned_ok_untouched():
    import torch
    c = ctx()
    rows = _valid_rows(8, 78)
    C, Q, Z, V = map(list, zip(*rows))
    n = len(C)
    Cd, Qd, Zd, Vd = _dev(C), _dev(Q), _u8(Z), _u8(V)
    _, _, G1, G2 = _srs()
    ok = torch.full((n + 8,), POISON, dtype=torch.uint8, device="cuda")
    o = ok[4:]
    base = [_p(Cd), _p(Qd), _p(Zd), _p(Vd), n, _p(G1), 7, _p(G2), 2, _p(o)]
    shifted = torch.empty(4 * n + 4, dtype=torch.uint8, device="cuda")
    shifted[1:4 * n + 1].copy_(Cd)
    big = torch.empty(4 * n + 8, dtype=torch.uint8, device="cuda")
    cases = {
        "n_g1 == 0": (EINVAL, {6: 0}),
        "n_g2 == 1": (EINVAL, {8: 1}),
        "n_g2 == 0": (EINVAL, {8: 0}),
        "null commitments": (EINVAL, {0: None}),
        "null proofs": (EINVAL, {1: None}),
        "null points": (EINVAL, {2: None}),
        "null values": (EINVAL, {3: None}),
        "null g1": (EINVAL, {5: None}),
        "null g2": (EINVAL, {7: None}),
        "misaligned commitments": (EINVAL, {0: _p(shifted[1:])}),
        "misaligned g2": (EINVAL, {7: _p(big[1:])}),
        "n >= 2^32": (EUNSUPPORTED, {4: 1 << 32}),
        "ok over commitments": (EINVAL, {9: _p(Cd[4:])}),
        "ok over values": (EINVAL, {9: _p(Vd)}),
        "ok over g2": (EINVAL, {9: _p(G2[3:])}),
    }
    for name, (want, patch) in cases.items():
        args = list(base)
        for k, v in patch.items():
            args[k] = v
        rc, launches = _rc(c, "ronk_kzg_check_pluto_ext_batch", *args)
        assert (rc, launches) == (want, 0), name
        assert (ok == POISON).all().item(), name
    rc, launches = _rc(c, "ronk_kzg_check_pluto_ext_batch", None, None, None, None, 0, _p(G1), 1, _p(G2), 2, None)
    assert (rc, launches) == (0, 0)
    rc, _ = _rc(c, "ronk_kzg_check_pluto_ext_batch", *base)
    assert rc == 0 and (ok[:4] == POISON).all().item() and (ok[4:4 + n] == 1).all().item() and (ok[4 + n:] == POISON).all().item()


def test_pairing_refusals_write_nothing():
    import torch
    c = ctx()
    pts = e17()
    P, Q = _dev(pts[1:9]), _dev(pts[9:17])
    out = torch.full((16,), POISON, dtype=torch.uint8, device="cuda")
    spare = torch.empty(40, dtype=torch.uint8, device="cuda")
    for args, want in (
            ((_p(P), None, 8, _p(out)), EINVAL),
            ((None, _p(Q), 8, _p(out)), EINVAL),
            ((_p(P), _p(Q), 8, None), EINVAL),
            ((_p(spare[1:]), _p(Q), 8, _p(out)), EINVAL),
            ((_p(P), _p(Q), 1 << 32, _p(out)), EUNSUPPORTED),
            ((_p(P), _p(Q), 8, _p(P[2:])), EINVAL)):
        rc, launches = _rc(c, "ronk_pairing_pluto_ext", *args)
        assert (rc, launches) == (want, 0), args
        assert (out == POISON).all().item()
    assert _rc(c, "ronk_pairing_pluto_ext", None, None, 0, None) == (0, 0)


def test_host_twins_refuse_before_staging():
    c = ctx()
    g1, g2 = oracle.setup()
    one = np.zeros(4, np.uint8)
    ok = np.full(1, POISON, np.uint8)
    g1a = np.frombuffer(b"".join(g1), np.uint8).copy()
    g2a = np.frombuffer(b"".join(g2), np.uint8).copy()
    for args, want in (
            ((_p(one), _p(one), _p(ok), _p(ok), 1, _p(g1a), 0, _p(g2a), 2, _p(ok)), EINVAL),
            ((_p(one), _p(one), _p(ok), _p(ok), 1, _p(g1a), 7, _p(g2a), 1, _p(ok)), EINVAL),
            ((None, _p(one), _p(ok), _p(ok), 1, _p(g1a), 7, _p(g2a), 2, _p(ok)), EINVAL),
            ((_p(one), _p(one), _p(ok), _p(ok), 1 << 32, _p(g1a), 7, _p(g2a), 2, _p(ok)), EUNSUPPORTED)):
        rc, launches = _rc(c, "ronk_kzg_check_pluto_ext_batch_host", *args)
        assert (rc, launches) == (want, 0)
        assert ok[0] == POISON
    out = np.full(2, POISON, np.uint8)
    assert _rc(c, "ronk_pairing_pluto_ext_host", _p(one), None, 1, _p(out)) == (EINVAL, 0)
    assert (out == POISON).all()
