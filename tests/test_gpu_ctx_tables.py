"""The tables a context builds on first use and keeps until ronk_ctx_destroy: transform plans, the 256-point-tile, pass-1
and inter-pass twiddle tables, the Bluestein spectra, the commit and pairing tables and the host pipeline's slot buffers.

One small call of each family runs on context A, then on context B created while A lives, then on B again after A is
destroyed, then on a context C created after that.  Every run must give the same words; B's and C's first calls must
build the same tables as A's, and B's calls after A's destruction must build none."""
import os

import numpy as np
import pytest

import oracle
from gpu_util import GL, BABYBEAR, dev, msm_inputs

pytestmark = pytest.mark.gpu

# profile names of the launches that fill a table the context keeps
TABLE_BUILDS = {"pow_table", "tw2d_gather", "interpass_table", "ntt3_t1", "ntt3_t2", "msm_tables", "pairing_table",
                "anyntt_chirp_table"}
# the switches of the contexts besides the default one: the inter-pass table and the histogram commit
ENVS = {"main": {}, "tw_table": {"RONK_TW_TABLE": "1"}, "hist": {"RONK_MSM_COORD": "0"}}
GEN = bytes([36, 0, 0, 31])


def _contexts():
    import torch
    from ronkathon_b200 import Context
    out = {}
    for name, env in ENVS.items():
        old = {k: os.environ.get(k) for k in env}
        os.environ.update(env)
        try:
            out[name] = Context(0, torch.cuda.current_stream().cuda_stream)
        finally:
            for k, v in old.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
        out[name].prof_enable(True)
    return out


def _ntt(log_n, batch=1, inverse=False, p=GL, g=7, seed=0):
    def run(c):
        from ronkathon_b200 import ops
        d = dev(oracle.splitmix(p, 7000 + seed, batch << log_n))
        ops.ntt_(c, d, log_n, batch, inverse=inverse, p=p, g=g)
        return ops.to_host(d)
    return run


def _ntt_any(n):
    def run(c):
        from ronkathon_b200 import ops
        d = dev(oracle.splitmix(GL, 7100, n))
        ops.ntt_any_(c, d, n)
        return ops.to_host(d)
    return run


def _commit(c):
    import torch
    from ronkathon_b200 import ops
    pts, sc = msm_inputs(200)
    return np.frombuffer(ops.msm(c, torch.from_numpy(pts).cuda(), torch.from_numpy(sc).cuda()), dtype=np.uint8)


def _pairing(c):
    import torch
    from ronkathon_b200 import ops
    g1 = bytes(oracle.setup()[0][0])
    P = np.frombuffer(g1 + GEN, dtype=np.uint8).copy()
    Q = np.frombuffer(GEN + oracle.point_add(g1, GEN), dtype=np.uint8).copy()
    return ops.pairing(c, torch.from_numpy(P).cuda(), torch.from_numpy(Q).cuda()).cpu().numpy()


def _host_slots(c):
    import torch
    bufs = [torch.from_numpy(oracle.splitmix(GL, 7200 + s, 1 << 12).view(np.int64)).pin_memory() for s in range(3)]
    for s, t in enumerate(bufs):
        c.call("ronk_ntt_u64_host_submit", GL, 7, t.data_ptr(), 12, 1, 0, s)
    for s in range(3):
        c.call("ronk_ntt_u64_host_wait", s)
    return np.concatenate([t.numpy().view(np.uint64) for t in bufs])


# (name, context, call): one small call of each table family, in this order on every context
CALLS = [
    ("single_tile", "main", _ntt(10)),
    ("two_pass", "main", _ntt(14)),
    ("babybear", "main", _ntt(14, p=BABYBEAR, g=31)),
    ("ntt16_cluster", "main", _ntt(16)),
    ("ntt16_tiles", "main", _ntt(16, batch=3, inverse=True)),
    ("split_2^17", "main", _ntt(17)),
    ("t1_2^20", "main", _ntt(20)),
    ("interpass", "tw_table", _ntt(14, seed=1)),
    ("bluestein", "main", _ntt_any(3 << 11)),
    ("commit_coord", "main", _commit),
    ("commit_hist", "hist", _commit),
    ("pairing", "main", _pairing),
    ("host_slots", "main", _host_slots),
]


def _run(ctxs):
    """{call: (words, profile names)}"""
    out = {}
    for name, which, call in CALLS:
        c = ctxs[which]
        words = call(c)
        c.sync()
        out[name] = (np.asarray(words).tobytes(), [n for n, _ in c.prof_fetch()])
    return out


def test_tables_survive_destroying_another_context():
    a = _contexts()
    first_a = _run(a)
    built = set().union(*(set(names) & TABLE_BUILDS for _, names in first_a.values()))
    assert built == TABLE_BUILDS, f"table families not exercised: {TABLE_BUILDS - built}"

    b = _contexts()
    first_b = _run(b)
    for name, _, _ in CALLS:
        assert first_b[name][0] == first_a[name][0], name
        assert first_b[name][1] == first_a[name][1], name

    for c in a.values():
        c.close()
    again_b = _run(b)
    for name, _, _ in CALLS:
        assert again_b[name][0] == first_a[name][0], name
        assert not set(again_b[name][1]) & TABLE_BUILDS, (name, again_b[name][1])

    c_ctxs = _contexts()
    first_c = _run(c_ctxs)
    for name, _, _ in CALLS:
        assert first_c[name][0] == first_a[name][0], name
        assert first_c[name][1] == first_b[name][1], name
    for c in list(b.values()) + list(c_ctxs.values()):
        c.close()
