"""The launch record of each public call: the profile names it records, in order, and the launch count it adds.

bench.py reports both (`kernel_ms` names, `gpu_launches`), and a change to the host-side launch plumbing must not add,
drop, rename or reorder a launch.  Every call is warmed once first, so one-time plan and table builds are not part of
the record."""
import ctypes as C

import numpy as np
import pytest

import oracle
from gpu_util import BABYBEAR, GL, MONT_PRIMES, ctx, dev, msm_inputs

pytestmark = pytest.mark.gpu

BB_G = MONT_PRIMES["babybear"][1]


def _ntt(log_n, batch=1, inverse=False, p=GL, g=7):
    from ronkathon_b200 import ops
    x = dev(oracle.splitmix(p, 11, batch << log_n))
    return lambda c: ops.ntt_(c, x, log_n, batch, inverse=inverse, p=p, g=g)


def _ntt_mul(log_n):
    from ronkathon_b200 import ops
    x, m = dev(oracle.splitmix(GL, 12, 1 << log_n)), dev(oracle.splitmix(GL, 13, 1 << log_n))
    return lambda c: ops.ntt_mul_(c, x, m, log_n)


def _poly_mul(da, db, p=GL, g=7):
    from ronkathon_b200 import ops
    a, b = dev(oracle.splitmix(p, 14, da)), dev(oracle.splitmix(p, 15, db))
    return lambda c: ops.poly_mul(c, a, b, p=p, g=g)


def _poly_mul_host(da, db):
    from ronkathon_b200 import _lib
    a, b = oracle.splitmix(GL, 14, da), oracle.splitmix(GL, 15, db)
    out = np.empty(da + db - 1, dtype=np.uint64)
    return lambda c: c.call("ronk_poly_mul_u64_host", GL, 7, _lib._ptr(a), da, _lib._ptr(b), db, _lib._ptr(out))


def _binop(name, p):
    import torch
    from ronkathon_b200 import _lib
    a, b = dev(oracle.splitmix(p, 16, 4096)), dev(oracle.splitmix(p - 1, 17, 4096) + 1)
    out = torch.empty_like(a)
    return lambda c: c.call(f"ronk_field_{name}_u64", p, _lib._ptr(a), _lib._ptr(b), _lib._ptr(out), 4096)


def _binop_host(op, p):
    from ronkathon_b200 import _lib
    a, b = oracle.splitmix(p, 16, 4096), oracle.splitmix(p - 1, 17, 4096) + 1
    out = np.empty(4096, dtype=np.uint64)
    return lambda c: c.call("ronk_field_binop_u64_host", op, p, _lib._ptr(a), _lib._ptr(b), _lib._ptr(out), 4096)


def _unop(name, p):
    import torch
    from ronkathon_b200 import _lib
    a = dev(oracle.splitmix(p - 1, 18, 4096) + 1)
    out = torch.empty_like(a)
    if name == "pow":
        return lambda c: c.call("ronk_field_pow_u64", p, _lib._ptr(a), 0xDEADBEEF, _lib._ptr(out), 4096)
    return lambda c: c.call(f"ronk_field_{name}_u64", p, _lib._ptr(a), _lib._ptr(out), 4096)


def _powers(p):
    import torch
    from ronkathon_b200 import _lib
    out = torch.empty(1 << 16, dtype=torch.int64, device="cuda")
    return lambda c: c.call("ronk_field_powers_u64", p, 3, 5, _lib._ptr(out), out.numel())


def _strided(p, g):
    from ronkathon_b200 import _lib
    x = dev(oracle.splitmix(p, 19, 1 << 12))
    return lambda c: c.call("ronk_ntt_strided_small_u64", p, g, _lib._ptr(x), 4, 256, 256, 0)


def _poly_addsub(name, p):
    import torch
    from ronkathon_b200 import _lib
    a, b = dev(oracle.splitmix(p, 20, 5000)), dev(oracle.splitmix(p, 21, 3000))
    out = torch.empty_like(a)
    return lambda c: c.call(f"ronk_poly_{name}_u64", p, _lib._ptr(a), 5000, _lib._ptr(b), 3000, _lib._ptr(out))


def _poly_eval(p):
    import torch
    from ronkathon_b200 import _lib
    a, xs = dev(oracle.splitmix(p, 22, 5000)), dev(oracle.splitmix(p, 23, 64))
    out = torch.empty_like(xs)
    return lambda c: c.call("ronk_poly_eval_u64", p, _lib._ptr(a), 5000, _lib._ptr(xs), 64, _lib._ptr(out))


def _dft(p, g):
    import torch
    from ronkathon_b200 import _lib
    a = dev(oracle.splitmix(p, 24, 1024))
    out = torch.empty_like(a)
    return lambda c: c.call("ronk_dft_u64", p, g, _lib._ptr(a), 1024, _lib._ptr(out))


def _dft_host(p, g):
    from ronkathon_b200 import _lib
    a = oracle.splitmix(p, 24, 1024)
    out = np.empty_like(a)
    return lambda c: c.call("ronk_dft_u64_host", p, g, _lib._ptr(a), 1024, _lib._ptr(out))


def _lagrange(p, g):
    from ronkathon_b200 import _lib
    coeffs = oracle.splitmix(p, 25, 256)
    res = C.c_uint64()
    return lambda c: c.call("ronk_poly_lagrange_eval_u64_host", p, g, _lib._ptr(coeffs), 256, 12345, C.byref(res))


def _interpolate(p):
    from ronkathon_b200 import _lib
    xs, ys = np.arange(1, 301, dtype=np.uint64), oracle.splitmix(p, 26, 300)
    out = np.empty(300, dtype=np.uint64)
    return lambda c: c.call("ronk_poly_interpolate_u64_host", p, _lib._ptr(xs), _lib._ptr(ys), 300, _lib._ptr(out))


def _divrem(divisor, p):
    from ronkathon_b200 import _lib
    a, b = oracle.splitmix(p, 27, 3000), np.array(divisor, dtype=np.uint64)
    q, r = np.empty(3000, dtype=np.uint64), np.empty(3000, dtype=np.uint64)
    return lambda c: c.call("ronk_poly_divrem_u64_host", p, _lib._ptr(a), 3000, _lib._ptr(b), len(b), _lib._ptr(q),
                            _lib._ptr(r))


def _div_linear(p):
    import torch
    from ronkathon_b200 import _lib
    d = 1 << 20
    a = dev(oracle.splitmix(p, 28, d))
    q, rem = torch.empty_like(a), torch.empty(1, dtype=torch.int64, device="cuda")
    return lambda c: c.call("ronk_poly_div_linear_u64", p, _lib._ptr(a), d, p - 5, 1, _lib._ptr(q), _lib._ptr(rem))


def _dist_virtual(flavour, p, g):
    from ronkathon_b200 import _lib
    x = dev(oracle.splitmix(p, 29, 3 << 12))
    return lambda c: c.call("ronk_ntt_u64_dist_virtual", p, g, _lib._ptr(x), 12, 3, 2, flavour)


def _msm():
    import torch
    from ronkathon_b200 import ops
    pts, sc = msm_inputs(1 << 16)
    P, S = torch.from_numpy(pts.reshape(-1)).cuda(), torch.from_numpy(sc).cuda()
    return lambda c: ops.msm(c, P, S)


def _msm_host():
    from ronkathon_b200 import _lib
    pts, sc = msm_inputs(1 << 16)
    out = np.empty(4, dtype=np.uint8)
    return lambda c: c.call("ronk_msm_pluto_ext_host", _lib._ptr(pts), len(sc), _lib._ptr(sc), len(sc), _lib._ptr(out))


def _splitmix():
    import torch
    from ronkathon_b200 import ops
    out = torch.empty(1 << 16, dtype=torch.int64, device="cuda")
    return lambda c: ops.splitmix_fill(c, out.numel(), 7)


_NTT3 = ["ntt3_pass1", "ntt3_pass2", "ntt3_pass3"]
_INTT3 = ["intt3_pass1", "intt3_pass2", "intt3_pass3"]
_POLY_MUL_SINGLE = ["ntt_single", "ntt_single", "intt_single"]
_DIV_LINEAR = ["div_linear_fold", "div_linear_carry", "div_linear_apply"]
CASES = {
    # id: (factory of the call, profile names it records in launch order)
    "ntt_gl_2^10": (lambda: _ntt(10), ["ntt_single"]),
    "ntt_gl_2^16": (lambda: _ntt(16), ["ntt16_cluster"]),
    "ntt_gl_2^16_batch512": (lambda: _ntt(16, 512), ["ntt3_pass2", "ntt3_pass3"]),
    "ntt_gl_2^18": (lambda: _ntt(18), ["ntt3_split", "ntt3_pass2", "ntt3_pass3"]),
    "ntt_gl_2^20": (lambda: _ntt(20), ["ntt3_a1", "ntt3_a2", "ntt3_c"]),
    "intt_gl_2^20": (lambda: _ntt(20, inverse=True), ["intt3_a1", "intt3_a2", "intt3_c"]),
    "ntt_gl_2^22": (lambda: _ntt(22), _NTT3),
    "ntt_gl_2^24": (lambda: _ntt(24), _NTT3),
    "intt_gl_2^24": (lambda: _ntt(24, inverse=True), _INTT3),
    "ntt_gl_2^25": (lambda: _ntt(25), ["ntt3_split"] + _NTT3),
    "ntt_mul_gl_2^16": (lambda: _ntt_mul(16), ["ntt16_cluster"]),
    "ntt_mul_gl_2^24": (lambda: _ntt_mul(24), _NTT3),
    "ntt_babybear_2^20": (lambda: _ntt(20, p=BABYBEAR, g=BB_G), ["ntt_pass1", "ntt_pass2"]),
    "poly_mul_schoolbook": (lambda: _poly_mul(64, 64), ["poly_mul_schoolbook"]),
    "poly_mul_ntt": (lambda: _poly_mul(256, 256), _POLY_MUL_SINGLE),
    "poly_mul_2^23x2^23": (lambda: _poly_mul(1 << 23, 1 << 23), _NTT3 + _NTT3 + _INTT3),
    "poly_mul_babybear_ntt": (lambda: _poly_mul(256, 256, p=BABYBEAR, g=BB_G), _POLY_MUL_SINGLE),
    "poly_mul_gl_g0": (lambda: _poly_mul(256, 256, g=0), ["poly_mul_schoolbook"]),
    "poly_mul_host_schoolbook": (lambda: _poly_mul_host(64, 64), ["poly_mul_schoolbook"]),
    "poly_mul_host_ntt": (lambda: _poly_mul_host(256, 256), _POLY_MUL_SINGLE),
    "msm": (_msm, ["msm_coord"]),
    "msm_host": (_msm_host, ["msm_coord"]),
    "splitmix_fill": (_splitmix, ["splitmix_fill"]),
}
for _pn, _p, _g in (("gl", GL, 7), ("babybear", BABYBEAR, BB_G)):
    CASES.update({
        **{f"field_{op}_{_pn}": ((lambda op=op, p=_p: _binop(op, p)), [f"field_{op}"]) for op in ("add", "sub", "mul", "div")},
        **{f"field_{op}_{_pn}": ((lambda op=op, p=_p: _unop(op, p)), [f"field_{op}"]) for op in ("neg", "inv", "pow")},
        f"field_powers_{_pn}": ((lambda p=_p: _powers(p)), ["field_powers"]),
        f"ntt_strided_small_{_pn}": ((lambda p=_p, g=_g: _strided(p, g)), ["ntt_cross_rank"]),
        f"poly_add_{_pn}": ((lambda p=_p: _poly_addsub("add", p)), ["poly_add"]),
        f"poly_sub_{_pn}": ((lambda p=_p: _poly_addsub("sub", p)), ["poly_sub"]),
        f"poly_eval_{_pn}": ((lambda p=_p: _poly_eval(p)), ["poly_eval"]),
        f"field_div_host_{_pn}": ((lambda p=_p: _binop_host(3, p)), ["field_div"]),
        f"dft_{_pn}": ((lambda p=_p, g=_g: _dft(p, g)), ["pow_table", "poly_eval"]),
        f"dft_host_{_pn}": ((lambda p=_p, g=_g: _dft_host(p, g)), ["pow_table", "poly_eval"]),
        f"lagrange_eval_{_pn}": ((lambda p=_p, g=_g: _lagrange(p, g)), ["pow_table", "lagrange_eval"]),
        f"interpolate_{_pn}": ((lambda p=_p: _interpolate(p)), ["interp_master", "interp_nodes", "interp_sum"]),
        f"divrem_linear_{_pn}": ((lambda p=_p: _divrem([5, 1], p)), _DIV_LINEAR),
        f"divrem_quadratic_{_pn}": ((lambda p=_p: _divrem([5, 2, 1], p)), ["poly_divrem"]),
        f"div_linear_{_pn}": ((lambda p=_p: _div_linear(p)), _DIV_LINEAR),
        # four virtual ranks: local transforms (ranks 1-3 build their twiddle column first), then four cross-rank stages
        f"dist_virtual_fused_{_pn}": ((lambda p=_p, g=_g: _dist_virtual(1, p, g)),
                                      ["ntt_single"] + ["field_powers", "ntt_single"] * 3 + ["ntt_cross_rank"] * 4),
        f"dist_virtual_exchange_{_pn}": ((lambda p=_p, g=_g: _dist_virtual(0, p, g)),
                                         ["ntt_single", "dist_pack"] + ["field_powers", "ntt_single", "dist_pack"] * 3
                                         + ["ntt_cross_rank"] * 4),
    })


def record(run):
    """Warm `run` once, then return (profile names of one profiled call, launches of one unprofiled call)."""
    c = ctx()
    run(c)
    c.sync()
    c.prof_fetch()
    c.prof_enable(True)
    try:
        run(c)
        names = [n for n, _ in c.prof_fetch()]
    finally:
        c.prof_enable(False)
    before = c.launches
    run(c)
    c.sync()
    return names, c.launches - before


@pytest.mark.parametrize("case", list(CASES))
def test_launch_record(case):
    factory, expected = CASES[case]
    names, launches = record(factory())
    assert names == expected
    assert launches == len(expected)
