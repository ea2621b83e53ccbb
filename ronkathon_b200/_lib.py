"""ctypes binding of libronk_b200.so (include/ronk_b200.h).  There is NO CPU fallback: if the
shared library is missing, or no H100 is visible when a context is created, this raises."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("RONK_LIB_PATH") or os.path.join(_HERE, "libronk_b200.so")  # override: experiments only

OK, EINVAL, ECUDA, ENOMEM, ENCCL, EUNSUPPORTED = 0, 1, 2, 3, 4, 5
GOLDILOCKS = 0xFFFFFFFF00000001

u64, u32, i32, sz = C.c_uint64, C.c_uint32, C.c_int, C.c_size_t
p64, pu8, vp = C.POINTER(C.c_uint64), C.POINTER(C.c_uint8), C.c_void_p

# name → (restype, argtypes); every symbol include/ronk_b200.h declares
SIGNATURES = {
    "ronk_ctx_create": (i32, [C.POINTER(vp), i32, vp]),
    "ronk_ctx_destroy": (i32, [vp]),
    "ronk_ctx_set_stream": (i32, [vp, vp]),
    "ronk_sync": (i32, [vp]),
    "ronk_strerror": (C.c_char_p, [i32]),
    "ronk_last_error": (C.c_char_p, [vp]),
    "ronk_launch_count": (u64, [vp]),
    "ronk_prof_enable": (i32, [vp, i32]),
    "ronk_prof_fetch": (i32, [vp, vp, C.POINTER(C.c_float), i32]),
    "ronk_dev_alloc": (i32, [vp, C.POINTER(vp), sz]),
    "ronk_dev_free": (i32, [vp, vp]),
    "ronk_memcpy_h2d": (i32, [vp, vp, vp, sz]),
    "ronk_memcpy_d2h": (i32, [vp, vp, vp, sz]),
    "ronk_field_generator": (i32, [u64, p64]),
    "ronk_root_of_unity": (i32, [u64, u64, u64, p64]),
    "ronk_field_add_u64": (i32, [vp, u64, vp, vp, vp, sz]),
    "ronk_field_sub_u64": (i32, [vp, u64, vp, vp, vp, sz]),
    "ronk_field_mul_u64": (i32, [vp, u64, vp, vp, vp, sz]),
    "ronk_field_div_u64": (i32, [vp, u64, vp, vp, vp, sz]),
    "ronk_field_neg_u64": (i32, [vp, u64, vp, vp, sz]),
    "ronk_field_inv_u64": (i32, [vp, u64, vp, vp, sz]),
    "ronk_field_pow_u64": (i32, [vp, u64, vp, u64, vp, sz]),
    "ronk_field_binop_u64_host": (i32, [vp, i32, u64, vp, vp, vp, sz]),
    "ronk_field_unop_u64_host": (i32, [vp, i32, u64, vp, vp, sz]),
    "ronk_field_pow_u64_host": (i32, [vp, u64, vp, u64, vp, sz]),
    "ronk_ntt_u64": (i32, [vp, u64, u64, vp, u32, u32, i32]),
    "ronk_ntt_u64_host": (i32, [vp, u64, u64, vp, u32, u32, i32]),
    "ronk_ntt_u64_host_submit": (i32, [vp, u64, u64, vp, u32, u32, i32, i32]),
    "ronk_ntt_u64_host_wait": (i32, [vp, i32]),
    "ronk_ntt_mul_u64": (i32, [vp, u64, u64, vp, vp, u32, u32]),
    "ronk_field_powers_u64": (i32, [vp, u64, u64, u64, vp, sz]),
    "ronk_ntt_strided_small_u64": (i32, [vp, u64, u64, vp, u32, sz, sz, i32]),
    "ronk_ntt_cross_rank_fused_u64": (i32, [vp, u64, u64, vp, u32, u32, u32, vp]),
    "ronk_ipc_export": (i32, [vp, vp, vp]),
    "ronk_ipc_open": (i32, [vp, vp, C.POINTER(vp)]),
    "ronk_ipc_close": (i32, [vp, vp]),
    "ronk_memcpy_d2d": (i32, [vp, vp, vp, sz]),
    "ronk_dft_u64": (i32, [vp, u64, u64, vp, u64, vp]),
    "ronk_dft_u64_host": (i32, [vp, u64, u64, vp, u64, vp]),
    "ronk_ntt_any_u64": (i32, [vp, u64, u64, vp, u64, u32, i32]),
    "ronk_ntt_any_u64_host": (i32, [vp, u64, u64, vp, u64, u32, i32]),
    "ronk_ntt_coset_u64": (i32, [vp, u64, u64, vp, u32, u32, u64, i32]),
    "ronk_ntt_coset_u64_host": (i32, [vp, u64, u64, vp, u32, u32, u64, i32]),
    "ronk_poly_lde_u64": (i32, [vp, u64, u64, vp, sz, u32, u64, u32, vp]),
    "ronk_poly_lde_u64_host": (i32, [vp, u64, u64, vp, sz, u32, u64, u32, vp]),
    "ronk_poly_mul_u64": (i32, [vp, u64, u64, vp, sz, vp, sz, vp]),
    "ronk_poly_mul_u64_host": (i32, [vp, u64, u64, vp, sz, vp, sz, vp]),
    "ronk_poly_mul_batch_u64": (i32, [vp, u64, u64, vp, sz, vp, sz, i32, u32, vp]),
    "ronk_poly_mul_batch_u64_host": (i32, [vp, u64, u64, vp, sz, vp, sz, i32, u32, vp]),
    "ronk_poly_add_u64": (i32, [vp, u64, vp, sz, vp, sz, vp]),
    "ronk_poly_sub_u64": (i32, [vp, u64, vp, sz, vp, sz, vp]),
    "ronk_poly_eval_u64": (i32, [vp, u64, vp, sz, vp, sz, vp]),
    "ronk_poly_eval_u64_host": (i32, [vp, u64, vp, sz, vp, sz, vp]),
    "ronk_poly_lagrange_eval_u64_host": (i32, [vp, u64, u64, vp, sz, u64, p64]),
    "ronk_poly_lagrange_eval_u64": (i32, [vp, u64, u64, vp, u64, u32, u64, vp, sz, vp]),
    "ronk_poly_lagrange_eval_batch_u64_host": (i32, [vp, u64, u64, vp, u64, u32, u64, vp, sz, vp]),
    "ronk_poly_lagrange_open_u64": (i32, [vp, u64, u64, vp, u64, u32, u64, u64, vp, vp]),
    "ronk_poly_lagrange_open_u64_host": (i32, [vp, u64, u64, vp, u64, u32, u64, u64, vp, vp]),
    "ronk_poly_divrem_u64_host": (i32, [vp, u64, vp, sz, vp, sz, vp, vp]),
    "ronk_poly_divrem_u64": (i32, [vp, u64, u64, vp, sz, vp, sz, vp, vp]),
    "ronk_poly_divrem_batch_u64": (i32, [vp, u64, u64, vp, sz, vp, sz, i32, u32, vp, vp]),
    "ronk_poly_divrem_batch_u64_host": (i32, [vp, u64, u64, vp, sz, vp, sz, i32, u32, vp, vp]),
    "ronk_poly_div_linear_u64": (i32, [vp, u64, vp, sz, u64, u64, vp, vp]),
    "ronk_poly_interpolate_u64_host": (i32, [vp, u64, vp, vp, sz, vp]),
    "ronk_poly_from_roots_u64": (i32, [vp, u64, u64, vp, sz, vp]),
    "ronk_poly_multieval_u64": (i32, [vp, u64, u64, vp, sz, vp, sz, vp]),
    "ronk_poly_interpolate_u64": (i32, [vp, u64, u64, vp, vp, sz, vp]),
    "ronk_poly_multieval_batch_u64": (i32, [vp, u64, u64, vp, sz, u32, vp, sz, vp]),
    "ronk_poly_multieval_batch_u64_host": (i32, [vp, u64, u64, vp, sz, u32, vp, sz, vp]),
    "ronk_poly_interpolate_batch_u64": (i32, [vp, u64, u64, vp, vp, sz, u32, vp]),
    "ronk_poly_interpolate_batch_u64_host": (i32, [vp, u64, u64, vp, vp, sz, u32, vp]),
    "ronk_rs_encode_u64": (i32, [vp, u64, u64, vp, u64, u64, u32, vp]),
    "ronk_rs_decode_u64": (i32, [vp, u64, u64, vp, vp, u64, u64, u32, vp, vp]),
    "ronk_rs_decode_u64_host": (i32, [vp, u64, u64, vp, vp, u64, u64, u32, vp, vp]),
    "ronk_rs_decode_at_u64": (i32, [vp, u64, u64, vp, vp, vp, u64, u64, u32, vp, vp]),
    "ronk_rs_decode_at_u64_host": (i32, [vp, u64, u64, vp, vp, vp, u64, u64, u32, vp, vp]),
    "ronk_point_add_pluto_ext_host": (i32, [vp, vp, vp, vp, sz]),
    "ronk_point_neg_pluto_ext_host": (i32, [vp, vp, vp, sz]),
    "ronk_point_smul_pluto_ext_host": (i32, [vp, vp, vp, vp, sz]),
    "ronk_msm_pluto_ext": (i32, [vp, vp, sz, vp, sz, vp]),
    "ronk_msm_pluto_ext_host": (i32, [vp, vp, sz, vp, sz, vp]),
    "ronk_msm_pluto_ext_batch": (i32, [vp, vp, sz, vp, sz, u32, vp]),
    "ronk_msm_pluto_ext_batch_host": (i32, [vp, vp, sz, vp, sz, u32, vp]),
    "ronk_pairing_pluto_ext": (i32, [vp, vp, vp, sz, vp]),
    "ronk_pairing_pluto_ext_host": (i32, [vp, vp, vp, sz, vp]),
    "ronk_kzg_check_pluto_ext_batch": (i32, [vp, vp, vp, vp, vp, sz, vp, sz, vp, sz, vp]),
    "ronk_kzg_check_pluto_ext_batch_host": (i32, [vp, vp, vp, vp, vp, sz, vp, sz, vp, sz, vp]),
    "ronk_poseidon_permute_u64": (i32, [vp, u64, u32, u64, u32, u32, vp, vp, vp, sz]),
    "ronk_poseidon_permute_u64_host": (i32, [vp, u64, u32, u64, u32, u32, vp, vp, vp, sz]),
    "ronk_poseidon_sponge_u64": (i32, [vp, u64, u32, u64, u32, u32, vp, vp, u32, vp, sz, sz, vp, sz]),
    "ronk_poseidon_sponge_u64_host": (i32, [vp, u64, u32, u64, u32, u32, vp, vp, u32, vp, sz, sz, vp, sz]),
    "ronk_sha256": (i32, [vp, vp, u64, vp, sz, vp]),
    "ronk_sha256_host": (i32, [vp, vp, u64, vp, sz, vp]),
    "ronk_merkle_build_sha256": (i32, [vp, vp, u64, vp, sz, vp]),
    "ronk_merkle_build_sha256_host": (i32, [vp, vp, u64, vp, sz, vp]),
    "ronk_merkle_proofs_sha256": (i32, [vp, vp, sz, vp, sz, vp, vp]),
    "ronk_merkle_proofs_sha256_host": (i32, [vp, vp, sz, vp, sz, vp, vp]),
    "ronk_merkle_verify_sha256": (i32, [vp, vp, vp, u64, vp, sz, vp, vp, u32, vp]),
    "ronk_merkle_verify_sha256_host": (i32, [vp, vp, vp, u64, vp, sz, vp, vp, u32, vp]),
    "ronk_msm_pluto_ext_buckets": (i32, [vp, vp, sz, vp, sz, vp]),
    "ronk_msm_combine_buckets_host": (i32, [vp, vp, sz, vp]),
    "ronk_splitmix_fill_u64": (i32, [vp, u64, u64, vp, sz]),
    "ronk_dist_unique_id": (i32, [vp]),
    "ronk_dist_init": (i32, [vp, vp, i32, i32]),
    "ronk_dist_init_comm": (i32, [vp, vp, i32, i32]),
    "ronk_dist_finalize": (i32, [vp]),
    "ronk_dist_rank": (i32, [vp, C.POINTER(i32), C.POINTER(i32)]),
    "ronk_dist_barrier": (i32, [vp]),
    "ronk_dist_shard_range": (i32, [u64, i32, i32, p64, p64]),
    "ronk_ntt_u64_batch_sharded": (i32, [vp, u64, u64, vp, u32, u64, i32, p64, p64]),
    "ronk_ntt_u64_dist": (i32, [vp, u64, u64, vp, u32, u32, i32]),
    "ronk_ntt_u64_dist_virtual": (i32, [vp, u64, u64, vp, u32, u32, u32, i32]),
    "ronk_msm_pluto_ext_dist": (i32, [vp, vp, sz, vp, sz, vp]),
}

_lib = None


class RonkError(RuntimeError):
    """A non-zero return code from libronk_b200 (code EINVAL = the reference would panic)."""

    def __init__(self, code: int, detail: str = ""):
        self.code = code
        super().__init__(f"ronk error {code}: {detail}")


class RonkPanic(RonkError):
    """RONK_EINVAL: the input on which ronkathon's own code panics / asserts / unwraps None."""


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU fallback)")
        _lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(_lib, name)
            fn.restype, fn.argtypes = res, args
    return _lib


def _ptr(x):
    """device pointer (int / torch tensor) or host numpy array → c_void_p"""
    if x is None:
        return None
    if isinstance(x, np.ndarray):
        return x.ctypes.data_as(vp)
    if hasattr(x, "data_ptr"):
        return vp(x.data_ptr())
    return vp(int(x))


class Context:
    """ronk_ctx: device + stream + plan cache.  `stream` is a raw cudaStream_t handle (int)."""

    def __init__(self, device: int = 0, stream: int | None = None):
        self._h = vp()
        rc = lib().ronk_ctx_create(C.byref(self._h), device, vp(stream) if stream else None)
        if rc != OK:
            self._h = None
            raise RonkError(rc, "ronk_ctx_create failed — an H100 (sm_90) GPU is required; no CPU fallback exists")
        self.device = device
        self.stream = int(stream) if stream else 0   # raw cudaStream_t the context enqueues on (0 = legacy default)

    def check(self, rc: int):
        if rc == OK:
            return
        detail = lib().ronk_last_error(self._h).decode() or lib().ronk_strerror(rc).decode()
        raise (RonkPanic if rc == EINVAL else RonkError)(rc, detail)

    def call(self, name: str, *args):
        self.check(getattr(lib(), name)(self._h, *args))

    def sync(self):
        self.call("ronk_sync")

    def set_stream(self, stream: int):
        self.call("ronk_ctx_set_stream", vp(stream) if stream else None)
        self.stream = int(stream) if stream else 0

    @property
    def launches(self) -> int:
        return lib().ronk_launch_count(self._h)

    def prof_enable(self, on: bool):
        self.call("ronk_prof_enable", int(on))

    def prof_fetch(self, max_records: int = 4096):
        names = (C.c_char * 32 * max_records)()
        ms = (C.c_float * max_records)()
        n = lib().ronk_prof_fetch(self._h, C.cast(names, vp), ms, max_records)
        return [(names[i].value.decode(), float(ms[i])) for i in range(n)]

    def close(self):
        if getattr(self, "_h", None):
            lib().ronk_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


_default_ctx = None


def default_context() -> Context:
    global _default_ctx
    if _default_ctx is None:
        _default_ctx = Context(int(os.environ.get("LOCAL_RANK", "0")) if os.environ.get("RONK_USE_LOCAL_RANK") else 0)
    return _default_ctx


def set_default_context(ctx: Context):
    global _default_ctx
    _default_ctx = ctx
