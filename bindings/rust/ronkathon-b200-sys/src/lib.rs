//! Raw FFI of libronk_b200.so — mirrors include/ronk_b200.h declaration by declaration.
//! UNBUILT: the environment this was written in has no Rust toolchain.
#![allow(non_camel_case_types)]
use core::ffi::{c_char, c_int, c_void};

pub const RONK_OK: c_int = 0;
pub const RONK_EINVAL: c_int = 1; // the reference would panic/assert
pub const RONK_ECUDA: c_int = 2;
pub const RONK_ENOMEM: c_int = 3;
pub const RONK_ENCCL: c_int = 4;
pub const RONK_EUNSUPPORTED: c_int = 5;
pub const RONK_GOLDILOCKS: u64 = 0xFFFF_FFFF_0000_0001;

#[repr(C)]
pub struct ronk_ctx {
  _private: [u8; 0],
}

extern "C" {
  pub fn ronk_ctx_create(out: *mut *mut ronk_ctx, device: c_int, stream: *mut c_void) -> c_int;
  pub fn ronk_ctx_destroy(ctx: *mut ronk_ctx) -> c_int;
  pub fn ronk_ctx_set_stream(ctx: *mut ronk_ctx, stream: *mut c_void) -> c_int;
  pub fn ronk_sync(ctx: *mut ronk_ctx) -> c_int;
  pub fn ronk_strerror(code: c_int) -> *const c_char;
  pub fn ronk_last_error(ctx: *mut ronk_ctx) -> *const c_char;
  pub fn ronk_launch_count(ctx: *mut ronk_ctx) -> u64;
  pub fn ronk_prof_enable(ctx: *mut ronk_ctx, on: c_int) -> c_int;
  pub fn ronk_prof_fetch(ctx: *mut ronk_ctx, names: *mut [c_char; 32], ms: *mut f32, max: c_int) -> c_int;
  pub fn ronk_dev_alloc(ctx: *mut ronk_ctx, dptr: *mut *mut c_void, bytes: usize) -> c_int;
  pub fn ronk_dev_free(ctx: *mut ronk_ctx, dptr: *mut c_void) -> c_int;
  pub fn ronk_memcpy_h2d(ctx: *mut ronk_ctx, dst: *mut c_void, src: *const c_void, bytes: usize) -> c_int;
  pub fn ronk_memcpy_d2h(ctx: *mut ronk_ctx, dst: *mut c_void, src: *const c_void, bytes: usize) -> c_int;

  // FiniteField (src/algebra/field/mod.rs:54-76, prime/mod.rs:87-123)
  pub fn ronk_field_generator(p: u64, g: *mut u64) -> c_int;
  pub fn ronk_root_of_unity(p: u64, g: u64, n: u64, out: *mut u64) -> c_int;

  // PrimeField<P> operators (prime/arithmetic.rs:3-71, prime/mod.rs:62-84)
  pub fn ronk_field_add_u64(ctx: *mut ronk_ctx, p: u64, a: *const u64, b: *const u64, out: *mut u64, n: usize) -> c_int;
  pub fn ronk_field_sub_u64(ctx: *mut ronk_ctx, p: u64, a: *const u64, b: *const u64, out: *mut u64, n: usize) -> c_int;
  pub fn ronk_field_mul_u64(ctx: *mut ronk_ctx, p: u64, a: *const u64, b: *const u64, out: *mut u64, n: usize) -> c_int;
  pub fn ronk_field_div_u64(ctx: *mut ronk_ctx, p: u64, a: *const u64, b: *const u64, out: *mut u64, n: usize) -> c_int;
  pub fn ronk_field_neg_u64(ctx: *mut ronk_ctx, p: u64, a: *const u64, out: *mut u64, n: usize) -> c_int;
  pub fn ronk_field_inv_u64(ctx: *mut ronk_ctx, p: u64, a: *const u64, out: *mut u64, n: usize) -> c_int;
  pub fn ronk_field_pow_u64(ctx: *mut ronk_ctx, p: u64, a: *const u64, e: u64, out: *mut u64, n: usize) -> c_int;
  pub fn ronk_field_binop_u64_host(ctx: *mut ronk_ctx, op: c_int, p: u64, a: *const u64, b: *const u64, out: *mut u64, n: usize) -> c_int;
  pub fn ronk_field_unop_u64_host(ctx: *mut ronk_ctx, op: c_int, p: u64, a: *const u64, out: *mut u64, n: usize) -> c_int;
  pub fn ronk_field_pow_u64_host(ctx: *mut ronk_ctx, p: u64, a: *const u64, e: u64, out: *mut u64, n: usize) -> c_int;
  pub fn ronk_field_powers_u64(ctx: *mut ronk_ctx, p: u64, base: u64, scale: u64, out: *mut u64, n: usize) -> c_int;

  // Polynomial::fft / ifft / dft (src/polynomial/mod.rs:240-323, :430-484)
  pub fn ronk_ntt_u64(ctx: *mut ronk_ctx, p: u64, g: u64, data: *mut u64, log_n: u32, batch: u32, inverse: c_int) -> c_int;
  pub fn ronk_ntt_u64_host(ctx: *mut ronk_ctx, p: u64, g: u64, data: *mut u64, log_n: u32, batch: u32, inverse: c_int) -> c_int;
  pub fn ronk_ntt_u64_host_submit(ctx: *mut ronk_ctx, p: u64, g: u64, data: *mut u64, log_n: u32, batch: u32, inverse: c_int, slot: c_int) -> c_int;
  pub fn ronk_ntt_u64_host_wait(ctx: *mut ronk_ctx, slot: c_int) -> c_int;
  pub fn ronk_ntt_mul_u64(ctx: *mut ronk_ctx, p: u64, g: u64, data: *mut u64, mul: *const u64, log_n: u32, batch: u32) -> c_int;
  pub fn ronk_ntt_strided_small_u64(ctx: *mut ronk_ctx, p: u64, g: u64, data: *mut u64, log_g: u32, stride: usize, count: usize, inverse: c_int) -> c_int;
  pub fn ronk_ntt_cross_rank_fused_u64(ctx: *mut ronk_ctx, p: u64, g: u64, peer_bufs: *const *const u64, log_g: u32, rank: u32, log_n: u32, out: *mut u64) -> c_int;
  pub fn ronk_ipc_export(ctx: *mut ronk_ctx, dptr: *const c_void, handle: *mut u8) -> c_int;
  pub fn ronk_ipc_open(ctx: *mut ronk_ctx, handle: *const u8, dptr: *mut *mut c_void) -> c_int;
  pub fn ronk_ipc_close(ctx: *mut ronk_ctx, dptr: *mut c_void) -> c_int;
  pub fn ronk_memcpy_d2d(ctx: *mut ronk_ctx, dst: *mut c_void, src: *const c_void, bytes: usize) -> c_int;
  pub fn ronk_dft_u64(ctx: *mut ronk_ctx, p: u64, g: u64, input: *const u64, n: u64, out: *mut u64) -> c_int;
  pub fn ronk_dft_u64_host(ctx: *mut ronk_ctx, p: u64, g: u64, input: *const u64, n: u64, out: *mut u64) -> c_int;
  pub fn ronk_ntt_any_u64(ctx: *mut ronk_ctx, p: u64, g: u64, data: *mut u64, n: u64, batch: u32, inverse: c_int) -> c_int;
  pub fn ronk_ntt_any_u64_host(ctx: *mut ronk_ctx, p: u64, g: u64, host_data: *mut u64, n: u64, batch: u32, inverse: c_int) -> c_int;
  pub fn ronk_ntt_coset_u64(ctx: *mut ronk_ctx, p: u64, g: u64, data: *mut u64, log_n: u32, batch: u32, shift: u64, inverse: c_int) -> c_int;
  pub fn ronk_ntt_coset_u64_host(ctx: *mut ronk_ctx, p: u64, g: u64, host_data: *mut u64, log_n: u32, batch: u32, shift: u64, inverse: c_int) -> c_int;
  pub fn ronk_poly_lde_u64(ctx: *mut ronk_ctx, p: u64, g: u64, coeffs: *const u64, d: usize, log_n: u32, shift: u64, batch: u32, out: *mut u64) -> c_int;
  pub fn ronk_poly_lde_u64_host(ctx: *mut ronk_ctx, p: u64, g: u64, coeffs: *const u64, d: usize, log_n: u32, shift: u64, batch: u32, out: *mut u64) -> c_int;

  // Polynomial arithmetic (src/polynomial/arithmetic.rs, mod.rs:133-225, :382-415)
  pub fn ronk_poly_mul_u64(ctx: *mut ronk_ctx, p: u64, g: u64, a: *const u64, da: usize, b: *const u64, db: usize, c: *mut u64) -> c_int;
  pub fn ronk_poly_mul_u64_host(ctx: *mut ronk_ctx, p: u64, g: u64, a: *const u64, da: usize, b: *const u64, db: usize, c: *mut u64) -> c_int;
  pub fn ronk_poly_mul_batch_u64(ctx: *mut ronk_ctx, p: u64, g: u64, a: *const u64, da: usize, b: *const u64, db: usize, b_shared: c_int, batch: u32, c: *mut u64) -> c_int;
  pub fn ronk_poly_mul_batch_u64_host(ctx: *mut ronk_ctx, p: u64, g: u64, a: *const u64, da: usize, b: *const u64, db: usize, b_shared: c_int, batch: u32, c: *mut u64) -> c_int;
  pub fn ronk_poly_add_u64(ctx: *mut ronk_ctx, p: u64, a: *const u64, da: usize, b: *const u64, db: usize, out: *mut u64) -> c_int;
  pub fn ronk_poly_sub_u64(ctx: *mut ronk_ctx, p: u64, a: *const u64, da: usize, b: *const u64, db: usize, out: *mut u64) -> c_int;
  pub fn ronk_poly_eval_u64(ctx: *mut ronk_ctx, p: u64, coeffs: *const u64, d: usize, xs: *const u64, m: usize, out: *mut u64) -> c_int;
  pub fn ronk_poly_eval_u64_host(ctx: *mut ronk_ctx, p: u64, coeffs: *const u64, d: usize, xs: *const u64, m: usize, out: *mut u64) -> c_int;
  pub fn ronk_poly_lagrange_eval_u64_host(ctx: *mut ronk_ctx, p: u64, g: u64, coeffs: *const u64, n: usize, x: u64, out: *mut u64) -> c_int;
  /// Lagrange-basis rows (batch × n) on the coset shift·H_n at m points, barycentric, O(n) per point; device pointers.
  pub fn ronk_poly_lagrange_eval_u64(ctx: *mut ronk_ctx, p: u64, g: u64, evals: *const u64, n: u64, batch: u32, shift: u64, xs: *const u64, m: usize, out: *mut u64) -> c_int;
  pub fn ronk_poly_lagrange_eval_batch_u64_host(ctx: *mut ronk_ctx, p: u64, g: u64, evals: *const u64, n: u64, batch: u32, shift: u64, xs: *const u64, m: usize, out: *mut u64) -> c_int;
  /// `kzg::open` in evaluation form (src/kzg/setup.rs:63-78): f_b(z) and the quotient's evaluations on the nodes.
  pub fn ronk_poly_lagrange_open_u64(ctx: *mut ronk_ctx, p: u64, g: u64, evals: *const u64, n: u64, batch: u32, shift: u64, z: u64, values: *mut u64, quotient: *mut u64) -> c_int;
  pub fn ronk_poly_lagrange_open_u64_host(ctx: *mut ronk_ctx, p: u64, g: u64, evals: *const u64, n: u64, batch: u32, shift: u64, z: u64, values: *mut u64, quotient: *mut u64) -> c_int;
  pub fn ronk_poly_divrem_u64_host(ctx: *mut ronk_ctx, p: u64, a: *const u64, da: usize, b: *const u64, db: usize, q: *mut u64, r: *mut u64) -> c_int;
  /// `quotient_and_remainder` on device pointers; Newton iteration on the transforms when the divisor's top word is nonzero.
  pub fn ronk_poly_divrem_u64(ctx: *mut ronk_ctx, p: u64, g: u64, a: *const u64, da: usize, b: *const u64, db: usize, q: *mut u64, r: *mut u64) -> c_int;
  pub fn ronk_poly_divrem_batch_u64(ctx: *mut ronk_ctx, p: u64, g: u64, a: *const u64, da: usize, b: *const u64, db: usize, b_shared: c_int, batch: u32, q: *mut u64, r: *mut u64) -> c_int;
  pub fn ronk_poly_divrem_batch_u64_host(ctx: *mut ronk_ctx, p: u64, g: u64, a: *const u64, da: usize, b: *const u64, db: usize, b_shared: c_int, batch: u32, q: *mut u64, r: *mut u64) -> c_int;
  /// Lagrange interpolation = `Message::decode` on the first K coordinates (src/codes/reed_solomon.rs:55-107); host pointers.
  pub fn ronk_poly_interpolate_u64_host(ctx: *mut ronk_ctx, p: u64, xs: *const u64, ys: *const u64, k: usize, out: *mut u64) -> c_int;
  /// Π (X - xs[i]) on device pointers, k + 1 coefficients; a subproduct tree on the transforms above the crossover.
  pub fn ronk_poly_from_roots_u64(ctx: *mut ronk_ctx, p: u64, g: u64, xs: *const u64, k: usize, out: *mut u64) -> c_int;
  /// `evaluate` at m points on device pointers (src/shamir/mod.rs:53-58); the same words as `ronk_poly_eval_u64`.
  pub fn ronk_poly_multieval_u64(ctx: *mut ronk_ctx, p: u64, g: u64, coeffs: *const u64, d: usize, xs: *const u64, m: usize, out: *mut u64) -> c_int;
  /// Device twin of `ronk_poly_interpolate_u64_host`; synchronous.
  pub fn ronk_poly_interpolate_u64(ctx: *mut ronk_ctx, p: u64, g: u64, xs: *const u64, ys: *const u64, k: usize, out: *mut u64) -> c_int;
  /// `evaluate` of `batch` rows (batch × d) at the same m points (Shamir split of many secrets), one shared tree; device
  /// pointers, out batch × m; asynchronous.  Every row is the words of `ronk_poly_multieval_u64`.
  pub fn ronk_poly_multieval_batch_u64(ctx: *mut ronk_ctx, p: u64, g: u64, coeffs: *const u64, d: usize, batch: u32, xs: *const u64, m: usize, out: *mut u64) -> c_int;
  pub fn ronk_poly_multieval_batch_u64_host(ctx: *mut ronk_ctx, p: u64, g: u64, coeffs: *const u64, d: usize, batch: u32, xs: *const u64, m: usize, out: *mut u64) -> c_int;
  /// Interpolation of `batch` rows of ys (batch × k) through the same k nodes, one shared tree; device pointers, out
  /// batch × k; synchronous.  Every row is the words of `ronk_poly_interpolate_u64`.
  pub fn ronk_poly_interpolate_batch_u64(ctx: *mut ronk_ctx, p: u64, g: u64, xs: *const u64, ys: *const u64, k: usize, batch: u32, out: *mut u64) -> c_int;
  pub fn ronk_poly_interpolate_batch_u64_host(ctx: *mut ronk_ctx, p: u64, g: u64, xs: *const u64, ys: *const u64, k: usize, batch: u32, out: *mut u64) -> c_int;
  /// Division by b0 + b1·x (the divisor `kzg::open` builds, src/kzg/setup.rs:72-75) as a device-wide scan; device pointers.
  pub fn ronk_poly_div_linear_u64(ctx: *mut ronk_ctx, p: u64, a: *const u64, d: usize, b0: u64, b1: u64, q: *mut u64, rem: *mut u64) -> c_int;

  // Reed–Solomon codes (src/codes/reed_solomon.rs:42-52): encoding, and errors-and-erasures decoding up to
  // n - k ≤ RONK_RS_MAX_PARITY; status[b] = errors corrected, or -1 for a row outside the decoding radius.
  pub fn ronk_rs_encode_u64(ctx: *mut ronk_ctx, p: u64, g: u64, msg: *const u64, k: u64, n: u64, batch: u32, codeword: *mut u64) -> c_int;
  pub fn ronk_rs_decode_u64(ctx: *mut ronk_ctx, p: u64, g: u64, received: *const u64, erased: *const u8, n: u64, k: u64, batch: u32, msg: *mut u64, status: *mut i32) -> c_int;
  pub fn ronk_rs_decode_u64_host(ctx: *mut ronk_ctx, p: u64, g: u64, received: *const u64, erased: *const u8, n: u64, k: u64, batch: u32, msg: *mut u64, status: *mut i32) -> c_int;
  pub fn ronk_rs_decode_at_u64(ctx: *mut ronk_ctx, p: u64, g: u64, xs: *const u64, received: *const u64, erased: *const u8, n: u64, k: u64, batch: u32, msg: *mut u64, status: *mut i32) -> c_int;
  pub fn ronk_rs_decode_at_u64_host(ctx: *mut ronk_ctx, p: u64, g: u64, xs: *const u64, received: *const u64, erased: *const u8, n: u64, k: u64, batch: u32, msg: *mut u64, status: *mut i32) -> c_int;

  // AffinePoint<PlutoExtendedCurve> + kzg::commit (src/curve/mod.rs:157-235, src/kzg/setup.rs:48-60)
  pub fn ronk_point_add_pluto_ext_host(ctx: *mut ronk_ctx, a: *const u8, b: *const u8, out: *mut u8, n: usize) -> c_int;
  pub fn ronk_point_neg_pluto_ext_host(ctx: *mut ronk_ctx, a: *const u8, out: *mut u8, n: usize) -> c_int;
  pub fn ronk_point_smul_pluto_ext_host(ctx: *mut ronk_ctx, a: *const u8, scalars: *const u8, out: *mut u8, n: usize) -> c_int;
  pub fn ronk_msm_pluto_ext(ctx: *mut ronk_ctx, points: *const u8, n_points: usize, scalars: *const u8, n_scalars: usize, out: *mut u8) -> c_int;
  pub fn ronk_msm_pluto_ext_host(ctx: *mut ronk_ctx, points: *const u8, n_points: usize, scalars: *const u8, n_scalars: usize, out: *mut u8) -> c_int;
  /// `kzg::commit` of `batch` contiguous scalar rows against one SRS; device pointers, out is batch × 4 bytes on the device.
  pub fn ronk_msm_pluto_ext_batch(ctx: *mut ronk_ctx, points: *const u8, n_points: usize, scalars: *const u8, n_scalars: usize, batch: u32, out: *mut u8) -> c_int;
  pub fn ronk_msm_pluto_ext_batch_host(ctx: *mut ronk_ctx, points: *const u8, n_points: usize, scalars: *const u8, n_scalars: usize, batch: u32, out: *mut u8) -> c_int;
  /// The reference's Tate pairing on n pairs of E[17]; out[2i], out[2i+1] = c0, c1.  Device pointers.
  pub fn ronk_pairing_pluto_ext(ctx: *mut ronk_ctx, p: *const u8, q: *const u8, n: usize, out: *mut u8) -> c_int;
  pub fn ronk_pairing_pluto_ext_host(ctx: *mut ronk_ctx, p: *const u8, q: *const u8, n: usize, out: *mut u8) -> c_int;
  /// `kzg::check` of n openings against one SRS: ok[r] = 1 when the row verifies, else 0.  Device pointers.
  pub fn ronk_kzg_check_pluto_ext_batch(ctx: *mut ronk_ctx, commitments: *const u8, proofs: *const u8, points: *const u8, values: *const u8, n: usize, g1_srs: *const u8, n_g1: usize, g2_srs: *const u8, n_g2: usize, ok: *mut u8) -> c_int;
  pub fn ronk_kzg_check_pluto_ext_batch_host(ctx: *mut ronk_ctx, commitments: *const u8, proofs: *const u8, points: *const u8, values: *const u8, n: usize, g1_srs: *const u8, n_g1: usize, g2_srs: *const u8, n_g2: usize, ok: *mut u8) -> c_int;
  /// The reference's Poseidon permutation on `batch` states of `width` words, in place.  Device pointers.
  pub fn ronk_poseidon_permute_u64(ctx: *mut ronk_ctx, p: u64, width: u32, alpha: u64, num_f: u32, num_p: u32, rc: *const u64, mds: *const u64, states: *mut u64, batch: usize) -> c_int;
  pub fn ronk_poseidon_permute_u64_host(ctx: *mut ronk_ctx, p: u64, width: u32, alpha: u64, num_f: u32, num_p: u32, rc: *const u64, mds: *const u64, states: *mut u64, batch: usize) -> c_int;
  /// One fresh Poseidon sponge per row: absorb `len` words, squeeze `n_out` words.  Device pointers.
  pub fn ronk_poseidon_sponge_u64(ctx: *mut ronk_ctx, p: u64, width: u32, alpha: u64, num_f: u32, num_p: u32, rc: *const u64, mds: *const u64, rate: u32, input: *const u64, len: usize, batch: usize, out: *mut u64, n_out: usize) -> c_int;
  pub fn ronk_poseidon_sponge_u64_host(ctx: *mut ronk_ctx, p: u64, width: u32, alpha: u64, num_f: u32, num_p: u32, rc: *const u64, mds: *const u64, rate: u32, input: *const u64, len: usize, batch: usize, out: *mut u64, n_out: usize) -> c_int;
  /// SHA-256 of n messages data[offsets[i], offsets[i+1]): out[32·i ..].  Device pointers.
  pub fn ronk_sha256(ctx: *mut ronk_ctx, data: *const u8, data_len: u64, offsets: *const u64, n: usize, out: *mut u8) -> c_int;
  pub fn ronk_sha256_host(ctx: *mut ronk_ctx, data: *const u8, data_len: u64, offsets: *const u64, n: usize, out: *mut u8) -> c_int;
  /// Every level of the SHA-256 Merkle tree of n messages, leaf level first.  Device pointers.
  pub fn ronk_merkle_build_sha256(ctx: *mut ronk_ctx, data: *const u8, data_len: u64, offsets: *const u64, n: usize, nodes: *mut u8) -> c_int;
  pub fn ronk_merkle_build_sha256_host(ctx: *mut ronk_ctx, data: *const u8, data_len: u64, offsets: *const u64, n: usize, nodes: *mut u8) -> c_int;
  /// `get_proof` of m leaf indices: L siblings and sides (0 = Left, 1 = Right) each.  Device pointers.
  pub fn ronk_merkle_proofs_sha256(ctx: *mut ronk_ctx, nodes: *const u8, n: usize, indices: *const u64, m: usize, siblings: *mut u8, sides: *mut u8) -> c_int;
  pub fn ronk_merkle_proofs_sha256_host(ctx: *mut ronk_ctx, nodes: *const u8, n: usize, indices: *const u64, m: usize, siblings: *mut u8, sides: *mut u8) -> c_int;
  /// `prove` of m messages with depth-step proofs against one root: ok[j] = 1 or 0.  Device pointers.
  pub fn ronk_merkle_verify_sha256(ctx: *mut ronk_ctx, root: *const u8, data: *const u8, data_len: u64, offsets: *const u64, m: usize, siblings: *const u8, sides: *const u8, depth: u32, ok: *mut u8) -> c_int;
  pub fn ronk_merkle_verify_sha256_host(ctx: *mut ronk_ctx, root: *const u8, data: *const u8, data_len: u64, offsets: *const u64, m: usize, siblings: *const u8, sides: *const u8, depth: u32, ok: *mut u8) -> c_int;
  pub fn ronk_msm_pluto_ext_buckets(ctx: *mut ronk_ctx, points: *const u8, n_points: usize, scalars: *const u8, n_scalars: usize, buckets: *mut u8) -> c_int;
  pub fn ronk_msm_combine_buckets_host(ctx: *mut ronk_ctx, buckets: *const u8, n_sets: usize, out: *mut u8) -> c_int;

  pub fn ronk_splitmix_fill_u64(ctx: *mut ronk_ctx, p: u64, seed: u64, out: *mut u64, n: usize) -> c_int;

  // multi-GPU modes (one context per GPU; NCCL inside the library).  `id` is RONK_NCCL_UNIQUE_ID_BYTES = 128 bytes:
  // made on rank 0, carried to the other ranks by the host (e.g. MPI_Bcast), then every rank calls ronk_dist_init.
  pub fn ronk_dist_unique_id(id: *mut u8) -> c_int;
  pub fn ronk_dist_init(ctx: *mut ronk_ctx, id: *const u8, rank: c_int, world: c_int) -> c_int;
  pub fn ronk_dist_init_comm(ctx: *mut ronk_ctx, nccl_comm: *mut c_void, rank: c_int, world: c_int) -> c_int;
  pub fn ronk_dist_finalize(ctx: *mut ronk_ctx) -> c_int;
  pub fn ronk_dist_rank(ctx: *mut ronk_ctx, rank: *mut c_int, world: *mut c_int) -> c_int;
  pub fn ronk_dist_barrier(ctx: *mut ronk_ctx) -> c_int;
  pub fn ronk_dist_shard_range(total: u64, rank: c_int, world: c_int, lo: *mut u64, hi: *mut u64) -> c_int;
  pub fn ronk_ntt_u64_batch_sharded(ctx: *mut ronk_ctx, p: u64, g: u64, shard: *mut u64, log_n: u32, total_batch: u64, inverse: c_int, lo: *mut u64, hi: *mut u64) -> c_int;
  pub fn ronk_ntt_u64_dist(ctx: *mut ronk_ctx, p: u64, g: u64, local: *mut u64, log_n: u32, batch: u32, flavour: c_int) -> c_int;
  pub fn ronk_ntt_u64_dist_virtual(ctx: *mut ronk_ctx, p: u64, g: u64, data: *mut u64, log_n: u32, batch: u32, log_g: u32, flavour: c_int) -> c_int;
  pub fn ronk_msm_pluto_ext_dist(ctx: *mut ronk_ctx, points: *const u8, n_points: usize, scalars: *const u8, n_scalars: usize, out: *mut u8) -> c_int;
}

pub const RONK_NCCL_UNIQUE_ID_BYTES: usize = 128;
pub const RONK_DIST_NCCL: c_int = 0;
pub const RONK_DIST_FUSED: c_int = 1;
