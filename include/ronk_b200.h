/*
 * ronk_b200.h — C ABI of libronk_b200.so: the H100-native (sm_90a) replacement for
 * pluto/ronkathon's PrimeField / Polynomial / kzg::commit hot path.
 *
 * The reference is a pure-Rust crate with no FFI of its own; this header is the boundary a
 * `ronkathon-b200-sys` crate would bind 1:1 (see INTEGRATION.md, bindings/rust/).  Each entry
 * point cites the reference item it replaces (file:line relative to the ronkathon tree).
 *
 * Conventions
 *  - Field elements are canonical residues in uint64_t (the reference's `PrimeField<P>{value: usize}`,
 *    src/algebra/field/prime/mod.rs:39-42).  Inputs must be canonical (< p); outputs always are.
 *  - `p` is the modulus, `g` the multiplicative generator (FiniteField::PRIMITIVE_ELEMENT).
 *    p = 0xFFFFFFFF00000001 (Goldilocks) takes the specialised kernels; any other odd prime
 *    < 2^64 takes the generic Montgomery kernels (same code path the p = 101 / 17 / 127
 *    cross-checks run through).  p = 2 is not supported (RONK_EUNSUPPORTED).
 *  - Pointers without a `_host` suffix in the function name are DEVICE pointers on the context's
 *    device; work is enqueued on the context's stream and is asynchronous unless stated.
 *    `_host` variants take host pointers, copy in, run, copy out and synchronise.
 *  - Every function returns 0 (RONK_OK) or an error code; nothing throws, aborts or falls back
 *    to a CPU path.  Where the reference would panic/assert, RONK_EINVAL is returned.
 *  - Curve points (AffinePoint<PlutoExtendedCurve>, src/curve/mod.rs:67-74) are 4 bytes
 *    x0,x1,y0,y1 with x = x0 + x1·t in GF(101²) = F101[t]/(t²+2); 0xFF,0xFF,0xFF,0xFF = Infinity.
 *    Scalars (PlutoScalarField = F17) are one byte each, < 17.
 *  - The caller owns every buffer; the library never retains caller pointers past stream order.
 */
#ifndef RONK_B200_H
#define RONK_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RONK_OK 0
#define RONK_EINVAL 1       /* the reference would panic/assert on this input */
#define RONK_ECUDA 2        /* CUDA runtime error (see ronk_last_error) */
#define RONK_ENOMEM 3       /* device allocation failed */
#define RONK_ENCCL 4        /* collective error */
#define RONK_EUNSUPPORTED 5 /* outside the supported envelope (e.g. log_n too large) */

#define RONK_GOLDILOCKS 0xFFFFFFFF00000001ULL

typedef struct ronk_ctx ronk_ctx;

/* ---- context ---------------------------------------------------------------------------- */
/* Opaque context: device, stream, twiddle/plan cache, workspace.  `stream` is a cudaStream_t
 * (NULL = the legacy default stream).  One context per host thread. */
int ronk_ctx_create(ronk_ctx **out, int device, void *stream);
int ronk_ctx_destroy(ronk_ctx *ctx);
int ronk_ctx_set_stream(ronk_ctx *ctx, void *stream);
int ronk_sync(ronk_ctx *ctx);
const char *ronk_strerror(int code);
const char *ronk_last_error(ronk_ctx *ctx);
/* Number of kernels this context has launched (bench.py's `gpu_launches`). */
uint64_t ronk_launch_count(ronk_ctx *ctx);
/* Kernel profiling: when on, every kernel launch is bracketed by CUDA events on the context's
 * stream.  ronk_prof_fetch synchronises, writes up to `max` (name, ms) records in launch order,
 * returns the number written and clears the log. */
int ronk_prof_enable(ronk_ctx *ctx, int on);
int ronk_prof_fetch(ronk_ctx *ctx, char (*names)[32], float *ms, int max);
/* Device memory helpers so a host-language binding needs no CUDA runtime of its own. */
int ronk_dev_alloc(ronk_ctx *ctx, void **dptr, size_t bytes);
int ronk_dev_free(ronk_ctx *ctx, void *dptr);
int ronk_memcpy_h2d(ronk_ctx *ctx, void *dst_dev, const void *src_host, size_t bytes);
int ronk_memcpy_d2h(ronk_ctx *ctx, void *dst_host, const void *src_dev, size_t bytes);

/* ---- FiniteField metadata (host side, O(log p)) ----------------------------------------- */
/* FiniteField::PRIMITIVE_ELEMENT — src/algebra/field/prime/mod.rs:87-123.  Known moduli only:
 * 101→2, 17→14, 127→3, 59→2 (the reference's own search results), Goldilocks→7 (SURVEY §8a D4). */
int ronk_field_generator(uint64_t p, uint64_t *g);
/* FiniteField::primitive_root_of_unity(n) — src/algebra/field/mod.rs:70-75.
 * RONK_EINVAL when n does not divide p-1 (the reference's assert). */
int ronk_root_of_unity(uint64_t p, uint64_t g, uint64_t n, uint64_t *out);

/* ---- PrimeField<P> element-wise arithmetic on arrays ------------------------------------ */
/* Add/Sub/Mul/Neg — src/algebra/field/prime/arithmetic.rs:6,22-27,37,64. out may alias a or b. */
int ronk_field_add_u64(ronk_ctx *ctx, uint64_t p, const uint64_t *a, const uint64_t *b, uint64_t *out, size_t n);
int ronk_field_sub_u64(ronk_ctx *ctx, uint64_t p, const uint64_t *a, const uint64_t *b, uint64_t *out, size_t n);
int ronk_field_mul_u64(ronk_ctx *ctx, uint64_t p, const uint64_t *a, const uint64_t *b, uint64_t *out, size_t n);
int ronk_field_neg_u64(ronk_ctx *ctx, uint64_t p, const uint64_t *a, uint64_t *out, size_t n);
/* Field::pow(self, power) — src/algebra/field/prime/mod.rs:74-84 (same value, O(log e)). */
int ronk_field_pow_u64(ronk_ctx *ctx, uint64_t p, const uint64_t *a, uint64_t e, uint64_t *out, size_t n);
/* Field::inverse — src/algebra/field/prime/mod.rs:62-72 (a^(p-2)).  Synchronous: returns
 * RONK_EINVAL if any input is 0 (the reference's None / unwrap panic); outputs for zeros are 0. */
int ronk_field_inv_u64(ronk_ctx *ctx, uint64_t p, const uint64_t *a, uint64_t *out, size_t n);
/* Div — src/algebra/field/prime/arithmetic.rs:54 (a * b^-1).  Synchronous; RONK_EINVAL on b=0. */
int ronk_field_div_u64(ronk_ctx *ctx, uint64_t p, const uint64_t *a, const uint64_t *b, uint64_t *out, size_t n);
/* Host-pointer variants (op: 0 add, 1 sub, 2 mul, 3 div; unary: 0 neg, 1 inverse). */
int ronk_field_binop_u64_host(ronk_ctx *ctx, int op, uint64_t p, const uint64_t *a, const uint64_t *b, uint64_t *out, size_t n);
int ronk_field_unop_u64_host(ronk_ctx *ctx, int op, uint64_t p, const uint64_t *a, uint64_t *out, size_t n);
int ronk_field_pow_u64_host(ronk_ctx *ctx, uint64_t p, const uint64_t *a, uint64_t e, uint64_t *out, size_t n);

/* ---- transforms -------------------------------------------------------------------------- */
/* Polynomial::fft / ifft — src/polynomial/mod.rs:273-323 / :430-484.  In place, `batch`
 * contiguous transforms of 2^log_n points, NATURAL order in and out, X[k] = Σ_j a_j ω^(jk),
 * ω = g^((p-1)/2^log_n); inverse uses ω^-1 and scales by (2^log_n)^-1.
 * RONK_EINVAL if 2^log_n does not divide p-1; RONK_EUNSUPPORTED if log_n > 26. */
int ronk_ntt_u64(ronk_ctx *ctx, uint64_t p, uint64_t g, uint64_t *data, uint32_t log_n, uint32_t batch, int inverse);
int ronk_ntt_u64_host(ronk_ctx *ctx, uint64_t p, uint64_t g, uint64_t *host_data, uint32_t log_n, uint32_t batch, int inverse);
/* Pipelined host-buffer transforms: `submit` enqueues H2D → transform → D2H for `host_data`
 * (pinned memory recommended) on slot 0, 1 or 2 and returns at once; `wait` blocks until that
 * slot's result is back in host memory.  With the slots in flight the PCIe upload of one step, the
 * kernels of the previous and the download of the one before overlap (PCIe is full duplex).
 * ronk_ntt_u64_host(…) == submit(slot 0) + wait(0). */
int ronk_ntt_u64_host_submit(ronk_ctx *ctx, uint64_t p, uint64_t g, uint64_t *host_data, uint32_t log_n, uint32_t batch, int inverse, int slot);
int ronk_ntt_u64_host_wait(ronk_ctx *ctx, int slot);
/* Forward transform whose last stage also multiplies point-wise by `mul` (same shape, natural
 * order): data[k] = NTT(data)[k] * mul[k].  The fused form of the evaluate→multiply step. */
int ronk_ntt_mul_u64(ronk_ctx *ctx, uint64_t p, uint64_t g, uint64_t *data, const uint64_t *mul, uint32_t log_n, uint32_t batch);
/* Polynomial::dft — src/polynomial/mod.rs:240-258.  Any n | p-1 (O(n²)); out must not alias in. */
int ronk_dft_u64(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *in, uint64_t n, uint64_t *out);
int ronk_dft_u64_host(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *in, uint64_t n, uint64_t *out);

/* Distributed-transform building blocks (SURVEY §8e: the top log2(G) stages of one large NTT across
 * G GPUs).  out[i] = scale * base^i — the twiddle column ω_n^(r·k') a rank multiplies into its
 * local transform before the exchange. */
int ronk_field_powers_u64(ronk_ctx *ctx, uint64_t p, uint64_t base, uint64_t scale, uint64_t *out, size_t n);
/* In-place 2^log_g-point transforms (log_g ≤ 4) over the strided sets {data[k + j*stride]}, j < 2^log_g,
 * for k < count: the cross-rank radix-G butterflies after the all-to-all.  Same ω convention as
 * ronk_ntt_u64 (ω_G = g^((p-1)/G)); inverse applies G^-1. */
int ronk_ntt_strided_small_u64(ronk_ctx *ctx, uint64_t p, uint64_t g, uint64_t *data, uint32_t log_g, size_t stride, size_t count, int inverse);

/* Peer-memory fused form of the same stage: ONE kernel per rank that loads the peers' local
 * transforms directly over NVLink (P2P loads through CUDA-IPC-mapped pointers), applies the twiddle
 * column ω_n^(r'·k') on the fly and runs the G-point cross-rank butterflies — twiddle multiply,
 * all-to-all and butterflies in a single launch, no staging buffer.  `peer_bufs[r']` (host array of
 * G device pointers, entry `rank` being this rank's own buffer) each hold that rank's n/G-point
 * local transform Y_r'; `out` (n/G words) receives X[(rank·m/G + k'') + m·q] at q·(m/G) + k''.
 * Callers must make sure every rank's Y is complete before the launch (host barrier). */
int ronk_ntt_cross_rank_fused_u64(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *const *peer_bufs, uint32_t log_g, uint32_t rank, uint32_t log_n, uint64_t *out);
/* CUDA-IPC plumbing for the above: export a handle for a buffer obtained from ronk_dev_alloc, open a
 * peer's handle (enables peer access), close it again; and a device-to-device copy. */
int ronk_ipc_export(ronk_ctx *ctx, const void *dptr, uint8_t handle[64]);
int ronk_ipc_open(ronk_ctx *ctx, const uint8_t handle[64], void **dptr);
int ronk_ipc_close(ronk_ctx *ctx, void *dptr);
int ronk_memcpy_d2d(ronk_ctx *ctx, void *dst_dev, const void *src_dev, size_t bytes);

/* ---- multi-GPU modes (SURVEY §8b / §8e) ---------------------------------------------------------
 * The reference is single-threaded and has no distributed layer; these are the modes BASELINE.json's
 * north_star adds around its hot path: independent batches sharded with no collective, the top log2(G)
 * stages of a transform across G GPUs with ONE exchange, and kzg::commit (src/kzg/setup.rs:48-60) over
 * index-range shards.  One context per GPU (one process or host thread each); NCCL (libnccl.so.2,
 * resolved with dlopen at the first call — RONK_ENCCL when absent) carries the collectives on the
 * context's stream.  G = world must be a power of two ≤ 16. */
#define RONK_NCCL_UNIQUE_ID_BYTES 128
#define RONK_DIST_NCCL 0  /* exchange = grouped ncclSend/ncclRecv (all-to-all) */
#define RONK_DIST_FUSED 1 /* exchange fused into the butterfly kernel: P2P loads from CUDA-IPC peer buffers */
/* Bootstrap.  Rank 0 makes an id and the host carries its 128 bytes to every rank (MPI_Bcast, a TCP
 * store, torch.distributed …); every rank then calls ronk_dist_init (collective).  Alternatively adopt
 * an ncclComm_t the host already owns (not destroyed by ronk_dist_finalize). */
int ronk_dist_unique_id(uint8_t id[RONK_NCCL_UNIQUE_ID_BYTES]);
int ronk_dist_init(ronk_ctx *ctx, const uint8_t id[RONK_NCCL_UNIQUE_ID_BYTES], int rank, int world);
int ronk_dist_init_comm(ronk_ctx *ctx, void *nccl_comm, int rank, int world);
int ronk_dist_finalize(ronk_ctx *ctx);
int ronk_dist_rank(ronk_ctx *ctx, int *rank, int *world);
/* Stream-ordered barrier over the communicator (a 4-byte all-reduce): the host does not wait. */
int ronk_dist_barrier(ronk_ctx *ctx);
/* Contiguous range [lo, hi) of `total` units owned by `rank` (remainder spread over the first ranks). */
int ronk_dist_shard_range(uint64_t total, int rank, int world, uint64_t *lo, uint64_t *hi);
/* Polynomial::fft / ifft (src/polynomial/mod.rs:273-323, :430-484) of a batch sharded by contiguous
 * ranges: this rank transforms its (hi - lo) × 2^log_n words at `shard` in place.  No collective. */
int ronk_ntt_u64_batch_sharded(ronk_ctx *ctx, uint64_t p, uint64_t g, uint64_t *shard, uint32_t log_n, uint64_t total_batch, int inverse, uint64_t *lo, uint64_t *hi);
/* Forward transforms of `batch` polynomials of 2^log_n coefficients, each spread CYCLICALLY over the
 * ranks: `local` holds [batch][n/G] with local[b][j] = a_b[rank + G·j].  In place; on return
 * local[b][q][k] = X_b[rank·(n/G²) + k + (n/G)·q], q < G, k < n/G² (block-cyclic).  Collective. */
int ronk_ntt_u64_dist(ronk_ctx *ctx, uint64_t p, uint64_t g, uint64_t *local, uint32_t log_n, uint32_t batch, int flavour);
/* The same decomposition with G = 2^log_g (2 … 16) VIRTUAL ranks on ONE device, no communicator: `data` holds the G
 * local slices rank-major ([rank][batch][n/G], slice r = a_b[r + G·j]) and receives the G local results in the
 * layout above.  Every kernel of the chosen flavour runs as in the collective call; only the wire (all-to-all / peer
 * buffers) is device-local.  Validation of G = 4, 8, 16 on a single GPU; not collective. */
int ronk_ntt_u64_dist_virtual(ronk_ctx *ctx, uint64_t p, uint64_t g, uint64_t *data, uint32_t log_n, uint32_t batch, uint32_t log_g, int flavour);
/* kzg::commit over index-range shards: this rank's terms in, the full commitment out on every rank
 * (RONK_EINVAL on every rank if any shard holds an invalid term).  Collective, synchronous. */
int ronk_msm_pluto_ext_dist(ronk_ctx *ctx, const uint8_t *points, size_t n_points, const uint8_t *scalars, size_t n_scalars, uint8_t out[4]);

/* ---- Polynomial<Monomial, F, D> ----------------------------------------------------------- */
/* Mul — src/polynomial/arithmetic.rs:97-119.  c has da+db-1 coefficients (no trimming).
 * NTT path (pad → NTT, NTT∘pointwise → iNTT) when a power of two ≥ da+db-1 divides p-1 and
 * the product is large enough to pay for it, else the schoolbook kernel (e.g. p = 101). */
int ronk_poly_mul_u64(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *a, size_t da, const uint64_t *b, size_t db, uint64_t *c);
int ronk_poly_mul_u64_host(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *a, size_t da, const uint64_t *b, size_t db, uint64_t *c);
/* Add/Sub/Neg — src/polynomial/arithmetic.rs:16-94: out has da terms, b zero-extended/truncated. */
int ronk_poly_add_u64(ronk_ctx *ctx, uint64_t p, const uint64_t *a, size_t da, const uint64_t *b, size_t db, uint64_t *out);
int ronk_poly_sub_u64(ronk_ctx *ctx, uint64_t p, const uint64_t *a, size_t da, const uint64_t *b, size_t db, uint64_t *out);
/* evaluate — src/polynomial/mod.rs:133-139: out[i] = Σ_j coeffs[j] * xs[i]^j for m points. */
int ronk_poly_eval_u64(ronk_ctx *ctx, uint64_t p, const uint64_t *coeffs, size_t d, const uint64_t *xs, size_t m, uint64_t *out);
int ronk_poly_eval_u64_host(ronk_ctx *ctx, uint64_t p, const uint64_t *coeffs, size_t d, const uint64_t *xs, size_t m, uint64_t *out);
/* Lagrange-basis evaluate — src/polynomial/mod.rs:382-415 (nodes ω_n^i, barycentric; returns 0 when x
 * is a node, because l(x) = 0 multiplies the fold).  Host pointers, n | p-1.  RONK_EINVAL when two
 * nodes coincide (ω of order below n: the reference divides by zero). */
int ronk_poly_lagrange_eval_u64_host(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *coeffs, size_t n, uint64_t x, uint64_t *out);
/* quotient_and_remainder / Div / Rem — src/polynomial/mod.rs:170-225, arithmetic.rs:121-146.
 * q and r both have da terms.  Host pointers.  RONK_EINVAL for an all-zero divisor. */
int ronk_poly_divrem_u64_host(ronk_ctx *ctx, uint64_t p, const uint64_t *a, size_t da, const uint64_t *b, size_t db, uint64_t *q, uint64_t *r);
/* Division by a linear factor b0 + b1*x — the divisor kzg::open builds (src/kzg/setup.rs:72-75,
 * [-z, 1]) fed to Polynomial::div (src/polynomial/mod.rs:170-225, arithmetic.rs:121-146) — as a
 * device-wide scan.  Device pointers: a (d terms), q (d terms, q[d-1] = 0 like the reference's
 * zero-padded quotient), rem (1 word = a(-b0/b1)).  q must not alias a.  RONK_EINVAL for b1 == 0.
 * ronk_poly_divrem_u64_host takes this path by itself when db == 2 and b[1] != 0. */
/* Lagrange interpolation through (xs[i], ys[i]), i < k: the monomial coefficients out[0..k).  This is
 * Message::decode of src/codes/reed_solomon.rs:55-107 applied to the first K coordinates of a
 * codeword (the reference enumerates combinations; the interpolant is unique).  Host pointers,
 * k <= 8192.  RONK_EINVAL for a repeated x (the reference's `/` panics on the zero denominator). */
int ronk_poly_interpolate_u64_host(ronk_ctx *ctx, uint64_t p, const uint64_t *xs, const uint64_t *ys, size_t k, uint64_t *out);
int ronk_poly_div_linear_u64(ronk_ctx *ctx, uint64_t p, const uint64_t *a, size_t d, uint64_t b0, uint64_t b1, uint64_t *q, uint64_t *rem);

/* ---- curve + kzg::commit ------------------------------------------------------------------ */
/* AffinePoint Add / Neg / Mul<ScalarField> — src/curve/mod.rs:178-213, :225-235, :157-172,
 * element-wise over n points (host pointers).  RONK_EINVAL for off-curve / malformed input. */
int ronk_point_add_pluto_ext_host(ronk_ctx *ctx, const uint8_t *a, const uint8_t *b, uint8_t *out, size_t n);
int ronk_point_neg_pluto_ext_host(ronk_ctx *ctx, const uint8_t *a, uint8_t *out, size_t n);
int ronk_point_smul_pluto_ext_host(ronk_ctx *ctx, const uint8_t *a, const uint8_t *scalars, uint8_t *out, size_t n);
/* kzg::commit — src/kzg/setup.rs:48-60: Σ points[i]·scalars[i] for i < n_scalars.  The group has
 * 102² points and exponent 102, i.e. E ≅ (Z/102)²: with a basis (G1, G2) found and checked on the host and
 * P_i = a_i·G1 + b_i·G2 the sum is (Σ s_i a_i mod 102)·G1 + (Σ s_i b_i mod 102)·G2 — two integer dot products and one
 * table lookup in ONE launch, the same affine point the reference's chain of additions yields (RONK_MSM_COORD=0
 * selects the point-indexed histogram kernels, RONK_MSM_COORD=0 RONK_MSM_HIST=0 the round-1 Pippenger bucket kernels).  RONK_EINVAL if n_points < n_scalars (the reference's assert), if a scalar ≥ 17
 * or if a point is off-curve.  `points`/`scalars` are device pointers, `out` is a 4-byte HOST
 * buffer; synchronous. */
int ronk_msm_pluto_ext(ronk_ctx *ctx, const uint8_t *points, size_t n_points, const uint8_t *scalars, size_t n_scalars, uint8_t out[4]);
int ronk_msm_pluto_ext_host(ronk_ctx *ctx, const uint8_t *points, size_t n_points, const uint8_t *scalars, size_t n_scalars, uint8_t out[4]);
/* Per-device partial MSM for the multi-GPU path: writes the 17 bucket sums (17×4 bytes, host)
 * so ranks can combine them; ronk_msm_combine_buckets folds world×17 buckets into one point. */
int ronk_msm_pluto_ext_buckets(ronk_ctx *ctx, const uint8_t *points, size_t n_points, const uint8_t *scalars, size_t n_scalars, uint8_t buckets[68]);
int ronk_msm_combine_buckets_host(ronk_ctx *ctx, const uint8_t *buckets, size_t n_sets, uint8_t out[4]);

/* ---- synthetic inputs (SURVEY §8d) --------------------------------------------------------- */
/* splitmix64 stream reduced mod p, generated on the device: out[i] = splitmix64(seed, i) % p. */
int ronk_splitmix_fill_u64(ronk_ctx *ctx, uint64_t p, uint64_t seed, uint64_t *out, size_t n);

#ifdef __cplusplus
}
#endif
#endif /* RONK_B200_H */
