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
 *    `_host` variants take host pointers, copy in, run, copy out and synchronise.  Each context keeps the
 *    device scratch of its calls, the `_host` staging included, grown as needed, until ronk_ctx_destroy; a
 *    `_host` output buffer is written only when the call returns RONK_OK.
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
/* Coset transforms: in place, `batch` contiguous transforms of n = 2^log_n points on the coset s·H_n of the subgroup
 * H_n = {ω_n^k}, natural order, ω_n as for ronk_ntt_u64, s = `shift`:
 *   forward  X[k] = Σ_j a_j (s·ω_n^k)^j;   inverse: the a with those X, a_j = s^-j · n^-1 Σ_k X_k ω_n^(-jk).
 * - Any s in F_p* (elements of H_n included).  s = 1 gives exactly ronk_ntt_u64's words, through its own path.
 *   log_n = 0 is the identity.  Residues are canonical.
 * - Errors: those of ronk_ntt_u64 (RONK_EINVAL if 2^log_n does not divide p - 1, for a null pointer, g == 0 or g >= p;
 *   RONK_EUNSUPPORTED if log_n > 26), and RONK_EINVAL for s == 0 or s >= p.  batch == 0 does nothing.  Every check is
 *   made and all scratch (RONK_ENOMEM) is taken before anything is enqueued; on failure nothing is written.
 * - Kernels: the factor s^j (forward) or s^-j (inverse) is applied to the word at natural index j of its transform in
 *   the load of the first pass or the store of the last, so the transform moves the bytes of the plain one.  One small
 *   launch per call builds the factor tables: s^±i for i < 2^h and s^±(i·2^h) for i < 2^(log_n - h), h = ⌈log_n / 2⌉.
 *   n ≤ 2^13: the single-tile kernel; Goldilocks with g = 7 at 2^21 … 2^24: the three 256-point-tile passes; every
 *   other size and field: the generic two-pass tile kernels.  The cluster, split and interleaved kernels of
 *   ronk_ntt_u64 (Goldilocks 2^16 … 2^20, 2^25, 2^26) are not used, whatever the context's transform switches say.
 * - Scratch: the factor tables, 2^h + 2^(log_n - h) words (≤ 16 Ki), and for n > 2^13 the transform's workspace of
 *   batch·n words.
 * - The device variant is asynchronous on the context's stream; the _host variant stages in and out and synchronises. */
int ronk_ntt_coset_u64(ronk_ctx *ctx, uint64_t p, uint64_t g, uint64_t *data, uint32_t log_n, uint32_t batch, uint64_t shift, int inverse);
int ronk_ntt_coset_u64_host(ronk_ctx *ctx, uint64_t p, uint64_t g, uint64_t *host_data, uint32_t log_n, uint32_t batch, uint64_t shift, int inverse);
/* Low-degree extension: row r of coeffs (d words each, 1 ≤ d ≤ N = 2^log_n) evaluated on shift·H_N,
 *   out[r][k] = Σ_{j<d} coeffs[r][j] (shift·ω_N^k)^j, out is batch × N words.
 * - One launch copies the rows into out zero-extended to N words (poly_rows_pad_kernel), then the forward coset
 *   transform of ronk_ntt_coset_u64 runs in place on out (ronk_ntt_u64's transform for shift = 1).  Scratch: that of the
 *   transform, nothing more.
 * - Errors: those of ronk_ntt_coset_u64 for (p, g, log_n, shift), and RONK_EINVAL for a null coeffs, d == 0, d > N or
 *   an out that overlaps coeffs; RONK_EUNSUPPORTED for batch·N > 2^32 words.  batch == 0 does nothing.  Every check is
 *   made and all scratch is taken before anything is enqueued; on failure nothing is written.  coeffs is only read.
 * - The device variant is asynchronous on the context's stream; the _host variant stages in and out and synchronises. */
int ronk_poly_lde_u64(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *coeffs, size_t d, uint32_t log_n, uint64_t shift, uint32_t batch, uint64_t *out);
int ronk_poly_lde_u64_host(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *coeffs, size_t d, uint32_t log_n, uint64_t shift, uint32_t batch, uint64_t *out);
/* Polynomial::dft — src/polynomial/mod.rs:240-258.  Any n | p-1 (O(n²)); out must not alias in. */
int ronk_dft_u64(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *in, uint64_t n, uint64_t *out);
int ronk_dft_u64_host(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *in, uint64_t n, uint64_t *out);
/* Polynomial::dft (src/polynomial/mod.rs:240-258) and its inverse for ANY n | p - 1, in place, `batch` contiguous
 * transforms of n points, natural order: X[k] = Σ_j a_j ω^(jk), ω = g^((p-1)/n); inverse uses ω^-1 and scales by n^-1.
 * g generates F_p*, as for ronk_poly_mul_u64.  The forward result is, for every n, the words ronk_dft_u64 gives for
 * each transform (any g whose g^((p-1)/N) has order N will do, N below); for n a power of two both directions are the
 * words of ronk_ntt_u64.  Path, in O(n log n) except the third:
 *   - n a power of two: ronk_ntt_u64's transform (n ≤ 2^26);
 *   - Bluestein, when N = 2^⌈log2(2n - 1)⌉ ≤ 2^26 divides p - 1 and n reaches a measured crossover (DESIGN.md §5):
 *     two batched N-point transforms and two memory-bound chirp passes.  For Goldilocks that is every n | p - 1 up to
 *     2^25.  Scratch: batch·N words.  The spectrum of the chirp, N words (512 MiB at n = 3·2^23), is kept on the context
 *     per (p, g, n) until ronk_ctx_destroy;
 *   - otherwise ronk_dft_u64's O(n²) kernels, up to n ≤ 2^17.
 * RONK_EINVAL: a null pointer, n == 0, n not dividing p - 1, g == 0 or g >= p.  RONK_EUNSUPPORTED: p = 2, or n off all
 * three paths.  batch == 0 does nothing.  Nothing is written on failure.  The device variant is asynchronous on the
 * context's stream; the _host variant stages in and out and synchronises. */
int ronk_ntt_any_u64(ronk_ctx *ctx, uint64_t p, uint64_t g, uint64_t *data, uint64_t n, uint32_t batch, int inverse);
int ronk_ntt_any_u64_host(ronk_ctx *ctx, uint64_t p, uint64_t g, uint64_t *host_data, uint64_t n, uint32_t batch, int inverse);

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
/* Mul — src/polynomial/arithmetic.rs:97-119.  c has L = da+db-1 coefficients (no trimming), the same words on every path.
 * - NTT path (pad → NTT, NTT∘pointwise → iNTT over p, with g's roots of unity) when g != 0, a power of two N ≥ L
 *   divides p-1 and the product is large enough to pay for it.
 * - Multi-modular path when g != 0, no power of two ≥ L divides p-1 (p = 101, or an NTT prime past its 2-adicity),
 *   L ≤ 2^26, da·db ≥ 2^16 / 2^20 / 2^20 and min(da, db) ≥ 256 / 512 / 1024 for k = 1 / 2 / 3 (the measured
 *   crossovers; RONK_CRT_MUL_MIN replaces both with one bound on da·db): the integer product is convolved modulo the k ≤ 3 NTT primes 0xFFFFFFFF00000001,
 *   0xFFFFFFFF70000001 and 29·2^57+1, k the fewest whose product exceeds min(da, db)·(p-1)² (k = 1 up to p ≈ 2^19.5,
 *   k = 2 up to p ≈ 2^51.5 at min(da, db) = 2^25), and rebuilt by the Chinese remainder theorem.  Here g is only an
 *   on/off switch: the transforms use the auxiliary primes' own generators.  Device scratch: 2·N + k·L words, plus
 *   the transforms' own workspace of up to N words (3 GiB at L = 2^26, k = 3).
 * - Otherwise (and always for g = 0) the schoolbook kernel.
 * Asynchronous on every path.  On the two transform paths c may alias a or b (both operands are consumed before the
 * last launch writes c); on the schoolbook path c must not overlap a or b.  a, b and c need only the 8-byte alignment
 * of a uint64_t, and no word behind a[da), b[db) or c[L) is ever read or written. */
int ronk_poly_mul_u64(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *a, size_t da, const uint64_t *b, size_t db, uint64_t *c);
int ronk_poly_mul_u64_host(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *a, size_t da, const uint64_t *b, size_t db, uint64_t *c);
/* `batch` products at once: c[r] = a[r] · b[b_shared ? 0 : r], r < batch.  Rows are contiguous: a is batch × da,
 * b is batch × db (or db words when b_shared), c is batch × L, L = da + db − 1, each row untrimmed.
 * - Same words: every row holds exactly the words ronk_poly_mul_u64 gives for that row's pair, on every prime and path.
 * - Paths, chosen once per call from (p, g, da, db); N = 2^⌈log2 L⌉:
 *   fused: g != 0, N ≤ 2^11 divides p − 1 and da·db is above the crossover: ONE launch for the whole batch, each CTA
 *     multiplying 2^11/N products in shared memory (no scratch);
 *   batched transforms: g != 0, 2^11 < N ≤ 2^26 divides p − 1, above the crossover: zero-padded rows, batched forward
 *     transforms (b's with the point-wise product fused in), batched inverse, clipped rows.  Scratch 2·batch·N words
 *     (batch·N + N with a shared b) plus the transforms' workspace of batch·N words;
 *   multi-modular: g != 0, no power of two ≥ L divides p − 1, L ≤ 2^26, above the crossover: the two paths above modulo
 *     each of ronk_poly_mul_u64's k ≤ 3 auxiliary primes and one Chinese-remainder pass.  Scratch k·batch·L words,
 *     batch·da + batch·db (or + db) more where an auxiliary prime is below p, plus what the paths above take;
 *   otherwise (always for g = 0 and L > 2^26) the schoolbook kernel over batch·L outputs.
 *   RONK_POLY_BATCH_PATH forces a path where it applies (INTEGRATION.md).
 * - Errors: RONK_EINVAL for a null pointer, da == 0 or db == 0, an invalid modulus, g >= p, or a c that overlaps a or
 *   b (unlike the single product, c may never alias an operand: its rows are longer).  RONK_EUNSUPPORTED for
 *   da or db above 2^32, more than 2^40 words in a, b or c, or more than 2^32 words of batched transforms (batch·N on
 *   the batched-transform and multi-modular paths with N > 2^11).
 * - Every check is made and all scratch (RONK_ENOMEM) is taken before anything is enqueued; on failure nothing is
 *   written.  batch == 0 does nothing.  Asynchronous (the _host variant stages its arguments and synchronises).
 * - No word past a[batch·da), b[batch·db) (b[db) when shared) or c[batch·L) is read or written; 8-byte alignment. */
int ronk_poly_mul_batch_u64(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *a, size_t da, const uint64_t *b, size_t db, int b_shared, uint32_t batch, uint64_t *c);
int ronk_poly_mul_batch_u64_host(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *a, size_t da, const uint64_t *b, size_t db, int b_shared, uint32_t batch, uint64_t *c);
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
/* Lagrange-basis rows on a coset, evaluated at many points and opened at one point, in O(n) per point and row.
 * Nodes x_j = s·ω^j, j < n, ω = g^((p-1)/n), s = `shift` (s = 1: the reference's nodes, mod.rs:363).  Any n | p - 1.
 * `evals` is batch × n, row-major: row b holds f_b(x_j).  With Z(X) = X^n - s^n and the weights w_j = x_j / (n·s^n):
 *   eval:  out[b·m + i] = L_b(xs[i]) = Z(xs[i]) · Σ_j w_j·evals[b·n + j] / (xs[i] - x_j)   (out is batch × m).
 *          At a node the value is 0, the reference's l(x)·fold; with s = 1 every word is the one the single-point
 *          ronk_poly_lagrange_eval_u64_host above gives.
 *   open:  values[b] = f_b(z), the true value (evals[b·n + k] when z = x_k), and quotient (batch × n) the evaluations on
 *          the nodes of (f_b - f_b(z)) / (X - z): q_j = (y_j - f(z)) / (x_j - z); at z = x_k, q_k = f_b'(x_k).  This is
 *          kzg::open (src/kzg/setup.rs:63-78) in evaluation form.
 * - Errors, in this order: RONK_EINVAL for a null pointer; the modulus's (RONK_EUNSUPPORTED for p = 2); RONK_EINVAL for
 *   g == 0 or g >= p, n == 0 or n not dividing p - 1; RONK_EUNSUPPORTED for n or batch·n above 2^32 words; RONK_EINVAL
 *   when ω has order below n (two nodes coincide: the reference divides by zero, for every x), for shift == 0 or
 *   shift >= p, and (open) z >= p; RONK_EUNSUPPORTED (eval) for batch·m above 2^32 words; RONK_EINVAL for an output that
 *   overlaps an input, or values that overlap quotient.  Past those, RONK_EUNSUPPORTED (eval) for more than 2^31 - 1
 *   tiles of nodes and points (about m·n > 2^42).  batch == 0 or m == 0 does nothing.
 * - xs are taken as canonical and not read on the host; the _host twin refuses a non-canonical point (RONK_EINVAL) before
 *   it stages anything.  Every check is made and all scratch is taken before the first launch; nothing is written on
 *   failure.  Scratch: ω^-1's two power tables (2^h + 2^(⌈log2 n⌉ - h) words, h = ⌈⌈log2 n⌉ / 2⌉) and the per-CTA partial
 *   sums, ⌈m / M⌉·⌈n·M / 4096⌉·batch·M words with M = 1, 2, 4 or 8 points per pass (at most 8, the smallest that holds m).
 * - Kernels: one CTA forms its 4096 coefficients x_j / (x - x_j) with one batch inversion per 16 per thread, then streams
 *   every row's tile through per-(row, point) accumulators, so each evaluation word is read once per group of 8 points;
 *   a finish launch sums the partials in a fixed order and scales by Z(x) / (n·s^n).  The launch sequence depends only on
 *   (p, g, n, shift), and for open on whether z ∈ s·H_n, which the host decides by (z/s)^n = 1:
 *   off the nodes the evaluation at z, then one quotient launch; on a node the device finds k, the quotient launch gathers
 *   the values, and the evaluation's partial and finish kernels fill q_k = -x_k^-1 Σ_{j≠k} x_j q_j.  Asynchronous on the
 *   context's stream; no readback.  The _host twins stage in and out and synchronise (the batched evaluation's twin has
 *   its own name, because the single-point Lagrange evaluate above holds the plain one). */
int ronk_poly_lagrange_eval_u64(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *evals, uint64_t n, uint32_t batch,
                                uint64_t shift, const uint64_t *xs, size_t m, uint64_t *out);
int ronk_poly_lagrange_eval_batch_u64_host(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *evals, uint64_t n,
                                           uint32_t batch, uint64_t shift, const uint64_t *xs, size_t m, uint64_t *out);
int ronk_poly_lagrange_open_u64(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *evals, uint64_t n, uint32_t batch,
                                uint64_t shift, uint64_t z, uint64_t *values, uint64_t *quotient);
int ronk_poly_lagrange_open_u64_host(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *evals, uint64_t n, uint32_t batch,
                                     uint64_t shift, uint64_t z, uint64_t *values, uint64_t *quotient);
/* quotient_and_remainder / Div / Rem — src/polynomial/mod.rs:170-225, arithmetic.rs:121-146.
 * q and r both have da terms.  Host pointers: ronk_poly_divrem_u64 below with g = 0, so a divisor that is not linear
 * keeps the literal long division.  RONK_EINVAL for an all-zero divisor. */
int ronk_poly_divrem_u64_host(ronk_ctx *ctx, uint64_t p, const uint64_t *a, size_t da, const uint64_t *b, size_t db, uint64_t *q, uint64_t *r);
/* quotient_and_remainder / Div / Rem — src/polynomial/mod.rs:170-225, arithmetic.rs:121-146, on DEVICE pointers.
 * q and r both have da terms (the reference's zero-padded arrays), exactly what ronk_poly_divrem_u64_host returns,
 * including RONK_EINVAL where the reference panics.  q and r must not alias a, b or each other.  Synchronous: the
 * host reads b[db-1] to choose a path.  A divisor with a zero top word keeps the literal long division (the
 * reference's partly reduced remainder and its panics).  Otherwise the division is Euclidean: a linear divisor takes
 * the scan of ronk_poly_div_linear_u64, and with g != 0 a generator of F_p* (as in ronk_poly_mul_u64) and every
 * transform of about 2(da - db + 1) and db - 1 points a power of two dividing p - 1 and ≤ 2^26, it runs as Newton
 * iteration on the transforms (a fixed number of transforms instead of O(da·(da - db)) sequential steps).  g == 0,
 * or a prime with too few 2-power roots of unity (p = 101, 17, 127), keeps the literal kernel.  Residues canonical. */
int ronk_poly_divrem_u64(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *a, size_t da, const uint64_t *b, size_t db, uint64_t *q, uint64_t *r);
/* `batch` divisions at once: row y of q and r is exactly what ronk_poly_divrem_u64(p, g, a[y], b_shared ? b : b[y]) gives,
 * on every prime and path, the reference's quirks for a zero top word included.  Rows are contiguous, in the order of
 * ronk_poly_mul_batch_u64: a is batch × da, b is batch × db (db words when b_shared), q and r are batch × da each.
 * - Errors, in this order: (1) without reading a pointer: RONK_EINVAL for a null pointer (when batch·da > 0), an invalid
 *   modulus or g >= p; RONK_EUNSUPPORTED for da or db above 0x7FFFFFF0, batch·da or batch·db above 2^40 words, and, where
 *   the path rule below puts rows with nonzero top words on Newton iteration, batch × the plan's larger transform above
 *   2^32 words; (2) RONK_EINVAL for a q or r that overlaps a, b or the other output; (3) the divisors' top words are read
 *   back; (4) RONK_EINVAL where any row panics in the reference, as the single-row entry does on it.  After (1) and (2)
 *   nothing is written; after (4) the words of q and r are unspecified.  batch == 0 or da == 0 does nothing.
 * - Batch 1 is ronk_poly_divrem_u64 itself: same words, same launches.  From batch 2, with L = da − db + 1, one path for
 *   the whole call:
 *   any top word 0 (any row, or the shared b; db == 0): every row on the literal kernel, one CTA per row.  A row with a
 *     nonzero top word gets its Euclidean words from that kernel too, so the batch is never split;
 *   da < db: q = 0 and r = a (one memset, one copy);
 *   db == 2: the scan of ronk_poly_div_linear_u64 over every row (z = −b0/b1 and b1^-1 per row: on the host for a shared
 *     divisor, in one launch otherwise); r[0] = a(z) and the rest of each r is 0.  Scratch 2·batch·⌈da/4096⌉ + 2·batch words;
 *   Newton iteration where its transforms fit (as ronk_poly_divrem_u64) and the measured rule prefers it (DESIGN.md §5):
 *     one inverse of rev(b) (shared) or one batched inversion of every row's, then the quotient and the remainder's low
 *     words as batched cyclic products.  Scratch rows·(L + min(db, L) + N) + batch·N words plus the transforms' workspace
 *     (batch·N words past 2^15 points) and 8·256 bytes, N = the larger of the plan's two transforms, rows = 1 when b_shared
 *     else batch.  Taken before the first launch that writes q or r;
 *   otherwise the literal kernel over every row.
 *   RONK_DIVREM_BATCH_PATH forces literal (1) or Newton wherever it fits (2) from batch 2 (INTEGRATION.md).
 * - Synchronous: the top words are read back once (one copy of a shared divisor's top, or b[0..2) when db == 2; one scan
 *   launch over per-row divisors), the literal path reads its panic flag.  The launch sequence from batch 2 depends on the
 *   batch only where ronk_ntt_u64 picks its kernels by batch at 2^16 points.
 * - The _host twin makes every check of (1) before it stages anything, stages in and out and synchronises.  Residues
 *   canonical; 8-byte alignment; no word past a[batch·da), b[batch·db) (b[db) when shared), q or r[batch·da) is touched. */
int ronk_poly_divrem_batch_u64(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *a, size_t da, const uint64_t *b, size_t db,
                               int b_shared, uint32_t batch, uint64_t *q, uint64_t *r);
int ronk_poly_divrem_batch_u64_host(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *a, size_t da, const uint64_t *b,
                                    size_t db, int b_shared, uint32_t batch, uint64_t *q, uint64_t *r);
/* Division by a linear factor b0 + b1*x — the divisor kzg::open builds (src/kzg/setup.rs:72-75,
 * [-z, 1]) fed to Polynomial::div (src/polynomial/mod.rs:170-225, arithmetic.rs:121-146) — as a
 * device-wide scan.  Device pointers: a (d terms), q (d terms, q[d-1] = 0 like the reference's
 * zero-padded quotient), rem (1 word = a(-b0/b1)).  q must not alias a.  RONK_EINVAL for b1 == 0.
 * ronk_poly_divrem_u64[_host] take this path by themselves when db == 2, b[1] != 0 and da >= 2. */
/* Lagrange interpolation through (xs[i], ys[i]), i < k: the monomial coefficients out[0..k).  This is
 * Message::decode of src/codes/reed_solomon.rs:55-107 applied to the first K coordinates of a
 * codeword (the reference enumerates combinations; the interpolant is unique).  Host pointers,
 * k <= 8192.  RONK_EINVAL for a repeated x (the reference's `/` panics on the zero denominator). */
int ronk_poly_interpolate_u64_host(ronk_ctx *ctx, uint64_t p, const uint64_t *xs, const uint64_t *ys, size_t k, uint64_t *out);
/* Multipoint evaluation and interpolation on a subproduct tree, DEVICE pointers, on the context's stream.
 * Path rule (as ronk_poly_divrem_u64): the tree runs in O(n log² n) when g != 0 is a generator of F_p*, every transform
 * of its plan is a power of two dividing p - 1 and ≤ 2^26, and the size reaches a measured crossover (DESIGN.md §3.5);
 * otherwise the existing kernels run.  Envelope: at most 2^24 points (tree leaves; the largest tree transform has 2^25
 * points), else RONK_EUNSUPPORTED.  RONK_EINVAL for a null pointer, g >= p, or an output that overlaps an input.
 * Nothing is written on failure.  Residues canonical. */
/* Π_{i<k} (X - xs[i]): out has k + 1 coefficients, out[k] = 1 (k = 0: out[0] = 1).  Off the tree: one CTA of k
 * sequential linear products, at most 8192 roots (RONK_EUNSUPPORTED above); k ≤ 64 is always the tree's shared-memory
 * kernel alone.  Asynchronous. */
int ronk_poly_from_roots_u64(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *xs, size_t k, uint64_t *out);
/* evaluate — src/polynomial/mod.rs:133-139 at m points, as Shamir split evaluates at 1..n (src/shamir/mod.rs:53-58):
 * out[i] = Σ_j coeffs[j]·xs[i]^j, i < m, the same words as ronk_poly_eval_u64 for every d (including 0) and m; repeated
 * points are fine.  The tree path also needs d ≤ 2^25 (its root division has transforms of 2·d points); off it,
 * ronk_poly_eval_u64's kernel runs.  Asynchronous. */
int ronk_poly_multieval_u64(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *coeffs, size_t d, const uint64_t *xs, size_t m, uint64_t *out);
/* Device twin of ronk_poly_interpolate_u64_host (Message::decode, src/codes/reed_solomon.rs:55-107): the unique
 * interpolant through (xs[i], ys[i]), k coefficients.  Off the tree path it runs the same kernels as the host variant,
 * capped at 8192 nodes (RONK_EUNSUPPORTED above); the tree takes every k > 8192 it fits.  Synchronous; RONK_EINVAL for a
 * repeated x (the reference's `/` panics on the zero denominator). */
int ronk_poly_interpolate_u64(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *xs, const uint64_t *ys, size_t k, uint64_t *out);
/* Batches over one shared point set (Shamir split and combine over many secrets, Message::decode of many codewords, a
 * prover's columns at the same points): one tree per call, shared by every row.  DEVICE pointers, row-major.
 * multieval: coeffs is batch × d, out is batch × m, out[b·m + i] = Σ_j coeffs[b·d + j]·xs[i]^j.
 * interpolate: ys is batch × k, out is batch × k, row b the interpolant through (xs[i], ys[b·k + i]).
 * - Words: every row is word for word what ronk_poly_multieval_u64 / ronk_poly_interpolate_u64 give for it.
 * - Path rule: the tree runs where tree_fits, as for one row, and from a crossover that depends on the batch, because
 *   the literal kernels' cost grows with it and the tree's barely does (DESIGN.md §5).  With n = min(d, m), multieval
 *   takes the tree from n ≥ 2^15, batch·n² ≥ 2^30 or batch·n ≥ 2^18; interpolation from k ≥ 2048 or batch·k² ≥ 2^28,
 *   and at every k > 8192.  At batch 1 that is the single-row rule.  RONK_TREE_MIN overrides it whatever the batch.
 * - Launches: at batch 1 the launch sequence is the single-row entry's; from batch 2 it does not depend on the batch (save where ronk_ntt_u64 picks its
 *   kernels by batch, at 2^16 points).  On the tree the node spectra are transformed once per level and met with every
 *   row in one launch; interpolation evaluates M'(x_i) once and inverts it once.  Off the tree one poly_eval launch, or
 *   one interp_master and one interp_nodes / interp_sum pair, serves every row.
 * - Errors, in the single-row order: RONK_EINVAL for a null pointer, a bad modulus, g >= p; RONK_EUNSUPPORTED above 2^24
 *   points; then RONK_EINVAL when out overlaps an input; RONK_EUNSUPPORTED when the tree's row buffers pass 2^32 words
 *   (batch·N, N = 2^⌈log2 m⌉ or 2^⌈log2 k⌉, for multieval at least the root's 2^⌈log2(2d - 1)⌉, as
 *   ronk_poly_mul_batch_u64), when off the tree the interpolation's partial sums pass 2^32 words
 *   (batch·⌈k/256⌉·8·k), or for more than 8192 nodes off the tree.  interpolate: RONK_EINVAL for a repeated node (the
 *   reference divides by zero), with out not written.  batch == 0, m == 0 or k == 0 does nothing.
 * - Every check is made and all scratch is taken before the first launch; nothing is written on failure.  Scratch on
 *   the tree: the stored levels (under 2N + 6·N/64 words), 2N words of node spectra, 3·batch·N words of rows (2N at
 *   batch 1), for interpolation 2k words, the root's 2·N_q + d + 1 + min(m + 1, d) + 3·batch·d words (N_q =
 *   2^⌈log2(2d - 1)⌉; interpolation evaluates M' as one row of k), and the largest transform workspace (batch·N words)
 *   or batched product's.  Off the tree: none for multieval; batch·k + 2(k + 1) + batch·⌈k/256⌉·8·k words for
 *   interpolation.
 * - multieval is asynchronous.  interpolate synchronises once to read the repeated-node flag, as the single-row entry.
 *   The _host twins make every check that reads no pointer, the size checks included, before they stage anything;
 *   they stage in and out and synchronise. */
int ronk_poly_multieval_batch_u64(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *coeffs, size_t d, uint32_t batch,
                                  const uint64_t *xs, size_t m, uint64_t *out);
int ronk_poly_multieval_batch_u64_host(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *coeffs, size_t d,
                                       uint32_t batch, const uint64_t *xs, size_t m, uint64_t *out);
int ronk_poly_interpolate_batch_u64(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *xs, const uint64_t *ys, size_t k,
                                    uint32_t batch, uint64_t *out);
int ronk_poly_interpolate_batch_u64_host(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *xs, const uint64_t *ys,
                                         size_t k, uint32_t batch, uint64_t *out);
int ronk_poly_div_linear_u64(ronk_ctx *ctx, uint64_t p, const uint64_t *a, size_t d, uint64_t b0, uint64_t b1, uint64_t *q, uint64_t *rem);

/* ---- Reed–Solomon codes ------------------------------------------------------------------- */
/* Position i < n of a codeword holds the value at ω_n^i, ω_n = g^((p-1)/n): the domain of Message::encode
 * (src/codes/reed_solomon.rs:42-52).  Row-major, DEVICE pointers, asynchronous on the context's stream.
 * Arguments: RONK_EINVAL for a null pointer, n == 0, k == 0, k > n, n not dividing p - 1, g == 0 or g >= p, ω_n of order
 * below n (two positions would share a point; g must generate a subgroup of order divisible by n), or an output that
 * overlaps an input.  RONK_EUNSUPPORTED for p = 2, n off ronk_ntt_any_u64's paths, or 3·batch·n ≥ 2^31 (decode;
 * batch·n for encode).  batch == 0 does nothing.  Every check is made before anything is enqueued; nothing is written
 * on failure.  The transforms are ronk_ntt_any_u64's: below its crossover, for n not a power of two, a batched O(n²)
 * kernel takes every row in one launch, so the launch sequence of a call does not depend on the batch (save where
 * ronk_ntt_u64 itself picks its kernels by batch, at 2^16 points). */
/* Message::encode of `batch` messages msg (batch × k): codeword[b][i] = m_b(ω_n^i), i < n (batch × n). */
int ronk_rs_encode_u64(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *msg, uint64_t k, uint64_t n, uint32_t batch,
                       uint64_t *codeword);
/* Errors-and-erasures decoding of `batch` received words (batch × n).  erased (batch × n bytes) may be NULL, meaning no
 * erasures; a nonzero byte marks that position as erased.  Writes msg (batch × k) and status (batch entries).
 * Guarantee: if row b differs from the codeword of a message m in e non-erased positions, with ε erased positions and
 * 2e + ε ≤ n - k, then msg[b] = m and status[b] = e.  Otherwise the row gets status[b] = -1 with msg[b] all zero, or a
 * message m' with status[b] = e' whose codeword differs from the row in e' non-erased positions, 2e' + ε ≤ n - k: the
 * decoder is bounded-distance and never returns a message outside the decoding radius.  A failed row is a result, not
 * an error; the call never reads back to the host.
 * n - k is at most RONK_RS_MAX_PARITY (the Berlekamp–Massey locator runs in one CTA per row, in shared memory);
 * above it RONK_EUNSUPPORTED.  Scratch: 4·batch·n words + batch·16 bytes (below the crossover also n + 3·batch·(n-k+1)
 * words), plus the transforms' own (Bluestein: 3·batch·N words, N = 2^⌈log2(2n - 1)⌉).
 * The _host variant takes host pointers, stages in and out and synchronises. */
#define RONK_RS_MAX_PARITY 8191
int ronk_rs_decode_u64(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *received, const uint8_t *erased, uint64_t n,
                       uint64_t k, uint32_t batch, uint64_t *msg, int32_t *status);
int ronk_rs_decode_u64_host(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *received, const uint8_t *erased,
                            uint64_t n, uint64_t k, uint32_t batch, uint64_t *msg, int32_t *status);
/* Errors-and-erasures decoding of `batch` received words (batch × n) whose positions share any n distinct points xs
 * (canonical residues; 0 is allowed): row b is meant to be f_b(xs[i]) for an f_b of degree < k, for example Shamir
 * shares at x = 1..n.  erased, msg, status and the guarantee are those of ronk_rs_decode_u64: within 2e + ε ≤ n - k
 * msg[b] = f_b and status[b] = e; otherwise -1 with a zero message, or a message whose evaluations differ from the row
 * in e' non-erased positions, 2e' + ε ≤ n - k.  The values at erased positions are never read.  At xs[i] = ω_n^i this
 * gives ronk_rs_decode_u64's words, beyond the radius too.
 * Steps, with m = n - k and M = Π (X - x_i): the interpolant of each row (erasures zeroed) gives the syndromes
 * S_j = Σ_i r_i·x_i^j / M'(x_i) through one product with 1 / (z^n·M(1/z)) mod z^m (ronk_poly_divrem_u64's quotient);
 * the Berlekamp–Massey locator of ronk_rs_decode_u64; one batched multieval of the 3·batch locator rows (m + 1 words)
 * and one of M' over xs; Forney's e_i = Ω̂(x_i)·M'(x_i)/σ'(x_i) at the roots; a second batched interpolation and the
 * check that it has degree < k.  Each step takes its entry point's path: the subproduct tree up to 2^24 points, the
 * literal kernels up to 8192; g = 0 keeps every step on the literal kernels.
 * Errors, in this order: RONK_EINVAL for a null pointer (xs, received, msg, status), a bad modulus, g >= p, n == 0, k == 0
 * or k > n; RONK_EUNSUPPORTED for n - k > RONK_RS_MAX_PARITY, n > 2^24, 3·batch ≥ 2^32, past the envelope of
 * ronk_poly_interpolate_batch_u64 over batch rows or of ronk_poly_multieval_batch_u64 over 3·batch rows of n - k + 1
 * words, or batch·2^⌈log2(2(n - k) - 1)⌉ > 2^32; then RONK_EINVAL for an output that overlaps an input, and for a
 * repeated point (found by the first interpolation, before anything is written).  batch == 0 does nothing.  Nothing is
 * written to msg or status on any error.
 * Scratch: 8·(batch·(5n + 6(n - k) + 4) + 6n + 4(n - k) + 1) bytes, with above it the largest that one step's entry
 * point takes: the batched interpolation's over batch rows, the batched multieval's over 3·batch rows, ronk_poly_divrem_u64's
 * of n + m words by n + 1 and ronk_poly_mul_batch_u64's of batch rows of n - k words by one shared row.
 * The call synchronises with the host: each interpolation reads its repeated-node flag and the division reads the
 * divisor's top word.  The _host variant makes every check above but the repeated point before it stages anything,
 * refuses a point x >= p with RONK_EINVAL, stages in and out and synchronises. */
int ronk_rs_decode_at_u64(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *xs, const uint64_t *received,
                          const uint8_t *erased, uint64_t n, uint64_t k, uint32_t batch, uint64_t *msg, int32_t *status);
int ronk_rs_decode_at_u64_host(ronk_ctx *ctx, uint64_t p, uint64_t g, const uint64_t *xs, const uint64_t *received,
                               const uint8_t *erased, uint64_t n, uint64_t k, uint32_t batch, uint64_t *msg, int32_t *status);

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
/* `batch` commitments against one SRS (kzg::commit of many coefficient rows: a prover's columns, the quotients of
 * kzg.open_batch).  scalars is batch × n_scalars bytes, row-major, rows contiguous with no padding and no stride; out is
 * batch × 4 bytes in the packed point format above.  All pointers are DEVICE pointers.
 * - Words: out[4r .. 4r+4) is exactly the point ronk_msm_pluto_ext(points, n_points, scalars + r·n_scalars, n_scalars)
 *   returns, for every r < batch.
 * - Errors, in this order: (1) without reading memory: RONK_EINVAL for a null ctx, a null points or scalars when
 *   batch·n_scalars > 0, a null out when batch > 0, n_points < n_scalars (the reference's assert, kzg/setup.rs:53), or
 *   points or out not 4-byte aligned (scalars may have any alignment); RONK_EUNSUPPORTED for batch·n_scalars above 2^40
 *   bytes; (2) RONK_EINVAL when out overlaps points[0, 4·n_scalars) or the scalar block; (3) scratch (RONK_ENOMEM) is
 *   taken before the first launch; (4) the call runs, then RONK_EINVAL if any of the first n_scalars points is off the
 *   curve or non-canonical, or any scalar of any row is ≥ 17, with out not written (the last launch decides that on the
 *   device).  After (1) and (2) nothing has been enqueued or written.  batch == 0 does nothing; n_scalars == 0 writes
 *   Infinity to every row (the empty sum, curve/mod.rs:219-223), with one memset.
 * - Launches, three whatever the batch: msm_coord_pack looks up each of the first n_scalars points' group coordinates
 *   (a_i, b_i) once and writes them as two byte planes; msm_rows streams the scalar rows once and takes each row's
 *   Σ s_i·a_i and Σ s_i·b_i mod 102 per column of 2048 scalars by __dp4a, four terms at a time; msm_rows_finish sums each
 *   row's columns and looks the point up.  The group tables are built once per context on first use, by either commit
 *   entry.  RONK_MSM_COORD, RONK_MSM_HIST and RONK_MSM_SPLIT select paths for ronk_msm_pluto_ext only.
 * - Scratch: 2·⌈n_scalars/16⌉·16 bytes of planes and 4·batch·⌈n_scalars/2048⌉ bytes of column sums.
 * - Synchronises once, to read the error flag, as ronk_msm_pluto_ext does.  The _host twin makes the checks of (1) but
 *   the alignment check (its staging aligns the device buffers) before it stages anything, ships only the first
 *   n_scalars points, stages in and out and synchronises. */
int ronk_msm_pluto_ext_batch(ronk_ctx *ctx, const uint8_t *points, size_t n_points, const uint8_t *scalars,
                             size_t n_scalars, uint32_t batch, uint8_t *out);
int ronk_msm_pluto_ext_batch_host(ronk_ctx *ctx, const uint8_t *points, size_t n_points, const uint8_t *scalars,
                                  size_t n_scalars, uint32_t batch, uint8_t *out);
/* The reference's Tate pairing (curve/pairing.rs:33-54) of PlutoExtendedCurve with R = 17 on n pairs:
 * out[2i], out[2i+1] = c0, c1 of pairing(p[i], q[i]) ∈ GF(101²).  And kzg::check (kzg/setup.rs:81-103) of n openings
 * against one SRS: ok[r] = 1 when pairing(proofs[r], g2_srs[1] − GEN·points[r]) == pairing(commitments[r] −
 * g1_srs[0]·values[r], GEN), else 0, with GEN = PlutoExtendedCurve::GENERATOR (36, 31t).
 * - Layout: points in the packed 4-byte format above, 0xFFFFFFFF is Infinity.  p, q, commitments and proofs are n × 4
 *   bytes; points and values are n bytes each, F17 residues; out is 2n bytes, ok is n bytes; g1_srs holds n_g1 points
 *   and g2_srs n_g2, of which the check reads only g1_srs[0] and g2_srs[1].  All pointers of the device entries are
 *   DEVICE pointers.
 * - Words: each output byte is exactly what the reference computes for its row.  Only points of E[17] pair: the 289
 *   points a·G1 + b·G2 with 6 | a and 6 | b in a basis of E ≅ (Z/102)².  The literal Miller loop (zero-skipping, the
 *   `zeros` counter, the final x^600) is run once per context on every pair of E[17] into an 83 521-byte table, built on
 *   first use by either entry after the commit's group tables; its values are not bilinear, so nothing is derived from
 *   a basis.  A row is then four coordinate lookups, a little arithmetic mod 102 and table lookups.
 * - Errors, in this order: (1) without reading memory: RONK_EINVAL for a null ctx, a null pointer when n > 0, n_g1 == 0
 *   or n_g2 < 2 (the reference's two panics, whatever n), or a point array (p, q, commitments, proofs, g1_srs, g2_srs)
 *   not 4-byte aligned; RONK_EUNSUPPORTED for n ≥ 2^32; (2) RONK_EINVAL when an output overlaps an input (for the
 *   check: commitments, proofs, points, values, g1_srs[0] or g2_srs[0..2)); (3) scratch and the one-time tables are
 *   taken (RONK_ENOMEM / RONK_ECUDA); (4) the call runs, then RONK_EINVAL if any row panics in the reference or holds
 *   input the ABI rejects: an off-curve or non-canonical point (for the check: a commitment, a proof, g1_srs[0] or
 *   g2_srs[1]), a scalar ≥ 17; for the pairing an argument outside E[17], Infinity, or P == Q; for the check either
 *   pairing panicking (the proof, g2_srs[1] − GEN·point or commitment − g1_srs[0]·value is Infinity or outside E[17],
 *   or the pair is one of the table's panics).  After (1) and (2) nothing has been enqueued or written; after (4) the
 *   output bytes are unspecified.  n == 0 does nothing.
 * - Launches: one whatever n (kzg_check keeps both tables in shared memory; pairing reads them through L1), plus the
 *   table build on a context's first call.  Synchronises once, to read the error flag, as ronk_msm_pluto_ext_batch does.
 * - The _host twins make the checks of (1) but the alignment check (their staging aligns the device buffers) before they
 *   stage anything; the check twin ships only g1_srs[0] and g2_srs[0..2). */
int ronk_pairing_pluto_ext(ronk_ctx *ctx, const uint8_t *p, const uint8_t *q, size_t n, uint8_t *out);
int ronk_pairing_pluto_ext_host(ronk_ctx *ctx, const uint8_t *p, const uint8_t *q, size_t n, uint8_t *out);
int ronk_kzg_check_pluto_ext_batch(ronk_ctx *ctx, const uint8_t *commitments, const uint8_t *proofs,
                                   const uint8_t *points, const uint8_t *values, size_t n,
                                   const uint8_t *g1_srs, size_t n_g1, const uint8_t *g2_srs, size_t n_g2, uint8_t *ok);
int ronk_kzg_check_pluto_ext_batch_host(ronk_ctx *ctx, const uint8_t *commitments, const uint8_t *proofs,
                                        const uint8_t *points, const uint8_t *values, size_t n,
                                        const uint8_t *g1_srs, size_t n_g1, const uint8_t *g2_srs, size_t n_g2, uint8_t *ok);
/* ---- Poseidon (src/hashes/poseidon) ------------------------------------------------------------ */
/* The reference's Poseidon permutation (poseidon/mod.rs:137-149) and sponge (sponge.rs:71-294) over F_p on batches of
 * rows.  A configuration is (width T, alpha, num_f, num_p, rc, mds) as PoseidonConfig::new (mod.rs:39-56) takes it:
 * rc holds R·T words with R = num_f + num_p, mds holds T² words row-major (mds[i·T + j] is mds[i][j]).  Round i adds
 * rc[i·T ..], raises every element to alpha when i < num_f/2 or i ≥ num_p + num_f/2 and element 0 only otherwise
 * (mod.rs:87-93), then multiplies by the MDS matrix, literally; x^0 = 1 for every x, as Field::pow gives.  Rows are
 * contiguous and row-major.  All pointers of the device entries are DEVICE pointers.
 * - ronk_poseidon_permute_u64: replaces each of the batch states (T words each) by its permutation.  Poseidon::hash is
 *   this on the state zero-padded to T words, then word 1.
 * - ronk_poseidon_sponge_u64: row y gets a fresh PoseidonSponge of this rate (capacity T − rate), absorbs
 *   in[y·len, (y+1)·len), starts squeezing and squeezes n_out words into out[y·n_out ..].  Any split of the absorbed
 *   words into absorb calls and of the squeezed count into squeeze calls gives these words.  len == 0 runs no
 *   permutation before the first squeeze, as start_squeezing runs one only when absorb_index != 0.
 * - Errors, in this order: (1) without reading a pointer: RONK_EINVAL for a null ctx, or a null pointer the call would
 *   read or write (states when batch > 0; in when batch·len > 0; out when batch·n_out > 0; rc and mds when batch > 0
 *   and R > 0); the modulus check every F_p entry makes (p = 2 is RONK_EUNSUPPORTED, a composite p RONK_EINVAL);
 *   RONK_EINVAL for T < 2 (the reference's assert), and for the sponge rate == 0 or rate > T; RONK_EUNSUPPORTED for
 *   T > 16, for R·T + T² above 6144 words of constants (48 KiB of shared memory: up to 368 rounds at T = 16), and for
 *   batch·T, batch·len or batch·n_out above 2^40 words; (2) RONK_EINVAL when the output (states, out) overlaps rc, mds
 *   (when R > 0) or, for the sponge, in.  On a refusal nothing has been enqueued or written.  batch == 0 does nothing,
 *   and so does n_out == 0.  The words must be canonical residues (< p); the device entries do not check them, and
 *   give unspecified words for others.
 * - Launches: one whatever the batch, one thread per row (128-thread CTAs, at most 8 per SM, grid-stride).  Each CTA
 *   holds the constants in shared memory.  Asynchronous on the context's stream.
 * - The _host twins make every check of (1), then refuse a non-canonical word of rc, mds and the states or in with
 *   RONK_EINVAL before they stage anything; they stage in and out and synchronise. */
int ronk_poseidon_permute_u64(ronk_ctx *ctx, uint64_t p, uint32_t width, uint64_t alpha, uint32_t num_f, uint32_t num_p,
                              const uint64_t *rc, const uint64_t *mds, uint64_t *states, size_t batch);
int ronk_poseidon_permute_u64_host(ronk_ctx *ctx, uint64_t p, uint32_t width, uint64_t alpha, uint32_t num_f,
                                   uint32_t num_p, const uint64_t *rc, const uint64_t *mds, uint64_t *states, size_t batch);
int ronk_poseidon_sponge_u64(ronk_ctx *ctx, uint64_t p, uint32_t width, uint64_t alpha, uint32_t num_f, uint32_t num_p,
                             const uint64_t *rc, const uint64_t *mds, uint32_t rate, const uint64_t *in, size_t len,
                             size_t batch, uint64_t *out, size_t n_out);
int ronk_poseidon_sponge_u64_host(ronk_ctx *ctx, uint64_t p, uint32_t width, uint64_t alpha, uint32_t num_f,
                                  uint32_t num_p, const uint64_t *rc, const uint64_t *mds, uint32_t rate,
                                  const uint64_t *in, size_t len, size_t batch, uint64_t *out, size_t n_out);
/* ---- SHA-256 and Merkle trees (src/hashes/sha.rs, src/tree/merkle.rs) ------------------------------------------ */
/* The reference's Sha256::digest (sha.rs:88-201: standard SHA-256) on batches of byte strings, and its MerkleTree
 * (merkle.rs:31-98) built, opened and verified on the device.  A digest is 32 bytes, h0 … h7 each big-endian.  A batch
 * of n messages is data[offsets[i], offsets[i+1]) for i < n: offsets holds n + 1 uint64_t, non-decreasing, with
 * offsets[n] ≤ data_len; any start alignment.  All pointers of the device entries are DEVICE pointers.
 * - Tree layout: level l (0 = the leaves' digests) holds s_l = ⌈n / 2^l⌉ nodes, l = 0 … L with L = ⌈log2 n⌉ for n ≥ 2
 *   and L = 0 for n = 1; level l + 1 node i is digest(level_l[2i] ‖ level_l[2i + 1]), the last node of an odd level
 *   paired with itself.  `nodes` holds the levels leaf level first, each contiguous: level l starts at node
 *   off_l = Σ_{k<l} s_k (byte 32·off_l), the root is node off_L, and the buffer is (off_L + 1)·32 bytes.  The reference
 *   stores the same levels root first (MerkleTree::hashes).
 * - ronk_sha256: out[32·i ..] = digest(message i).  One launch.
 * - ronk_merkle_build_sha256: every level of the tree of the n messages into nodes.  n == 0 does nothing (the
 *   reference's tree of no leaves has no root).  1 + ⌈max(L − 9, 0) / 9⌉ launches: each CTA reduces 512 nodes through
 *   up to 9 levels in shared memory.
 * - ronk_merkle_proofs_sha256: get_proof (merkle.rs:66-81) of each of the m leaf indices against the tree of n leaves
 *   in nodes (as built above): for l < L, siblings[(j·L + l)·32 ..] = node (indices[j] >> l) ^ 1 of level l and
 *   sides[j·L + l] = 1 (Right) when indices[j] >> l is even, else 0 (Left).  An index at which that sibling lies past
 *   its level is where the reference panics (e.g. n = 5: indices 4 and 5; n = 3: index 3 is accepted).  n ≤ 1 gives
 *   L = 0 and empty proofs.  One launch when m·L > 0.
 * - ronk_merkle_verify_sha256: ok[j] = 1 when prove (merkle.rs:84-98) holds for message j of the m messages with the
 *   depth steps siblings[(j·depth + l)·32 ..], sides[j·depth + l] (0 = Left: digest(sibling ‖ h), 1 = Right:
 *   digest(h ‖ sibling)) against the 32-byte root, else 0.  depth may be 0.  One launch.
 * - Errors, in this order: (1) without reading memory: RONK_EINVAL for a null ctx or a null pointer the call would use
 *   (data may be null when data_len == 0; offsets and the output when n or m is 0; the proofs' pointers when m·L == 0;
 *   siblings and sides when depth == 0), and for offsets or indices not 8-byte aligned (device entries);
 *   RONK_EUNSUPPORTED for n or m ≥ 2^32, data_len > 2^40 or depth > 32; (2) RONK_EINVAL for an output that overlaps an
 *   input (or, for the proofs, the other output); nothing is enqueued or written before this point, and no scratch is
 *   taken; (3) the call runs, synchronises once, and returns RONK_EINVAL if the device saw offsets that decrease or pass
 *   data_len, a proof index at which get_proof panics, or a side byte other than 0 or 1.  Output contents are then
 *   unspecified.  No kernel reads data outside [offsets[0], offsets[n]) or nodes outside the tree, whatever the input.
 * - The _host twins take host pointers, make the checks of (1), refuse bad offsets and side bytes on the host before
 *   they stage anything, then stage and synchronise. */
int ronk_sha256(ronk_ctx *ctx, const uint8_t *data, uint64_t data_len, const uint64_t *offsets, size_t n, uint8_t *out);
int ronk_sha256_host(ronk_ctx *ctx, const uint8_t *data, uint64_t data_len, const uint64_t *offsets, size_t n,
                     uint8_t *out);
int ronk_merkle_build_sha256(ronk_ctx *ctx, const uint8_t *data, uint64_t data_len, const uint64_t *offsets, size_t n,
                             uint8_t *nodes);
int ronk_merkle_build_sha256_host(ronk_ctx *ctx, const uint8_t *data, uint64_t data_len, const uint64_t *offsets,
                                  size_t n, uint8_t *nodes);
int ronk_merkle_proofs_sha256(ronk_ctx *ctx, const uint8_t *nodes, size_t n, const uint64_t *indices, size_t m,
                              uint8_t *siblings, uint8_t *sides);
int ronk_merkle_proofs_sha256_host(ronk_ctx *ctx, const uint8_t *nodes, size_t n, const uint64_t *indices, size_t m,
                                   uint8_t *siblings, uint8_t *sides);
int ronk_merkle_verify_sha256(ronk_ctx *ctx, const uint8_t *root, const uint8_t *data, uint64_t data_len,
                              const uint64_t *offsets, size_t m, const uint8_t *siblings, const uint8_t *sides,
                              uint32_t depth, uint8_t *ok);
int ronk_merkle_verify_sha256_host(ronk_ctx *ctx, const uint8_t *root, const uint8_t *data, uint64_t data_len,
                                   const uint64_t *offsets, size_t m, const uint8_t *siblings, const uint8_t *sides,
                                   uint32_t depth, uint8_t *ok);
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
