// ntt_any.cu — forward and inverse transforms of ANY length n dividing p - 1 (Polynomial::dft, src/polynomial/mod.rs:240-258,
// and its inverse), in O(n log n) on the power-of-two transforms of ntt.cu by Bluestein's algorithm.
//
// With jk = C(j+k, 2) - C(j, 2) - C(k, 2) and ω = g^((p-1)/n) (only ωⁿ = 1 is needed, so every n | p - 1 works, even n at
// the full two-adicity):
//   X_k = ω^-C(k,2) · Σ_j u_j · v_(j+k),   u_j = a_j · ω^-C(j,2),   v_t = ω^C(t,2), t ≤ 2n - 2.
// The correlation is one cyclic convolution of N = 2^⌈log2(2n - 1)⌉ points.  v is stored reflected, r_s = v_((-s) mod N),
// zeros in the gap, so that u stays in natural order and X_k = ω^-C(k,2) · (u ⊛ r)[(-k) mod N]: the wrap of the 3n - 2
// linear terms never reaches the n indices read.  The inverse is the forward transform read backwards,
// X'_k = n^-1 · X_((n-k) mod n), so one spectrum R = NTT_N(r) per (p, g, n) serves both directions; it is cached on the
// context.  Per call: anyntt_chirp_in (data → B×N scratch), a batched forward transform with R multiplied in by its
// store phase, the batched inverse in place, anyntt_chirp_out (scratch → data).
// tests/test_anyntt_model.py is a Python model of the same index arithmetic.
#include "ntt_kernel.cuh"
#include "ronk_internal.h"

namespace ronk {

constexpr int AN_THREADS = 256;  // thread i of a block takes t = base + i + 256·r, r < AN_RUN: coalesced and stepped
constexpr int AN_RUN = 32;
constexpr u64 AN_CHUNK = (u64)AN_THREADS * AN_RUN;

template <class F>
RONK_DEV u64 pow_tw(const F& f, u64 b_tw, u64 e) {  // b^e, twiddle form in and out
  u64 r = f.to_tw(1 % f.modulus());
  while (e) {
    if (e & 1) r = f.mul_tw(r, b_tw);
    b_tw = f.mul_tw(b_tw, b_tw);
    e >>= 1;
  }
  return r;
}

// scale · w^C(t,2) along t, t + S, t + 2S, … (S = AN_THREADS), twiddle form, two multiplies per step:
// C(t+S, 2) - C(t, 2) = S·t + C(S, 2), so z ← z·e, e ← e·w^(S²) with e = w^(S·t + C(S, 2)).  Exponents are reduced
// mod n (wⁿ = 1); t < 2^26 keeps t(t - 1) below 2^52.
template <class F>
struct Chirp {
  u64 z, e, step;
  RONK_DEV Chirp(const F& f, u64 w_tw, u64 n, u64 t, u64 scale_tw) {
    constexpr u64 S = AN_THREADS;
    z = f.mul_tw(pow_tw(f, w_tw, (t * (t - 1) / 2) % n), scale_tw);
    e = pow_tw(f, w_tw, (S * t + S * (S - 1) / 2) % n);
    step = pow_tw(f, w_tw, (S * S) % n);
  }
  RONK_DEV u64 next(const F& f) {
    const u64 v = z;
    z = f.mul_tw(z, e);
    e = f.mul_tw(e, step);
    return v;
  }
};

// Block → (transform b, first index of its chunk); `len` indices per transform, chunks of AN_CHUNK.
RONK_DEV void an_block(u64 len, u64* b, u64* t0) {
  const u64 chunks = (len + AN_CHUNK - 1) / AN_CHUNK;
  *b = blockIdx.x / chunks;
  *t0 = (blockIdx.x % chunks) * AN_CHUNK + threadIdx.x;
}

// W[b·N + j] = a[b·n + j] · w^C(j,2) for j < n, 0 for n ≤ j < N   (w = ω^-1)
template <class F>
__global__ void __launch_bounds__(AN_THREADS)
anyntt_chirp_in_kernel(const F f, const u64* __restrict__ a, u64 n, u64 N, u64 w_tw, u64* __restrict__ W) {
  u64 b, t;
  an_block(N, &b, &t);
  const u64* src = a + b * n;
  u64* dst = W + b * N;
  if (t >= n) {
    for (int r = 0; r < AN_RUN && t < N; r++, t += AN_THREADS) dst[t] = 0;
    return;
  }
  Chirp<F> c(f, w_tw, n, t, f.to_tw(1 % f.modulus()));
  for (int r = 0; r < AN_RUN && t < N; r++, t += AN_THREADS) {
    const u64 z = c.next(f);
    dst[t] = t < n ? f.mul_tw(src[t], z) : 0ULL;
  }
}

// out[b·n + k] = scale · w^C(t,2) · W[b·N + (N - t) mod N] with k = t (forward) or k = (n - t) mod n (REV: the inverse, scale =
// n^-1).  w = ω^-1.  With w = 1 and N = n it is the reversal and scaling alone.
template <class F, bool REV>
__global__ void __launch_bounds__(AN_THREADS)
anyntt_chirp_out_kernel(const F f, const u64* __restrict__ W, u64 n, u64 N, u64 w_tw, u64 scale_tw, u64* __restrict__ out) {
  u64 b, t;
  an_block(n, &b, &t);
  if (t >= n) return;
  const u64* src = W + b * N;
  u64* dst = out + b * n;
  Chirp<F> c(f, w_tw, n, t, scale_tw);
  for (int r = 0; r < AN_RUN && t < n; r++, t += AN_THREADS) {
    const u64 z = c.next(f);
    const u64 v = f.mul_tw(src[t ? N - t : 0], z);
    dst[REV ? (t ? n - t : 0) : t] = v;
  }
}

// r[(N - t) mod N] = w^C(t,2), t ≤ 2n - 2 (w = ω; the gap is zeroed before)
template <class F>
__global__ void __launch_bounds__(AN_THREADS)
anyntt_chirp_table_kernel(const F f, u64 n, u64 N, u64 w_tw, u64* __restrict__ r) {
  u64 b, t;
  const u64 len = 2 * n - 1;
  an_block(len, &b, &t);
  if (t >= len) return;
  Chirp<F> c(f, w_tw, n, t, f.to_tw(1 % f.modulus()));
  for (int q = 0; q < AN_RUN && t < len; q++, t += AN_THREADS) {
    const u64 z = c.next(f);
    r[t ? N - t : 0] = f.mul_tw(1 % f.modulus(), z);  // plain residue: the transform's multiplier is plain
  }
}

// Which kernels run a transform of n points (anyntt_path, AnyNttPath in ronk_internal.h): the power-of-two transform;
// Bluestein when its convolution of N = 2^⌈log2(2n - 1)⌉ ≤ 2^26 points divides p - 1 and n reaches the crossover; the
// literal evaluation at n roots of unity (ronk_dft_u64's kernels) up to kAnyNttLiteralMax; else nothing.
constexpr u64 kAnyNttLiteralMax = (u64)1 << 17;
// Smallest n that takes Bluestein where it fits: tools/anyntt_timing.py on an H100 80GB HBM3 at 700 W (DESIGN.md §5), the
// smallest n from which Bluestein won at every larger n measured (4080: 0.081 vs 0.081 ms; 3840: 0.082 vs 0.077).
// RONK_ANYNTT_MIN overrides it.
constexpr u64 kAnyNttMin = 4080;

static AnyNttPath anyntt_path(const ronk_ctx* ctx, u64 p, u64 n) {
  if ((n & (n - 1)) == 0) return AN_POW2;
  const u32 log_N = log2_ceil(2 * n - 1);
  const u64 min_n = ctx->tune.anyntt_min >= 0 ? (u64)ctx->tune.anyntt_min : kAnyNttMin;
  if (pow2_fits(p, log_N) && n >= min_n) return AN_BLUESTEIN;
  if (n <= kAnyNttLiteralMax) return AN_LITERAL;
  return AN_NONE;
}

// Checks of both variants; *path set on RONK_OK.
int anyntt_args(ronk_ctx* ctx, u64 p, u64 g, const void* data, u64 n, AnyNttPath* path) {
  if (!ctx || !data) return set_err(ctx, RONK_EINVAL, "null argument");
  RONK_TRY(validate_modulus(ctx, p));
  if (g == 0 || g >= p) return set_err(ctx, RONK_EINVAL, "generator out of range");
  if (n == 0 || (p - 1) % n != 0) return set_err(ctx, RONK_EINVAL, "n must divide p - 1 (no primitive n-th root of unity)");
  *path = anyntt_path(ctx, p, n);
  if (*path == AN_NONE)
    return set_err(ctx, RONK_EUNSUPPORTED, "n off the Bluestein envelope (N = 2^⌈log2(2n-1)⌉ ≤ 2^26 dividing p - 1) and above 2^17");
  if (*path == AN_POW2 && n > ((u64)1 << 26)) return set_err(ctx, RONK_EUNSUPPORTED, "log_n > 26 not supported");
  return RONK_OK;
}

static unsigned an_grid(u64 len, u32 batch) { return (unsigned)((len + AN_CHUNK - 1) / AN_CHUNK * batch); }

// R = NTT_N(r) of (p, g, n), built on first use on ctx->stream and kept until ronk_ctx_destroy (N words).
static int anyntt_spectrum(ronk_ctx* ctx, u64 p, u64 g, u64 n, u32 log_N, const u64** out) {
  DevBuf<u64>& R = ctx->anyntt_spec[std::make_tuple((uint64_t)p, (uint64_t)g, (uint64_t)n)];  // empty until built
  const u64 N = (u64)1 << log_N;
  if (!R) RONK_TRY(build_table(ctx, &R, N, [&](u64* r) {
    RONK_CUDA(ctx, cudaMemsetAsync(r, 0, N * sizeof(u64), ctx->stream));
    RONK_TRY(with_field(ctx, p, 0, false, [&](const auto& f) {
      using F = std::decay_t<decltype(f)>;
      return launch(ctx, "anyntt_chirp_table", anyntt_chirp_table_kernel<F>, an_grid(2 * n - 1, 1), AN_THREADS, 0, false, f, n,
                    N, f.to_tw(h_powmod(g, (p - 1) / n, p)), r);
    }));
    return ntt_device(ctx, p, g, r, nullptr, log_N, 1, 0);
  }));
  *out = R.get();
  return RONK_OK;
}

static int anyntt_bluestein(ronk_ctx* ctx, u64 p, u64 g, u64* data, u64 n, u32 batch, int inverse) {
  const u32 log_N = log2_ceil(2 * n - 1);
  const u64 N = (u64)1 << log_N;
  if ((u64)an_grid(N, 1) * batch > 0x7FFFFFFFULL) return set_err(ctx, RONK_EUNSUPPORTED, "batch too large");
  const u64* R = nullptr;
  RONK_TRY(anyntt_spectrum(ctx, p, g, n, log_N, &R));
  Frame fr(ctx);
  u64* W = nullptr;
  RONK_TRY(fr.take(&W, (size_t)batch * N));
  const u64 winv = h_powmod(h_powmod(g, (p - 1) / n, p), p - 2, p);
  RONK_TRY(with_field(ctx, p, 0, false, [&](const auto& f) {
    using F = std::decay_t<decltype(f)>;
    return launch(ctx, "anyntt_chirp_in", anyntt_chirp_in_kernel<F>, an_grid(N, batch), AN_THREADS, 0, false, f, data, n, N,
                  f.to_tw(winv), W);
  }));
  RONK_TRY(ntt_device_shared_mul(ctx, p, g, W, W, R, log_N, batch));
  RONK_TRY(ntt_device(ctx, p, g, W, nullptr, log_N, batch, 1));
  return with_field(ctx, p, 0, false, [&](const auto& f) {
    using F = std::decay_t<decltype(f)>;
    const unsigned grid = an_grid(n, batch);
    if (inverse)
      return launch(ctx, "anyntt_chirp_out", anyntt_chirp_out_kernel<F, true>, grid, AN_THREADS, 0, false, f, W, n, N,
                    f.to_tw(winv), f.to_tw(h_powmod(n % p, p - 2, p)), data);
    return launch(ctx, "anyntt_chirp_out", anyntt_chirp_out_kernel<F, false>, grid, AN_THREADS, 0, false, f, W, n, N,
                  f.to_tw(winv), f.to_tw(1), data);
  });
}

// ronk_dft_u64's kernels (pow_table + poly_eval per transform) into scratch, then a copy back, or for the inverse the
// reversal and the n^-1 scaling (anyntt_chirp_out with w = 1).
static int anyntt_literal(ronk_ctx* ctx, u64 p, u64 g, u64* data, u64 n, u32 batch, int inverse) {
  Frame fr(ctx);
  u64 *nodes = nullptr, *X = nullptr;
  RONK_TRY(fr.take(&nodes, n));
  RONK_TRY(fr.take(&X, (size_t)batch * n));
  RONK_TRY(roots_table(ctx, p, g, n, nodes));
  for (u32 b = 0; b < batch; b++) RONK_TRY(poly_eval_device(ctx, p, data + (size_t)b * n, n, nodes, n, X + (size_t)b * n));
  if (!inverse) {
    RONK_CUDA(ctx, cudaMemcpyAsync(data, X, (size_t)batch * n * sizeof(u64), cudaMemcpyDeviceToDevice, ctx->stream));
    return RONK_OK;
  }
  if ((u64)an_grid(n, 1) * batch > 0x7FFFFFFFULL) return set_err(ctx, RONK_EUNSUPPORTED, "batch too large");
  return with_field(ctx, p, 0, false, [&](const auto& f) {
    using F = std::decay_t<decltype(f)>;
    return launch(ctx, "anyntt_chirp_out", anyntt_chirp_out_kernel<F, false>, an_grid(n, batch), AN_THREADS, 0, false, f, X, n,
                  n, f.to_tw(1), f.to_tw(h_powmod(n % p, p - 2, p)), data);
  });
}

int anyntt_device(ronk_ctx* ctx, u64 p, u64 g, u64* data, u64 n, u32 batch, int inverse) {
  AnyNttPath path;
  RONK_TRY(anyntt_args(ctx, p, g, data, n, &path));
  if (batch == 0) return RONK_OK;
  switch (path) {
    case AN_POW2: return ntt_device(ctx, p, g, data, nullptr, log2_ceil(n), batch, inverse);
    case AN_BLUESTEIN: return anyntt_bluestein(ctx, p, g, data, n, batch, inverse);
    default: return anyntt_literal(ctx, p, g, data, n, batch, inverse);
  }
}

}  // namespace ronk

using namespace ronk;

extern "C" int ronk_ntt_any_u64(ronk_ctx* ctx, uint64_t p, uint64_t g, uint64_t* data, uint64_t n, uint32_t batch,
                                int inverse) {
  ronk::DeviceGuard _dg(ctx);
  return anyntt_device(ctx, p, g, (u64*)data, n, batch, inverse);
}

extern "C" int ronk_ntt_any_u64_host(ronk_ctx* ctx, uint64_t p, uint64_t g, uint64_t* host_data, uint64_t n, uint32_t batch,
                                     int inverse) {
  ronk::DeviceGuard _dg(ctx);
  AnyNttPath path;
  RONK_TRY(anyntt_args(ctx, p, g, host_data, n, &path));  // before staging: an unsupported n is refused before its copy
  if (batch == 0) return RONK_OK;
  Staged s[] = {{(size_t)batch * n * 8, host_data, host_data}};
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  return stage_out(ctx, anyntt_device(ctx, p, g, s[0].dev, n, batch, inverse), s);
}
