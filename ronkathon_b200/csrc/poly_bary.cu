// poly_bary.cu — Lagrange-basis rows on a coset s·H_n evaluated at many points and opened at one point, in O(n) per
// point (ronk_poly_lagrange_eval_u64, ronk_poly_lagrange_open_u64 and their _host twins, include/ronk_b200.h).
//
// Nodes x_j = s·ω^j, j < n, ω = g^((p-1)/n) of order exactly n, so Π_{m≠j}(x_j - x_m) = n·s^n / x_j and the barycentric
// weights are w_j = x_j / (n·s^n), with Z(X) = X^n - s^n:
//   L(x)  = Z(x) · Σ_j w_j y_j / (x - x_j)                      (the reference's l(x)·fold, mod.rs:382-415: 0 at a node)
//   q_j   = (y_j - v) / (x_j - z),  v = L(z)                     z off the nodes: the quotient (f - f(z)) / (X - z)
//   q_j   = (y_j - y_k) / (x_j - x_k),  q_k = -x_k^-1 Σ_{j≠k} x_j q_j     z = x_k (q has degree ≤ n - 2, so Σ w_j q_j = 0)
// The kernels never build an n-word node table: u_j = x_j^-1 = s^-1·ω^-j comes from the two O(√n)-word power tables of
// coset_table_kernel (ntt_kernel.cuh).  With c_ij = x_j / (x_i - x_j) = 1 / (x_i·u_j - 1), every coefficient is one
// inverse, and the inverses come from batch_invert (batch_inv.cuh), BI_K per thread.
#include "batch_inv.cuh"
#include "ntt_kernel.cuh"
#include "ronk_internal.h"

namespace ronk {

constexpr int BARY_THREADS = 256;
constexpr u32 BARY_WORDS = BARY_THREADS * BI_K;  // coefficients one CTA inverts at once (32 KiB of shared memory)
constexpr int BARY_MAX_M = 8;                     // points per pass over the rows (accumulators per lane)
constexpr u64 kBaryMaxWords = (u64)1 << 32;       // batch·n and batch·m bound

// u_j = x_j^-1 = sinv · lo[j mod 2^h] · hi[j >> h]: lo[i] = ω^-i, hi[i] = ω^-(i·2^h) in twiddle form, sinv plain.
struct BaryNodes {
  const u64* lo;
  const u64* hi;
  u32 h;
  u64 sinv;
};

template <class F>
RONK_DEV u64 bary_node_inv(const F& f, const BaryNodes& nd, u64 j) {
  return f.mul_tw(f.mul_tw(nd.sinv, nd.lo[j & (((u64)1 << nd.h) - 1)]), nd.hi[j >> nd.h]);
}

// Per-CTA partial sums over one tile of T = BARY_WORDS / M nodes and one group of M points (blockIdx.x = group·ntiles +
// tile): partial[((group·ntiles + tile)·batch + b)·M + i] = Σ_{j in tile} c_ij y_bj.  The CTA forms its M·T coefficients
// once (BI_K per thread, batch-inverted), then each warp streams whole rows of the tile through M accumulators and one
// shuffle reduction per row, so each y word is read once per group.
//   WEIGHT = false: c_ij = x_j / (x_i - x_j) = (x_i·u_j - 1)^-1 at the points xs[group·M + i] (x0 when xs is null); 0 at
//                   a node x_i = x_j and for the slots past m.
//   WEIGHT = true:  M = 1, c_j = x_j = u_j^-1 (the weighted sum Σ x_j q_j of an on-domain opening).
template <class F, int M, bool WEIGHT>
__global__ void __launch_bounds__(BARY_THREADS)
bary_partial_kernel(const F f, const u64* __restrict__ y, u64 n, u32 batch, const BaryNodes nd, const u64* __restrict__ xs,
                    u64 x0, u64 m, u32 ntiles, u64* __restrict__ partial) {
  static_assert(M == 1 || M == 2 || M == 4 || M == 8, "M");
  constexpr u32 T = BARY_WORDS / M;
  __shared__ u64 c[BARY_WORDS];  // c[i·T + jj]: the denominators, then their inverses in twiddle form
  const u32 t = threadIdx.x, tile = blockIdx.x % ntiles, grp = blockIdx.x / ntiles;
  const u64 j0 = (u64)tile * T, i0 = (u64)grp * M;
  const u64 one = 1 % f.modulus();
  u64 x[M];
#pragma unroll
  for (int i = 0; i < M; i++) x[i] = (WEIGHT || i0 + i >= m) ? 0 : (xs ? xs[i0 + i] : x0);
  // element k of this thread: e = t + 256k, point i = e / T (= k·M / BI_K, fixed per k), node jj = e mod T
#pragma unroll
  for (int k = 0; k < BI_K; k++) {
    const u32 e = t + BARY_THREADS * k, jj = e % T;
    const int i = k * M / BI_K;
    u64 d = 0;
    if (j0 + jj < n && (WEIGHT || i0 + i < m)) {
      const u64 u = bary_node_inv(f, nd, j0 + jj);
      d = WEIGHT ? u : f.sub(f.mul(x[i], u), one);
    }
    c[e] = d;
  }
  batch_invert<BI_K>(
      f, [&](int k) { return c[t + BARY_THREADS * k]; }, [&](int k, u64 v) { c[t + BARY_THREADS * k] = f.to_tw(v); });
  __syncthreads();
  const u32 lane = t & 31, lim = (u32)min((u64)T, n - j0);
  for (u32 b = t >> 5; b < batch; b += BARY_THREADS / 32) {
    const u64* row = y + (u64)b * n + j0;
    u64 acc[M];
#pragma unroll
    for (int i = 0; i < M; i++) acc[i] = 0;
#pragma unroll 4
    for (u32 q = lane; q < lim; q += 32) {
      const u64 v = row[q];
#pragma unroll
      for (int i = 0; i < M; i++) acc[i] = f.add(acc[i], f.mul_tw(v, c[i * T + q]));
    }
#pragma unroll
    for (int i = 0; i < M; i++)
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) acc[i] = f.add(acc[i], __shfl_down_sync(0xFFFFFFFFu, acc[i], off));
    if (lane == 0) {
      u64* dst = partial + (((u64)grp * ntiles + tile) * batch + b) * M;
#pragma unroll
      for (int i = 0; i < M; i++) dst[i] = acc[i];
    }
  }
}

// One warp per output: S = Σ_tile partial (lanes take the tiles in a fixed order, then a shuffle tree), then
//   WEIGHT = false: out[b·m + i] = S · Z(x_i) / (n·s^n) = S · (x_i^n · inv_nsn - ninv);
//   WEIGHT = true:  m = 1, out[b·n + k] = S · neg_zinv, k = *kidx (q_k = -x_k^-1 Σ_{j≠k} x_j q_j).
template <class F, bool WEIGHT>
__global__ void __launch_bounds__(256)
bary_finish_kernel(const F f, const u64* __restrict__ partial, u32 ntiles, u32 batch, u32 M, const u64* __restrict__ xs,
                   u64 x0, u64 m, u64 n, u64 inv_nsn, u64 ninv, const u64* __restrict__ kidx, u64 neg_zinv,
                   u64* __restrict__ out) {
  const u32 lane = threadIdx.x & 31;
  const u64 outputs = (u64)batch * m, wstride = (u64)gridDim.x * (blockDim.x >> 5);
  for (u64 o = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5; o < outputs; o += wstride) {
    const u64 b = o / m, i = o - b * m, grp = i / M, il = i - grp * M;
    u64 s = 0;
    for (u32 tl = lane; tl < ntiles; tl += 32) s = f.add(s, partial[((grp * ntiles + tl) * batch + b) * M + il]);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) s = f.add(s, __shfl_down_sync(0xFFFFFFFFu, s, off));
    if (lane) continue;
    if (WEIGHT) {
      out[b * n + *kidx] = f.mul(s, neg_zinv);
    } else {
      const u64 x = xs ? xs[i] : x0;
      out[o] = f.mul(s, f.sub(f.mul(field_pow(f, x, n), inv_nsn), ninv));
    }
  }
}

// z = x_k: *kidx = k, the one j < n with z·u_j = 1 (the host has checked (z/s)^n = 1).
template <class F>
__global__ void bary_locate_kernel(const F f, u64 n, const BaryNodes nd, u64 z, u64* __restrict__ kidx) {
  const u64 one = 1 % f.modulus();
  for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (u64)gridDim.x * blockDim.x)
    if (f.mul(z, bary_node_inv(f, nd, j)) == one) *kidx = j;
}

// The quotient over one tile of BARY_WORDS nodes: r_j = 1 / (x_j - z) = u_j / (1 - z·u_j), batch-inverted once per
// node and shared by every row, then q_bj = (y_bj - v_b)·r_j, one warp per row.
//   ON = false: v_b = values[b] (L_b(z), written by bary_finish_kernel before this launch).
//   ON = true:  z = x_k, k = *kidx: r_k = 0, so q_bk = 0 until bary_finish_kernel fills it; v_b = y_bk, which the CTA
//               holding node k also writes to values[b].
template <class F, bool ON>
__global__ void __launch_bounds__(BARY_THREADS)
bary_quotient_kernel(const F f, const u64* __restrict__ y, u64 n, u32 batch, const BaryNodes nd, u64 z,
                     const u64* __restrict__ kidx, u64* __restrict__ values, u64* __restrict__ q) {
  __shared__ u64 r[BARY_WORDS];
  const u32 t = threadIdx.x;
  const u64 j0 = (u64)blockIdx.x * BARY_WORDS, one = 1 % f.modulus();
#pragma unroll
  for (int k = 0; k < BI_K; k++) {
    const u64 j = j0 + t + BARY_THREADS * k;
    r[t + BARY_THREADS * k] = j < n ? f.sub(one, f.mul(z, bary_node_inv(f, nd, j))) : 0;
  }
  batch_invert<BI_K>(f, [&](int k) { return r[t + BARY_THREADS * k]; }, [&](int k, u64 v) {
    const u64 j = j0 + t + BARY_THREADS * k;
    r[t + BARY_THREADS * k] = v ? f.to_tw(f.mul(v, bary_node_inv(f, nd, j))) : 0;
  });
  __syncthreads();
  const u32 lane = t & 31, lim = (u32)min((u64)BARY_WORDS, n - j0);
  const u64 k = ON ? *kidx : 0;
  const bool holds_k = ON && k >= j0 && k - j0 < BARY_WORDS;
  for (u32 b = t >> 5; b < batch; b += BARY_THREADS / 32) {
    const u64* row = y + (u64)b * n;
    const u64 v = ON ? row[k] : values[b];
    if (holds_k && lane == 0) values[b] = v;
    u64* qrow = q + (u64)b * n + j0;
#pragma unroll 4
    for (u32 i = lane; i < lim; i += 32) qrow[i] = f.mul_tw(f.sub(row[j0 + i], v), r[i]);
  }
}

// ---- host side ---------------------------------------------------------------------------------------------------------

// Everything a call derives from (p, g, n, shift) on the host.
struct BaryPlan {
  u64 w;        // ω
  u32 log_n;    // ⌈log2 n⌉, the size the power tables cover
  u32 h;        // lo has 2^h words, hi 2^(log_n - h)
  u64 sinv, sn, inv_nsn, ninv;
  size_t table_words() const { return ((size_t)1 << h) + ((size_t)1 << (log_n - h)); }
};

// The checks shared by eval and open, in the order of ronk_poly_lagrange_eval_u64_host: null, modulus, g, n | p - 1,
// n's size, ω's order, shift.
static int bary_args(ronk_ctx* ctx, u64 p, u64 g, bool null_arg, u64 n, u32 batch, u64 shift, BaryPlan* pl) {
  if (!ctx || null_arg) return set_err(ctx, RONK_EINVAL, "null argument");
  RONK_TRY(validate_modulus(ctx, p));
  if (g == 0 || g >= p) return set_err(ctx, RONK_EINVAL, "generator out of range");
  if (n == 0 || (p - 1) % n != 0) return set_err(ctx, RONK_EINVAL, "n must divide p - 1 (Lagrange::new asserts)");
  if (n > kBaryMaxWords || (u64)batch * n > kBaryMaxWords)
    return set_err(ctx, RONK_EUNSUPPORTED, "more than 2^32 words of evaluations");
  pl->w = h_powmod(g, (p - 1) / n, p);
  if (!root_has_order(pl->w, n, p))
    return set_err(ctx, RONK_EINVAL, "Lagrange evaluate: ω has order below n, two nodes coincide (the reference divides by zero)");
  if (shift == 0 || shift >= p) return set_err(ctx, RONK_EINVAL, "shift must be in [1, p)");
  pl->log_n = log2_ceil(n);
  pl->h = (pl->log_n + 1) / 2;
  pl->sinv = h_powmod(shift, p - 2, p);
  pl->sn = h_powmod(shift, n, p);
  pl->inv_nsn = h_powmod(h_mulmod(n % p, pl->sn, p), p - 2, p);
  pl->ninv = h_powmod(n % p, p - 2, p);
  return RONK_OK;
}

// M: points per pass, the smallest of 1, 2, 4, 8 that holds m (8 past that).  Tiles: ⌈n / (BARY_WORDS / M)⌉.
static u32 bary_m_per_pass(u64 m) { return m > 4 ? BARY_MAX_M : m > 2 ? 4 : (u32)m; }

struct BaryGrid {
  u32 M, ntiles;
  u64 groups;
  size_t partial_words;
};

static int bary_grid(ronk_ctx* ctx, u64 n, u32 batch, u64 m, BaryGrid* gr) {
  gr->M = bary_m_per_pass(m);
  gr->ntiles = (u32)((n + BARY_WORDS / gr->M - 1) / (BARY_WORDS / gr->M));
  gr->groups = (m + gr->M - 1) / gr->M;
  if (gr->groups * gr->ntiles > 0x7FFFFFFFULL) return set_err(ctx, RONK_EUNSUPPORTED, "more than 2^31 - 1 tiles of (nodes, points)");
  const unsigned __int128 words = (unsigned __int128)gr->groups * gr->ntiles * batch * gr->M;
  if (words > ((unsigned __int128)1 << 40)) return set_err(ctx, RONK_ENOMEM, "partial sums beyond any device's memory");
  gr->partial_words = (size_t)words;
  return RONK_OK;
}

// The power tables of ω^-1 (coset_table_kernel, one launch) into tab.
template <class F>
static int bary_tables(ronk_ctx* ctx, const F& f, u64 p, const BaryPlan& pl, u64* tab, BaryNodes* nd) {
  const u32 words = (u32)pl.table_words();
  RONK_TRY(launch(ctx, "lagrange_table", coset_table_kernel<F>, (words + 255) / 256, 256, 0, false, f,
                  h_powmod(pl.w, p - 2, p), pl.h, pl.log_n, tab));
  *nd = BaryNodes{tab, tab + ((size_t)1 << pl.h), pl.h, pl.sinv};
  return RONK_OK;
}

// The partial and finish launches of an evaluation at m points (xs, or x0 when xs is null) into out.
template <class F>
static int bary_eval_launch(ronk_ctx* ctx, const F& f, const BaryPlan& pl, const BaryNodes& nd, const u64* y, u64 n,
                            u32 batch, const u64* xs, u64 x0, u64 m, const BaryGrid& gr, u64* partial, u64* out) {
  auto part = [&](auto kernel) {
    return launch(ctx, "lagrange_partial", kernel, (u32)(gr.groups * gr.ntiles), BARY_THREADS, 0, false, f, y, n, batch, nd,
                  xs, x0, m, gr.ntiles, partial);
  };
  switch (gr.M) {
    case 1: RONK_TRY(part(bary_partial_kernel<F, 1, false>)); break;
    case 2: RONK_TRY(part(bary_partial_kernel<F, 2, false>)); break;
    case 4: RONK_TRY(part(bary_partial_kernel<F, 4, false>)); break;
    default: RONK_TRY(part(bary_partial_kernel<F, 8, false>)); break;
  }
  return launch(ctx, "lagrange_finish", bary_finish_kernel<F, false>, grid_for(ctx, (u64)batch * m * 32, 256), 256, 0, false,
                f, partial, gr.ntiles, batch, gr.M, xs, x0, m, n, pl.inv_nsn, pl.ninv, nullptr, (u64)0, out);
}

// Every check of an evaluation, in the order include/ronk_b200.h states (xs is not read).
static int lagrange_eval_args(ronk_ctx* ctx, u64 p, u64 g, const u64* evals, u64 n, u32 batch, u64 shift, const u64* xs,
                              size_t m, const u64* out, BaryPlan* pl) {
  RONK_TRY(bary_args(ctx, p, g, !evals || (m && (!xs || !out)), n, batch, shift, pl));
  if ((u64)batch * m > kBaryMaxWords) return set_err(ctx, RONK_EUNSUPPORTED, "more than 2^32 words of output");
  if (overlaps(out, (size_t)batch * m, evals, (size_t)batch * n) || overlaps(out, (size_t)batch * m, xs, m))
    return set_err(ctx, RONK_EINVAL, "out may not overlap evals or xs");
  return RONK_OK;
}

static int lagrange_eval_device(ronk_ctx* ctx, u64 p, u64 g, const u64* evals, u64 n, u32 batch, u64 shift, const u64* xs,
                                size_t m, u64* out) {
  BaryPlan pl;
  RONK_TRY(lagrange_eval_args(ctx, p, g, evals, n, batch, shift, xs, m, out, &pl));
  if (batch == 0 || m == 0) return RONK_OK;
  BaryGrid gr;
  RONK_TRY(bary_grid(ctx, n, batch, m, &gr));
  Frame fr(ctx);
  u64 *tab = nullptr, *partial = nullptr;
  RONK_TRY(fr.take(&tab, pl.table_words()));
  RONK_TRY(fr.take(&partial, gr.partial_words));
  return with_field(ctx, p, g, false, [&](const auto& f) {
    BaryNodes nd;
    RONK_TRY(bary_tables(ctx, f, p, pl, tab, &nd));
    return bary_eval_launch(ctx, f, pl, nd, evals, n, batch, xs, 0, m, gr, partial, out);
  });
}

// Every check of an opening, in the order include/ronk_b200.h states.
static int lagrange_open_args(ronk_ctx* ctx, u64 p, u64 g, const u64* evals, u64 n, u32 batch, u64 shift, u64 z,
                              const u64* values, const u64* quotient, BaryPlan* pl) {
  RONK_TRY(bary_args(ctx, p, g, !evals || !values || !quotient, n, batch, shift, pl));
  if (z >= p) return set_err(ctx, RONK_EINVAL, "z must be canonical (< p)");
  const size_t rows = (size_t)batch * n;
  if (overlaps(values, batch, evals, rows) || overlaps(quotient, rows, evals, rows) || overlaps(values, batch, quotient, rows))
    return set_err(ctx, RONK_EINVAL, "values and quotient may not overlap evals or each other");
  return RONK_OK;
}

static int lagrange_open_device(ronk_ctx* ctx, u64 p, u64 g, const u64* evals, u64 n, u32 batch, u64 shift, u64 z,
                                u64* values, u64* quotient) {
  BaryPlan pl;
  RONK_TRY(lagrange_open_args(ctx, p, g, evals, n, batch, shift, z, values, quotient, &pl));
  if (batch == 0) return RONK_OK;
  // z ∈ s·H_n  ⇔  (z / s)^n = 1; which node it is, the device finds
  const bool on = h_powmod(h_mulmod(z, pl.sinv, p), n, p) == 1;
  BaryGrid gr;
  RONK_TRY(bary_grid(ctx, n, batch, 1, &gr));
  const u32 qtiles = (u32)((n + BARY_WORDS - 1) / BARY_WORDS);
  Frame fr(ctx);
  u64 *tab = nullptr, *partial = nullptr, *kidx = nullptr;
  RONK_TRY(fr.take(&tab, pl.table_words()));
  RONK_TRY(fr.take(&partial, gr.partial_words));
  RONK_TRY(fr.take(&kidx, 1));
  return with_field(ctx, p, g, false, [&](const auto& f) {
    using F = std::decay_t<decltype(f)>;
    BaryNodes nd;
    RONK_TRY(bary_tables(ctx, f, p, pl, tab, &nd));
    if (!on) {
      RONK_TRY(bary_eval_launch(ctx, f, pl, nd, evals, n, batch, nullptr, z, 1, gr, partial, values));
      return launch(ctx, "lagrange_quotient", bary_quotient_kernel<F, false>, qtiles, BARY_THREADS, 0, false, f, evals, n,
                    batch, nd, z, (const u64*)nullptr, values, quotient);
    }
    RONK_TRY(launch(ctx, "lagrange_locate", bary_locate_kernel<F>, grid_for(ctx, n, 256), 256, 0, false, f, n, nd, z, kidx));
    RONK_TRY(launch(ctx, "lagrange_quotient", bary_quotient_kernel<F, true>, qtiles, BARY_THREADS, 0, false, f, evals, n,
                    batch, nd, z, (const u64*)kidx, values, quotient));
    RONK_TRY(launch(ctx, "lagrange_partial", bary_partial_kernel<F, 1, true>, gr.ntiles, BARY_THREADS, 0, false, f,
                    (const u64*)quotient, n, batch, nd, (const u64*)nullptr, (u64)0, (u64)1, gr.ntiles, partial));
    const u64 neg_zinv = (p - h_powmod(z, p - 2, p)) % p;
    return launch(ctx, "lagrange_finish", bary_finish_kernel<F, true>, grid_for(ctx, (u64)batch * 32, 256), 256, 0, false, f,
                  (const u64*)partial, gr.ntiles, batch, (u32)1, (const u64*)nullptr, (u64)0, (u64)1, n, (u64)0, (u64)0,
                  (const u64*)kidx, neg_zinv, quotient);
  });
}

}  // namespace ronk

using namespace ronk;

extern "C" {

int ronk_poly_lagrange_eval_u64(ronk_ctx* ctx, uint64_t p, uint64_t g, const uint64_t* evals, uint64_t n, uint32_t batch,
                                uint64_t shift, const uint64_t* xs, size_t m, uint64_t* out) {
  ronk::DeviceGuard _dg(ctx);
  return lagrange_eval_device(ctx, p, g, (const u64*)evals, n, batch, shift, (const u64*)xs, m, (u64*)out);
}

int ronk_poly_lagrange_open_u64(ronk_ctx* ctx, uint64_t p, uint64_t g, const uint64_t* evals, uint64_t n, uint32_t batch,
                                uint64_t shift, uint64_t z, uint64_t* values, uint64_t* quotient) {
  ronk::DeviceGuard _dg(ctx);
  return lagrange_open_device(ctx, p, g, (const u64*)evals, n, batch, shift, z, (u64*)values, (u64*)quotient);
}

// The device function's checks run first on the host buffers, so that a refused call copies nothing; then the points'.
int ronk_poly_lagrange_eval_batch_u64_host(ronk_ctx* ctx, uint64_t p, uint64_t g, const uint64_t* evals, uint64_t n,
                                           uint32_t batch, uint64_t shift, const uint64_t* xs, size_t m, uint64_t* out) {
  ronk::DeviceGuard _dg(ctx);
  BaryPlan pl;
  RONK_TRY(lagrange_eval_args(ctx, p, g, (const u64*)evals, n, batch, shift, (const u64*)xs, m, (const u64*)out, &pl));
  for (size_t i = 0; i < m; i++)
    if (xs[i] >= p) return set_err(ctx, RONK_EINVAL, "non-canonical point");
  if (batch == 0 || m == 0) return RONK_OK;
  Staged s[] = {{(size_t)batch * n * 8, evals}, {m * 8, xs}, {(size_t)batch * m * 8, nullptr, out}};
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  return stage_out(ctx, lagrange_eval_device(ctx, p, g, s[0].dev, n, batch, shift, s[1].dev, m, s[2].dev), s);
}

int ronk_poly_lagrange_open_u64_host(ronk_ctx* ctx, uint64_t p, uint64_t g, const uint64_t* evals, uint64_t n, uint32_t batch,
                                     uint64_t shift, uint64_t z, uint64_t* values, uint64_t* quotient) {
  ronk::DeviceGuard _dg(ctx);
  BaryPlan pl;
  RONK_TRY(lagrange_open_args(ctx, p, g, (const u64*)evals, n, batch, shift, z, (const u64*)values, (const u64*)quotient, &pl));
  if (batch == 0) return RONK_OK;
  const size_t rows = (size_t)batch * n;
  Staged s[] = {{rows * 8, evals}, {(size_t)batch * 8, nullptr, values}, {rows * 8, nullptr, quotient}};
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  return stage_out(ctx, lagrange_open_device(ctx, p, g, s[0].dev, n, batch, shift, z, s[1].dev, s[2].dev), s);
}

}  // extern "C"
