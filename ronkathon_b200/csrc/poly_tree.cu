// poly_tree.cu — multipoint evaluation (evaluate, src/polynomial/mod.rs:133-139, at many points: shamir/mod.rs:53-58) and
// interpolation (Message::decode, codes/reed_solomon.rs:55-107) in O(n log² n) on a subproduct tree, built on the
// batched natural-order transforms of ntt.cu and the Newton inversion of poly_div.cu.
//
// Tree over k points, K = ⌈log2 k⌉, N = 2^K leaves X - x_i; the leaves past k are the constant 1, so the nodes on the
// right spine have a degree below 2^j and every other node at level j has degree 2^j.  Node i of level j is stored
// explicitly (monic, zeros above its degree) in 2^j + 1 words; levels TREE_B … K are kept, the ones below are rebuilt in
// shared memory by the kernels that need them (one CTA per 2^TREE_B leaves).
//   up (product):  level j → j + 1, D = 2^(j+1): both children spread into D-word slots, one batched forward transform
//                  per side (the point-wise product fused into the second), one batched inverse; a parent of two full
//                  children has degree D, whose X^D term wrapped onto X^0: subtract 1 there and set word D to 1.
//   down (scaled remainder tree, after Bernstein and Bostan–Lecerf–Schost): node v of degree δ carries
//                  ρ_v[u] = coefficient of X^(u-δ) in (f mod M_v)/M_v, u < δ.  Root: with h = rev_d(f)·rev_k(M)^-1
//                  mod y^d (one Newton inversion), ρ[u] = h[d-1-u] for u < min(d, k), 0 above.  Children: ρ_L is
//                  words [δ_R, δ) of M_R·ρ and ρ_R words [δ_L, δ) of M_L·ρ; a D-point cyclic product gives both,
//                  because its wrap only reaches words below δ_R (δ_L).  Bottom: f mod M = the polynomial part of
//                  M·ρ·X^-δ, Horner-evaluated at the subtree's points.
//   interpolation: c_i = y_i / M'(x_i) (M' evaluated down the same tree), then r_parent = r_L·M_R + r_R·M_L up the tree,
//                  r_leaf = c_i; degrees stay below D, so nothing wraps.
// tests/test_multipoint_model.py is a Python model of the same index arithmetic.
#include <algorithm>
#include <utility>

#include "ronk_internal.h"

namespace ronk {

constexpr u32 TREE_B = 6;                  // levels built in shared memory
constexpr u32 TREE_NL = 1u << TREE_B;      // leaves per CTA (kTreeLeaves)
static_assert(TREE_NL == kTreeLeaves, "kTreeLeaves");

// Degree of node i at level j of a tree over k leaves.
RONK_HD size_t node_deg(size_t k, u32 j, size_t i) {
  const size_t lo = i << j, w = (size_t)1 << j;
  return lo >= k ? 0 : (k - lo < w ? k - lo : w);
}

// The product of the 2^lb leaves of subtree blockIdx.x, schoolbook level by level in shared memory (nodes of level j
// at stride 2^j + 1), to out[blockIdx.x·(2^lb + 1) …].  With cs: also the interpolation sums r (leaf r = cs[i], level
// j at stride 2^j) to rout[blockIdx.x·2^lb …].
template <class F, bool INTERP>
__global__ void __launch_bounds__(128)
tree_leaves_kernel(const F f, const u64* __restrict__ xs, const u64* __restrict__ cs, size_t k, u32 lb, u64* __restrict__ out,
                   u64* __restrict__ rout) {
  __shared__ u64 m[2][2 * TREE_NL];
  __shared__ u64 r[2][TREE_NL];
  const u32 nl = 1u << lb, t0 = threadIdx.x, nt = blockDim.x;
  const size_t base = (size_t)blockIdx.x << lb;
  const u64 one = 1 % f.modulus();
  for (u32 i = t0; i < nl; i += nt) {
    const bool live = base + i < k;
    m[0][2 * i] = live ? f.neg(xs[base + i]) : one;
    m[0][2 * i + 1] = live ? one : 0ULL;
    if (INTERP) r[0][i] = live ? cs[base + i] : 0ULL;
  }
  __syncthreads();
  u32 c = 0;
  for (u32 j = 0; j < lb; j++) {
    const u32 w = 1u << j, sc = w + 1, sp = 2 * w + 1, np = nl >> (j + 1);
    for (u32 t = t0; t < np * sp; t += nt) {
      const u32 i = t / sp, e = t % sp;
      const u64* L = &m[c][2 * i * sc];
      const u64* R = L + sc;
      const u32 lo = e > w ? e - w : 0, hi = e < w ? e : w;
      u64 acc = 0;
      for (u32 a = lo; a <= hi; a++) acc = f.add(acc, f.mul(L[a], R[e - a]));
      m[c ^ 1][i * sp + e] = acc;
    }
    if (INTERP) {  // r_L·M_R + r_R·M_L, degree < 2w
      for (u32 t = t0; t < np * 2 * w; t += nt) {
        const u32 i = t / (2 * w), e = t % (2 * w);
        const u64* rL = &r[c][2 * i * w];
        const u64* rR = rL + w;
        const u64* ML = &m[c][2 * i * sc];
        const u64* MR = ML + sc;
        const u32 lo = e > w ? e - w : 0, hi = e < w ? e : w - 1;
        u64 acc = 0;
        for (u32 a = lo; a <= hi; a++) acc = f.add(acc, f.add(f.mul(rL[a], MR[e - a]), f.mul(rR[a], ML[e - a])));
        r[c ^ 1][i * 2 * w + e] = acc;
      }
    }
    __syncthreads();
    c ^= 1;
  }
  for (u32 e = t0; e <= nl; e += nt) out[(size_t)blockIdx.x * (nl + 1) + e] = m[c][e];
  if (INTERP)
    for (u32 e = t0; e < nl; e += nt) rout[(size_t)blockIdx.x * nl + e] = r[c][e];
}

// A[i·D + t] = src[2i·stride + t], B[i·D + t] = src[(2i + 1)·stride + t] for t < len, zero up to D, i < P.
__global__ void tree_spread_kernel(const u64* __restrict__ src, size_t stride, size_t len, u32 log_d, size_t P,
                                   u64* __restrict__ A, u64* __restrict__ B) {
  const size_t D = (size_t)1 << log_d, n = P << log_d, step = (size_t)gridDim.x * blockDim.x;
  for (size_t x = (size_t)blockIdx.x * blockDim.x + threadIdx.x; x < n; x += step) {
    const size_t i = x >> log_d, t = x & (D - 1);
    A[x] = t < len ? src[2 * i * stride + t] : 0ULL;
    B[x] = t < len ? src[(2 * i + 1) * stride + t] : 0ULL;
  }
}

// Parents of level log_d (D-word cyclic products in C) to their (D + 1)-word slots, with the wrap correction.
template <class F>
__global__ void tree_fix_kernel(const F f, const u64* __restrict__ C, size_t k, u32 log_d, size_t P, u64* __restrict__ dst) {
  const size_t D = (size_t)1 << log_d, n = P * (D + 1), step = (size_t)gridDim.x * blockDim.x;
  const u64 one = 1 % f.modulus();
  for (size_t x = (size_t)blockIdx.x * blockDim.x + threadIdx.x; x < n; x += step) {
    const size_t i = x / (D + 1), t = x % (D + 1);
    const bool full = node_deg(k, log_d, i) == D;
    u64 v = t < D ? C[i * D + t] : (full ? one : 0ULL);
    if (t == 0 && full) v = f.sub(v, one);
    dst[x] = v;
  }
}

// Children of level j from their parents' products A = M_L·ρ, B = M_R·ρ (D = 2^(j+1) words each): ρ_L = B[δ_R, δ),
// ρ_R = A[δ_L, δ), zero-filled to 2^j words.
__global__ void tree_extract_kernel(const u64* __restrict__ A, const u64* __restrict__ B, size_t k, u32 j, size_t nchild,
                                    u64* __restrict__ dst) {
  const size_t w = (size_t)1 << j, n = nchild << j, step = (size_t)gridDim.x * blockDim.x;
  for (size_t x = (size_t)blockIdx.x * blockDim.x + threadIdx.x; x < n; x += step) {
    const size_t c = x >> j, u = x & (w - 1), i = c >> 1;
    const size_t dl = node_deg(k, j, 2 * i), dr = node_deg(k, j, 2 * i + 1);
    dst[x] = (c & 1) ? (u < dr ? A[2 * i * w + dl + u] : 0ULL) : (u < dl ? B[2 * i * w + dr + u] : 0ULL);
  }
}

// out[i] = (i + 1)·M[i + 1], i < k
template <class F>
__global__ void tree_deriv_kernel(const F f, const u64* __restrict__ M, size_t k, u64* __restrict__ out) {
  const size_t step = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < k; i += step)
    out[i] = f.mul((u64)((i + 1) % f.modulus()), M[i + 1]);
}

// Subtree blockIdx.x at level lb: r = f mod M = polynomial part of M·ρ·X^-δ, then out[i] = r(xs[i]) for its points.
template <class F>
__global__ void __launch_bounds__(TREE_NL)
tree_eval_leaves_kernel(const F f, const u64* __restrict__ M, const u64* __restrict__ R, const u64* __restrict__ xs, size_t k,
                        u32 lb, u64* __restrict__ out) {
  __shared__ u64 sM[TREE_NL + 1], sR[TREE_NL], sr[TREE_NL];
  const u32 w = 1u << lb, t0 = threadIdx.x, nt = blockDim.x;
  const size_t s = blockIdx.x, base = s << lb;
  const u32 dl = (u32)node_deg(k, lb, s);
  for (u32 e = t0; e <= w; e += nt) sM[e] = M[s * (w + 1) + e];
  for (u32 u = t0; u < w; u += nt) sR[u] = R[s * w + u];
  __syncthreads();
  for (u32 e = t0; e < dl; e += nt) {
    u64 acc = 0;
    for (u32 u = e; u < dl; u++) acc = f.add(acc, f.mul(sM[e + dl - u], sR[u]));
    sr[e] = acc;
  }
  __syncthreads();
  for (u32 i = t0; i < dl; i += nt) {
    const u64 x = xs[base + i];
    u64 acc = 0;
    for (u32 e = dl; e-- > 0;) acc = f.add(f.mul(acc, x), sr[e]);
    out[base + i] = acc;
  }
}

// Shape of the tree over k leaves and its place in the scratch of the function that builds it: the stored levels
// lb … K, then four N-word buffers.
struct Tree {
  size_t k = 0, N = 1;
  u32 K = 0, lb = 0;
  size_t off[27] = {};  // first word of level j, j in [lb, K]
  size_t mwords = 0;
  u64* M = nullptr;     // levels
  u64* T[4] = {};       // transform buffers
  u64* extra = nullptr; // 3k words (interpolation)
};

static int tree_alloc(Frame& fr, size_t k, size_t extra_words, Tree* t) {
  t->k = k;
  t->K = log2_ceil(k);
  t->N = (size_t)1 << t->K;
  t->lb = std::min(t->K, TREE_B);
  size_t at = 0;
  for (u32 j = t->lb; j <= t->K; j++) {
    t->off[j] = at;
    at += (t->N >> j) * (((size_t)1 << j) + 1);
  }
  t->mwords = at;
  RONK_TRY(fr.take(&t->M, at + 4 * t->N + extra_words));
  for (int i = 0; i < 4; i++) t->T[i] = t->M + at + i * t->N;
  t->extra = t->M + at + 4 * t->N;
  return RONK_OK;
}

static int spread(ronk_ctx* ctx, const u64* src, size_t stride, size_t len, u32 log_d, size_t P, u64* A, u64* B) {
  return launch(ctx, "tree_spread", tree_spread_kernel, grid_for(ctx, P << log_d, 256), 256, 0, false, src, stride, len, log_d, P,
                A, B);
}

// Levels lb … K of the product tree (T[0], T[1] scratch).
template <class F>
static int tree_build(ronk_ctx* ctx, const F& f, u64 p, u64 g, const Tree& t, const u64* xs) {
  RONK_TRY(launch(ctx, "tree_leaves", tree_leaves_kernel<F, false>, (u32)(t.N >> t.lb), 128, 0, false, f, xs, (const u64*)nullptr,
                  t.k, t.lb, t.M + t.off[t.lb], (u64*)nullptr));
  for (u32 j = t.lb; j < t.K; j++) {
    const u32 ld = j + 1;
    const size_t w = (size_t)1 << j, P = t.N >> ld;
    u64 *A = t.T[0], *B = t.T[1];
    RONK_TRY(spread(ctx, t.M + t.off[j], w + 1, w + 1, ld, P, A, B));
    RONK_TRY(ntt_device(ctx, p, g, A, nullptr, ld, (u32)P, 0));
    RONK_TRY(ntt_device(ctx, p, g, B, A, ld, (u32)P, 0));
    RONK_TRY(ntt_device(ctx, p, g, B, nullptr, ld, (u32)P, 1));
    RONK_TRY(launch(ctx, "tree_fix", tree_fix_kernel<F>, grid_for(ctx, P * (2 * w + 1), 256), 256, 0, false, f, (const u64*)B,
                    t.k, ld, P, t.M + t.off[ld]));
  }
  return RONK_OK;
}

// out[i] = f(xs[i]) down the built tree; d ≥ 1.  Uses T[0 … 3].
template <class F>
static int tree_down(ronk_ctx* ctx, const F& f, u64 p, u64 g, const Tree& t, const u64* c, size_t d, const u64* xs, u64* out) {
  const size_t k = t.k, hl = std::min(k + 1, d);
  u64 *A = t.T[0], *B = t.T[1], *R = t.T[2], *Rn = t.T[3];
  // root: h = rev_d(f)·rev_k(M)^-1 mod y^d, ρ[u] = h[d-1-u]
  const u32 lq = std::max<u32>(1, log2_ceil(2 * d - 1));
  const size_t nq = (size_t)1 << lq;
  Frame fr(ctx);
  u64* X = nullptr;
  RONK_TRY(fr.take(&X, 2 * nq + 2 * d + hl));
  u64* Y = X + nq;
  u64* G = Y + nq;
  u64* FR = G + d;
  u64* HR = FR + d;
  RONK_TRY(reverse_words(ctx, "tree_reverse", t.M + t.off[t.K], k, hl, HR, hl));  // rev_k(M) mod y^hl; M monic: HR[0] = 1
  RONK_TRY(newton_inverse_device(ctx, p, g, HR, hl, d, 1, G, X, Y));
  RONK_TRY(reverse_words(ctx, "tree_reverse", c, d - 1, d, FR, d));
  RONK_TRY(product_bounded(ctx, p, g, FR, d, G, d, lq, X, Y, FR, d));
  RONK_TRY(reverse_words(ctx, "tree_reverse", FR, d - 1, std::min(d, k), R, t.N));
  for (u32 j = t.K; j-- > t.lb;) {  // parents at level j + 1
    const u32 ld = j + 1;
    const size_t w = (size_t)1 << j, P = t.N >> ld;
    RONK_TRY(ntt_device(ctx, p, g, R, nullptr, ld, (u32)P, 0));
    RONK_TRY(spread(ctx, t.M + t.off[j], w + 1, w + 1, ld, P, A, B));
    RONK_TRY(ntt_device(ctx, p, g, A, R, ld, (u32)P, 0));
    RONK_TRY(ntt_device(ctx, p, g, B, R, ld, (u32)P, 0));
    RONK_TRY(ntt_device(ctx, p, g, A, nullptr, ld, (u32)P, 1));
    RONK_TRY(ntt_device(ctx, p, g, B, nullptr, ld, (u32)P, 1));
    RONK_TRY(launch(ctx, "tree_extract", tree_extract_kernel, grid_for(ctx, t.N, 256), 256, 0, false, (const u64*)A, (const u64*)B,
                    k, j, 2 * P, Rn));
    std::swap(R, Rn);
  }
  return launch(ctx, "tree_eval_leaves", tree_eval_leaves_kernel<F>, (u32)(t.N >> t.lb), TREE_NL, 0, false, f,
                (const u64*)(t.M + t.off[t.lb]), (const u64*)R, xs, k, t.lb, out);
}

bool tree_fits(u64 p, u64 g, size_t k, size_t d) {
  if (g == 0 || k == 0 || k > kTreeMaxLeaves) return false;
  const u32 K = log2_ceil(k);
  u32 lmax = K > TREE_B ? K : 0;
  if (d) lmax = std::max(lmax, std::max<u32>(1, log2_ceil(2 * d - 1)));
  return pow2_fits(p, lmax);
}

int tree_from_roots(ronk_ctx* ctx, u64 p, u64 g, const u64* xs, size_t k, u64* out) {
  Frame fr(ctx);
  Tree t;
  RONK_TRY(tree_alloc(fr, k, 0, &t));
  RONK_TRY(with_field(ctx, p, 0, false, [&](const auto& f) { return tree_build(ctx, f, p, g, t, xs); }));
  RONK_CUDA(ctx, cudaMemcpyAsync(out, t.M + t.off[t.K], (k + 1) * sizeof(u64), cudaMemcpyDeviceToDevice, ctx->stream));
  return RONK_OK;
}

int tree_multieval(ronk_ctx* ctx, u64 p, u64 g, const u64* c, size_t d, const u64* xs, size_t m, u64* out) {
  Frame fr(ctx);
  Tree t;
  RONK_TRY(tree_alloc(fr, m, 0, &t));
  return with_field(ctx, p, 0, false, [&](const auto& f) {
    RONK_TRY(tree_build(ctx, f, p, g, t, xs));
    return tree_down(ctx, f, p, g, t, c, d, xs, out);
  });
}

int tree_interpolate(ronk_ctx* ctx, u64 p, u64 g, const u64* xs, const u64* ys, size_t k, u64* out) {
  Frame fr(ctx);
  Tree t;
  RONK_TRY(tree_alloc(fr, k, 2 * k, &t));
  u64* Mp = t.extra;  // M', then c_i = y_i / M'(x_i)
  u64* W = Mp + k;    // M'(x_i)
  return with_field(ctx, p, 0, false, [&](const auto& f) {
    using F = std::decay_t<decltype(f)>;
    RONK_TRY(tree_build(ctx, f, p, g, t, xs));
    RONK_TRY(launch(ctx, "tree_deriv", tree_deriv_kernel<F>, grid_for(ctx, k, 256), 256, 0, false, f,
                    (const u64*)(t.M + t.off[t.K]), k, Mp));
    RONK_TRY(tree_down(ctx, f, p, g, t, Mp, k, xs, W));
    const int rc = ronk_field_div_u64(ctx, p, ys, W, Mp, k);  // synchronises; M'(x_i) = 0 exactly for a repeated x_i
    if (rc == RONK_EINVAL)
      return set_err(ctx, RONK_EINVAL, "interpolation: repeated x coordinate (the reference divides by zero)");
    RONK_TRY(rc);
    // the bottom levels rebuild M in shared memory alongside r (rewriting level lb with the same words); then
    // r_parent = r_L·M_R + r_R·M_L, r in T[2]
    u64 *A = t.T[0], *B = t.T[1], *R = t.T[2], *C = t.T[3];
    RONK_TRY(launch(ctx, "tree_interp_leaves", tree_leaves_kernel<F, true>, (u32)(t.N >> t.lb), 128, 0, false, f, xs,
                    (const u64*)Mp, k, t.lb, t.M + t.off[t.lb], R));
    for (u32 j = t.lb; j < t.K; j++) {
      const u32 ld = j + 1;
      const size_t w = (size_t)1 << j, P = t.N >> ld;
      RONK_TRY(spread(ctx, R, w, w, ld, P, A, B));                                // r_L, r_R
      RONK_TRY(spread(ctx, t.M + t.off[j], w + 1, w + 1, ld, P, R, C));           // M_L, M_R
      RONK_TRY(ntt_device(ctx, p, g, A, nullptr, ld, (u32)P, 0));
      RONK_TRY(ntt_device(ctx, p, g, B, nullptr, ld, (u32)P, 0));
      RONK_TRY(ntt_device(ctx, p, g, C, A, ld, (u32)P, 0));                       // r̂_L·M̂_R
      RONK_TRY(ntt_device(ctx, p, g, R, B, ld, (u32)P, 0));                       // r̂_R·M̂_L
      RONK_TRY(ronk_field_add_u64(ctx, p, R, C, R, P << ld));
      RONK_TRY(ntt_device(ctx, p, g, R, nullptr, ld, (u32)P, 1));
    }
    RONK_CUDA(ctx, cudaMemcpyAsync(out, R, k * sizeof(u64), cudaMemcpyDeviceToDevice, ctx->stream));
    RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return RONK_OK;
  });
}

}  // namespace ronk
