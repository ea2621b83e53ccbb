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
// Batches: `batch` rows share one tree over one point set.  Row b of every row buffer sits at b·N, so a level's P parents
// per row are batch·P contiguous transforms.  At batch 1 the node spectra are fused into the rows' transforms (the
// single-row sequence); from batch 2 the node spectra M̂_L, M̂_R are transformed once per level and met with every row
// in one point-wise launch, 3 transforms per row and level instead of 5.
// tests/test_multipoint_model.py is a Python model of the same index arithmetic (test_multipoint_batch_model.py: rows).
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

// The product of the 2^lb leaves of subtree blockIdx.x, schoolbook level by level in shared memory (every level kept,
// nodes of level j at stride 2^j + 1), to out[blockIdx.x·(2^lb + 1) …].  With INTERP, for every row b < rows
// (blockIdx.y, stepping by gridDim.y) against those node products: also the interpolation sums r of row b (leaf r =
// cs[b·k + i], times scale[i] where scale is set; level j at stride 2^j) to rout[b·N + blockIdx.x·2^lb …], N =
// gridDim.x·2^lb.  The CTA's first row writes out.
template <class F, bool INTERP>
__global__ void __launch_bounds__(128)
tree_leaves_kernel(const F f, const u64* __restrict__ xs, const u64* __restrict__ cs, const u64* __restrict__ scale, size_t k,
                   u32 lb, u32 rows, u64* __restrict__ out, u64* __restrict__ rout) {
  __shared__ u64 m[(TREE_B + 3) * TREE_NL];  // level j: 2^lb + 2^(lb-j) words
  __shared__ u64 r[2][TREE_NL];
  const u32 nl = 1u << lb, t0 = threadIdx.x, nt = blockDim.x;
  const size_t base = (size_t)blockIdx.x << lb, N = (size_t)gridDim.x << lb;
  const u64 one = 1 % f.modulus();
  for (u32 i = t0; i < nl; i += nt) {
    const bool live = base + i < k;
    m[2 * i] = live ? f.neg(xs[base + i]) : one;
    m[2 * i + 1] = live ? one : 0ULL;
  }
  __syncthreads();
  u32 at = 0;  // first word of level j
  for (u32 j = 0; j < lb; j++) {
    const u32 w = 1u << j, sc = w + 1, sp = 2 * w + 1, np = nl >> (j + 1), next = at + (nl >> j) * sc;
    for (u32 t = t0; t < np * sp; t += nt) {
      const u32 i = t / sp, e = t % sp;
      const u64* L = &m[at + 2 * i * sc];
      const u64* R = L + sc;
      const u32 lo = e > w ? e - w : 0, hi = e < w ? e : w;
      u64 acc = 0;
      for (u32 a = lo; a <= hi; a++) acc = f.add(acc, f.mul(L[a], R[e - a]));
      m[next + i * sp + e] = acc;
    }
    __syncthreads();
    at = next;
  }
  if (blockIdx.y == 0)
    for (u32 e = t0; e <= nl; e += nt) out[(size_t)blockIdx.x * (nl + 1) + e] = m[at + e];
  if constexpr (INTERP) {
    for (u64 b = blockIdx.y; b < rows; b += gridDim.y) {
      for (u32 i = t0; i < nl; i += nt) {
        const bool live = base + i < k;
        const u64 c = live ? cs[b * k + base + i] : 0ULL;
        r[0][i] = live && scale ? f.mul(c, scale[base + i]) : c;
      }
      __syncthreads();
      u32 c = 0, lv = 0;
      for (u32 j = 0; j < lb; j++) {  // r_L·M_R + r_R·M_L, degree < 2w
        const u32 w = 1u << j, sc = w + 1, np = nl >> (j + 1);
        for (u32 t = t0; t < np * 2 * w; t += nt) {
          const u32 i = t / (2 * w), e = t % (2 * w);
          const u64* rL = &r[c][2 * i * w];
          const u64* rR = rL + w;
          const u64* ML = &m[lv + 2 * i * sc];
          const u64* MR = ML + sc;
          const u32 lo = e > w ? e - w : 0, hi = e < w ? e : w - 1;
          u64 acc = 0;
          for (u32 a = lo; a <= hi; a++) acc = f.add(acc, f.add(f.mul(rL[a], MR[e - a]), f.mul(rR[a], ML[e - a])));
          r[c ^ 1][i * 2 * w + e] = acc;
        }
        __syncthreads();
        c ^= 1;
        lv += (nl >> j) * sc;
      }
      for (u32 e = t0; e < nl; e += nt) rout[b * N + base + e] = r[c][e];
      __syncthreads();  // the next row rewrites r
    }
  }
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
// ρ_R = A[δ_L, δ), zero-filled to 2^j words.  Over rows of P = pmask + 1 parents each: parent i is node i & pmask of its
// level.
__global__ void tree_extract_kernel(const u64* __restrict__ A, const u64* __restrict__ B, size_t k, u32 j, size_t nchild,
                                    size_t pmask, u64* __restrict__ dst) {
  const size_t w = (size_t)1 << j, n = nchild << j, step = (size_t)gridDim.x * blockDim.x;
  for (size_t x = (size_t)blockIdx.x * blockDim.x + threadIdx.x; x < n; x += step) {
    const size_t c = x >> j, u = x & (w - 1), i = c >> 1, il = i & pmask;
    const size_t dl = node_deg(k, j, 2 * il), dr = node_deg(k, j, 2 * il + 1);
    dst[x] = (c & 1) ? (u < dr ? A[2 * i * w + dl + u] : 0ULL) : (u < dl ? B[2 * i * w + dr + u] : 0ULL);
  }
}

// Down-sweep from batch 2: the node spectra SA = M̂_L and SB = M̂_R of one level (nmask + 1 = N words, shared by every
// row) met with each row's ρ̂ (R, total = rows·N words): PA = M̂_L·ρ̂, PB = M̂_R·ρ̂.
template <class F>
__global__ void tree_node_mul_kernel(const F f, const u64* __restrict__ SA, const u64* __restrict__ SB,
                                     const u64* __restrict__ R, size_t nmask, size_t total, u64* __restrict__ PA,
                                     u64* __restrict__ PB) {
  const size_t step = (size_t)gridDim.x * blockDim.x;
  for (size_t x = (size_t)blockIdx.x * blockDim.x + threadIdx.x; x < total; x += step) {
    const u64 v = R[x];
    PA[x] = f.mul(SA[x & nmask], v);
    PB[x] = f.mul(SB[x & nmask], v);
  }
}

// Up-sweep from batch 2: R = r̂_L·M̂_R + r̂_R·M̂_L over every row (A = r̂_L, B = r̂_R, total = rows·N words; SA = M̂_L and
// SB = M̂_R, nmask + 1 = N words shared by every row).
template <class F>
__global__ void tree_node_mac_kernel(const F f, const u64* __restrict__ A, const u64* __restrict__ B, const u64* __restrict__ SA,
                                     const u64* __restrict__ SB, size_t nmask, size_t total, u64* __restrict__ R) {
  const size_t step = (size_t)gridDim.x * blockDim.x;
  for (size_t x = (size_t)blockIdx.x * blockDim.x + threadIdx.x; x < total; x += step)
    R[x] = f.add(f.mul(A[x], SB[x & nmask]), f.mul(B[x], SA[x & nmask]));
}

// reverse_words over rows: dst[b·ds + i] = i < n ? src[b·ss + last - i] : 0, i < len, over total = rows·len words.
__global__ void tree_reverse_rows_kernel(const u64* __restrict__ src, size_t ss, size_t last, size_t n, u64* __restrict__ dst,
                                         size_t ds, size_t len, size_t total) {
  const size_t step = (size_t)gridDim.x * blockDim.x;
  for (size_t x = (size_t)blockIdx.x * blockDim.x + threadIdx.x; x < total; x += step) {
    const size_t b = x / len, i = x - b * len;
    dst[b * ds + i] = i < n ? src[b * ss + last - i] : 0ULL;
  }
}

// out[i] = (i + 1)·M[i + 1], i < k
template <class F>
__global__ void tree_deriv_kernel(const F f, const u64* __restrict__ M, size_t k, u64* __restrict__ out) {
  const size_t step = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < k; i += step)
    out[i] = f.mul((u64)((i + 1) % f.modulus()), M[i + 1]);
}

// Subtree blockIdx.x at level lb, for every row b < rows (blockIdx.y, stepping by gridDim.y): r = f_b mod M = polynomial
// part of M·ρ_b·X^-δ (ρ_b at R + b·N, N = gridDim.x·2^lb), then out[b·k + i] = r(xs[i]) for the subtree's points.
template <class F>
__global__ void __launch_bounds__(TREE_NL)
tree_eval_leaves_kernel(const F f, const u64* __restrict__ M, const u64* __restrict__ R, const u64* __restrict__ xs, size_t k,
                        u32 lb, u32 rows, u64* __restrict__ out) {
  __shared__ u64 sM[TREE_NL + 1], sR[TREE_NL], sr[TREE_NL];
  const u32 w = 1u << lb, t0 = threadIdx.x, nt = blockDim.x;
  const size_t s = blockIdx.x, base = s << lb, N = (size_t)gridDim.x << lb;
  const u32 dl = (u32)node_deg(k, lb, s);
  for (u32 e = t0; e <= w; e += nt) sM[e] = M[s * (w + 1) + e];
  for (u64 b = blockIdx.y; b < rows; b += gridDim.y) {
    for (u32 u = t0; u < w; u += nt) sR[u] = R[b * N + s * w + u];
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
      out[b * k + base + i] = acc;
    }
  }
}

// Shape of the tree over k leaves and its place in the scratch of the function that builds it: the stored levels
// lb … K, two N-word node buffers S, the row buffers X of batch·N words each (two at batch 1, three above), then `extra`.
struct Tree {
  size_t k = 0, N = 1;
  u32 K = 0, lb = 0, batch = 1;
  size_t off[27] = {};  // first word of level j, j in [lb, K]
  size_t mwords = 0;
  u64* M = nullptr;     // levels
  u64* S[2] = {};       // node buffers
  u64* X[3] = {};       // row buffers
  u64* extra = nullptr; // 2k words (interpolation)
};

static size_t tree_shape(size_t k, u32 batch, Tree* t) {
  t->k = k;
  t->batch = batch;
  t->K = log2_ceil(k);
  t->N = (size_t)1 << t->K;
  t->lb = std::min(t->K, TREE_B);
  size_t at = 0;
  for (u32 j = t->lb; j <= t->K; j++) {
    t->off[j] = at;
    at += (t->N >> j) * (((size_t)1 << j) + 1);
  }
  t->mwords = at;
  return at + 2 * t->N + (batch == 1 ? 2 : 3) * (size_t)batch * t->N;
}

static int tree_alloc(Frame& fr, size_t k, u32 batch, size_t extra_words, Tree* t) {
  const size_t words = tree_shape(k, batch, t);
  RONK_TRY(fr.take(&t->M, words + extra_words));
  const size_t rows = (size_t)batch * t->N;
  t->S[0] = t->M + t->mwords;
  t->S[1] = t->S[0] + t->N;
  t->X[0] = t->S[1] + t->N;
  t->X[1] = t->X[0] + rows;
  t->X[2] = batch == 1 ? nullptr : t->X[1] + rows;
  t->extra = t->M + words;
  return RONK_OK;
}

static int spread(ronk_ctx* ctx, const u64* src, size_t stride, size_t len, u32 log_d, size_t P, u64* A, u64* B) {
  return launch(ctx, "tree_spread", tree_spread_kernel, grid_for(ctx, P << log_d, 256), 256, 0, false, src, stride, len, log_d, P,
                A, B);
}

int reverse_rows(ronk_ctx* ctx, const u64* src, size_t ss, size_t last, size_t n, u64* dst, size_t ds, size_t len,
                        u32 batch) {
  const size_t total = (size_t)batch * len;
  return launch(ctx, "tree_reverse", tree_reverse_rows_kernel, grid_for(ctx, total, 256), 256, 0, false, src, ss, last, n, dst,
                ds, len, total);
}

// Levels lb … K of the product tree (S scratch).
template <class F>
static int tree_build(ronk_ctx* ctx, const F& f, u64 p, u64 g, const Tree& t, const u64* xs) {
  RONK_TRY(launch(ctx, "tree_leaves", tree_leaves_kernel<F, false>, (u32)(t.N >> t.lb), 128, 0, false, f, xs, (const u64*)nullptr,
                  (const u64*)nullptr, t.k, t.lb, 1u, t.M + t.off[t.lb], (u64*)nullptr));
  for (u32 j = t.lb; j < t.K; j++) {
    const u32 ld = j + 1;
    const size_t w = (size_t)1 << j, P = t.N >> ld;
    u64 *A = t.S[0], *B = t.S[1];
    RONK_TRY(spread(ctx, t.M + t.off[j], w + 1, w + 1, ld, P, A, B));
    RONK_TRY(ntt_device(ctx, p, g, A, nullptr, ld, (u32)P, 0));
    RONK_TRY(ntt_device(ctx, p, g, B, A, ld, (u32)P, 0));
    RONK_TRY(ntt_device(ctx, p, g, B, nullptr, ld, (u32)P, 1));
    RONK_TRY(launch(ctx, "tree_fix", tree_fix_kernel<F>, grid_for(ctx, P * (2 * w + 1), 256), 256, 0, false, f, (const u64*)B,
                    t.k, ld, P, t.M + t.off[ld]));
  }
  return RONK_OK;
}

// The words tree_down's root step takes for h = rev_d(f)·rev_k(M)^-1 of every row: Newton's two transform buffers, the
// inverse, rev_k(M), and from batch 2 the reversed rows and their products (2d words each) against the shared inverse.
static size_t root_words(size_t k, size_t d, u32 batch) {
  const size_t hl = std::min(k + 1, d), nq = (size_t)1 << std::max<u32>(1, log2_ceil(2 * d - 1));
  if (batch == 1) return 2 * nq + 2 * d + hl;
  return 2 * nq + (d + 1) + hl + 3 * (size_t)batch * d;
}

// Row b of out (out + b·t.k) = f_b(xs[i]) down the built tree, f_b = c + b·d, d ≥ 1, b < batch ≤ t.batch.  Uses S and X.
template <class F>
static int tree_down(ronk_ctx* ctx, const F& f, u64 p, u64 g, const Tree& t, u32 batch, const u64* c, size_t d, const u64* xs,
                     u64* out) {
  const size_t k = t.k, hl = std::min(k + 1, d), N = t.N;
  u64 *R = t.X[0], *Rn = t.X[1], *Q = t.X[2];
  // root: h = rev_d(f)·rev_k(M)^-1 mod y^d, ρ[u] = h[d-1-u]
  const u32 lq = std::max<u32>(1, log2_ceil(2 * d - 1));
  const size_t nq = (size_t)1 << lq;
  Frame fr(ctx);
  u64* X = nullptr;
  RONK_TRY(fr.take(&X, root_words(k, d, batch)));
  u64* Y = X + nq;
  u64* G = Y + nq;
  u64* HR = G + (batch == 1 ? d : d + 1);
  u64* FR = HR + hl;
  RONK_TRY(reverse_words(ctx, "tree_reverse", t.M + t.off[t.K], k, hl, HR, hl));  // rev_k(M) mod y^hl; M monic: HR[0] = 1
  RONK_TRY(newton_inverse_device(ctx, p, g, HR, hl, d, 1, G, X, Y));
  if (batch == 1) {
    RONK_TRY(reverse_words(ctx, "tree_reverse", c, d - 1, d, FR, d));
    RONK_TRY(product_bounded(ctx, p, g, FR, d, G, d, lq, X, Y, FR, d));
    RONK_TRY(reverse_words(ctx, "tree_reverse", FR, d - 1, std::min(d, k), R, N));
  } else {  // G gets a zero word d, so that the rows' product has 2d words: the bounded transform product of d = 1 too
    u64* H = FR + (size_t)batch * d;
    RONK_CUDA(ctx, cudaMemsetAsync(G + d, 0, sizeof(u64), ctx->stream));
    RONK_TRY(reverse_rows(ctx, c, d, d - 1, d, FR, d, d, batch));
    RONK_TRY(poly_mul_rows_pow2(ctx, p, g, FR, d, G, d + 1, true, batch, H));
    RONK_TRY(reverse_rows(ctx, H, 2 * d, d - 1, std::min(d, k), R, N, N, batch));
  }
  for (u32 j = t.K; j-- > t.lb;) {  // parents at level j + 1
    const u32 ld = j + 1;
    const size_t w = (size_t)1 << j, P = N >> ld;
    const u32 rows = (u32)(batch * P);
    RONK_TRY(ntt_device(ctx, p, g, R, nullptr, ld, rows, 0));
    RONK_TRY(spread(ctx, t.M + t.off[j], w + 1, w + 1, ld, P, t.S[0], t.S[1]));
    u64 *PA = t.S[0], *PB = t.S[1], *dst = Rn;
    if (batch == 1) {  // the node spectra fused into the rows' transforms
      RONK_TRY(ntt_device(ctx, p, g, PA, R, ld, rows, 0));
      RONK_TRY(ntt_device(ctx, p, g, PB, R, ld, rows, 0));
    } else {           // the node spectra once, met with every row in one launch
      RONK_TRY(ntt_device(ctx, p, g, t.S[0], nullptr, ld, (u32)P, 0));
      RONK_TRY(ntt_device(ctx, p, g, t.S[1], nullptr, ld, (u32)P, 0));
      const size_t total = (size_t)batch * N;
      PA = Rn, PB = Q, dst = R;
      RONK_TRY(launch(ctx, "tree_node_mul", tree_node_mul_kernel<F>, grid_for(ctx, total, 256), 256, 0, false, f,
                      (const u64*)t.S[0], (const u64*)t.S[1], (const u64*)R, N - 1, total, PA, PB));
    }
    RONK_TRY(ntt_device(ctx, p, g, PA, nullptr, ld, rows, 1));
    RONK_TRY(ntt_device(ctx, p, g, PB, nullptr, ld, rows, 1));
    RONK_TRY(launch(ctx, "tree_extract", tree_extract_kernel, grid_for(ctx, (size_t)batch * N, 256), 256, 0, false,
                    (const u64*)PA, (const u64*)PB, k, j, 2 * (size_t)rows, P - 1, dst));
    if (batch == 1) std::swap(R, Rn);
  }
  return launch(ctx, "tree_eval_leaves", tree_eval_leaves_kernel<F>, dim3((u32)(N >> t.lb), grid_rows(ctx, batch, N >> t.lb)), TREE_NL, 0, false,
                f, (const u64*)(t.M + t.off[t.lb]), (const u64*)R, xs, k, t.lb, batch, out);
}

bool tree_fits(u64 p, u64 g, size_t k, size_t d) {
  if (g == 0 || k == 0 || k > kTreeMaxLeaves) return false;
  const u32 K = log2_ceil(k);
  u32 lmax = K > TREE_B ? K : 0;
  if (d) lmax = std::max(lmax, std::max<u32>(1, log2_ceil(2 * d - 1)));
  return pow2_fits(p, lmax);
}

size_t tree_scratch_words(const ronk_ctx* ctx, size_t k, size_t d, u32 batch, bool interp) {
  Tree t;
  const size_t tree = tree_shape(k, batch, &t) + (interp ? 2 * k : 0);
  if (interp) d = k;  // M'(x_i) down the tree as one row
  const size_t root = root_words(k, d, interp ? 1 : batch), nq = (size_t)1 << std::max<u32>(1, log2_ceil(2 * d - 1));
  // above them the largest of: a level's transform workspace (batch·N words), Newton's (nq), the rows' product's
  size_t above = std::max((size_t)batch * t.N, nq);
  if (!interp && batch > 1) above = std::max(above, poly_mul_rows_pow2_scratch(ctx, d, d + 1, true, batch));
  return tree + root + above + 16 * Frame::kAlign / 8;  // and each take's rounding to 256 bytes
}

int poly_deriv(ronk_ctx* ctx, u64 p, const u64* M, size_t k, u64* out) {
  return with_field(ctx, p, 0, false, [&](const auto& f) {
    return launch(ctx, "tree_deriv", tree_deriv_kernel<std::decay_t<decltype(f)>>, grid_for(ctx, k, 256), 256, 0, false, f, M, k,
                  out);
  });
}

int tree_from_roots(ronk_ctx* ctx, u64 p, u64 g, const u64* xs, size_t k, u64* out) {
  Frame fr(ctx);
  Tree t;
  RONK_TRY(tree_alloc(fr, k, 1, 0, &t));
  RONK_TRY(with_field(ctx, p, 0, false, [&](const auto& f) { return tree_build(ctx, f, p, g, t, xs); }));
  RONK_CUDA(ctx, cudaMemcpyAsync(out, t.M + t.off[t.K], (k + 1) * sizeof(u64), cudaMemcpyDeviceToDevice, ctx->stream));
  return RONK_OK;
}

int tree_multieval(ronk_ctx* ctx, u64 p, u64 g, const u64* c, size_t d, u32 batch, const u64* xs, size_t m, u64* out) {
  Frame fr(ctx);
  Tree t;
  RONK_TRY(tree_alloc(fr, m, batch, 0, &t));
  return with_field(ctx, p, 0, false, [&](const auto& f) {
    RONK_TRY(tree_build(ctx, f, p, g, t, xs));
    return tree_down(ctx, f, p, g, t, batch, c, d, xs, out);
  });
}

int tree_interpolate(ronk_ctx* ctx, u64 p, u64 g, const u64* xs, const u64* ys, size_t k, u32 batch, u64* out) {
  Frame fr(ctx);
  Tree t;
  RONK_TRY(tree_alloc(fr, k, batch, 2 * k, &t));
  u64* Mp = t.extra;  // M', then c_i = y_i / M'(x_i) (batch 1) or M'(x_i)^-1
  u64* W = Mp + k;    // M'(x_i)
  return with_field(ctx, p, 0, false, [&](const auto& f) {
    using F = std::decay_t<decltype(f)>;
    RONK_TRY(tree_build(ctx, f, p, g, t, xs));
    RONK_TRY(launch(ctx, "tree_deriv", tree_deriv_kernel<F>, grid_for(ctx, k, 256), 256, 0, false, f,
                    (const u64*)(t.M + t.off[t.K]), k, Mp));
    RONK_TRY(tree_down(ctx, f, p, g, t, 1, Mp, k, xs, W));
    // synchronises; M'(x_i) = 0 exactly for a repeated x_i.  From batch 2 the inverse is taken once and the leaves
    // kernel multiplies each row's y by it.
    const int rc = batch == 1 ? ronk_field_div_u64(ctx, p, ys, W, Mp, k) : ronk_field_inv_u64(ctx, p, W, Mp, k);
    if (rc == RONK_EINVAL)
      return set_err(ctx, RONK_EINVAL, "interpolation: repeated x coordinate (the reference divides by zero)");
    RONK_TRY(rc);
    // the bottom levels rebuild M in shared memory alongside r (rewriting level lb with the same words); then
    // r_parent = r_L·M_R + r_R·M_L, r in X[0]
    const size_t N = t.N;
    u64 *R = t.X[0], *A = t.X[1], *B = batch == 1 ? t.S[0] : t.X[2];
    u64 *ML = batch == 1 ? R : t.S[0], *MR = t.S[1];
    RONK_TRY(launch(ctx, "tree_interp_leaves", tree_leaves_kernel<F, true>, dim3((u32)(N >> t.lb), grid_rows(ctx, batch, N >> t.lb)), 128, 0,
                    false, f, xs, batch == 1 ? (const u64*)Mp : ys, batch == 1 ? (const u64*)nullptr : (const u64*)Mp, k,
                    t.lb, batch, t.M + t.off[t.lb], R));
    for (u32 j = t.lb; j < t.K; j++) {
      const u32 ld = j + 1;
      const size_t w = (size_t)1 << j, P = N >> ld;
      const u32 rows = (u32)(batch * P);
      RONK_TRY(spread(ctx, R, w, w, ld, rows, A, B));                             // r_L, r_R
      RONK_TRY(spread(ctx, t.M + t.off[j], w + 1, w + 1, ld, P, ML, MR));         // M_L, M_R
      RONK_TRY(ntt_device(ctx, p, g, A, nullptr, ld, rows, 0));
      RONK_TRY(ntt_device(ctx, p, g, B, nullptr, ld, rows, 0));
      if (batch == 1) {  // the node spectra fused into the rows' products
        RONK_TRY(ntt_device(ctx, p, g, MR, A, ld, rows, 0));                      // r̂_L·M̂_R
        RONK_TRY(ntt_device(ctx, p, g, ML, B, ld, rows, 0));                      // r̂_R·M̂_L
        RONK_TRY(ronk_field_add_u64(ctx, p, ML, MR, R, P << ld));
      } else {           // the node spectra once, met with every row in one launch
        RONK_TRY(ntt_device(ctx, p, g, ML, nullptr, ld, (u32)P, 0));
        RONK_TRY(ntt_device(ctx, p, g, MR, nullptr, ld, (u32)P, 0));
        const size_t total = (size_t)batch * N;
        RONK_TRY(launch(ctx, "tree_node_mac", tree_node_mac_kernel<F>, grid_for(ctx, total, 256), 256, 0, false, f,
                        (const u64*)A, (const u64*)B, (const u64*)ML, (const u64*)MR, N - 1, total, R));
      }
      RONK_TRY(ntt_device(ctx, p, g, R, nullptr, ld, rows, 1));
    }
    RONK_CUDA(ctx, cudaMemcpy2DAsync(out, k * sizeof(u64), R, N * sizeof(u64), k * sizeof(u64), batch, cudaMemcpyDeviceToDevice,
                                     ctx->stream));
    RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return RONK_OK;
  });
}

}  // namespace ronk
