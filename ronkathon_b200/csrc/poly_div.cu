// poly_div.cu — quotient_and_remainder (src/polynomial/mod.rs:170-225, Div/Rem arithmetic.rs:121-146) for a divisor
// with a nonzero top word, by power-series inversion (Newton iteration) on the transform kernels.  With L = da - db + 1
// and rev_n(x) the first n words of x reversed:
//   (1) ar = rev(a)[0, L), hr = rev(b) truncated to min(db, L) words;
//   (2) inv = hr^-1 mod x^L by doubling: g_1 = b[db-1]^-1, g_2t = g_t·(2 - hr·g_t) mod x^2t, on transforms of 4t points;
//   (3) rev(q) = ar·inv mod x^L, reversed into q[0, L);
//   (4) r = a - b·q on its first db - 1 words (r has degree < db - 1): from the low db - 1 words of b and q when the
//       quotient is that long, else with a, b, q taken mod x^N - 1 for an N ≥ db - 1 (the cyclic difference is r itself).
// The cost is a fixed number of transforms of about 2L points; the literal kernel (poly.cu) is quadratic.
// ronk_poly_divrem_u64 (poly.cu) chooses this path; it owns the checks and the quirky divisors.
#include <algorithm>

#include "ronk_internal.h"

namespace ronk {

// dst[i] = i < n ? src[last - i] : 0, i < dst_len: reverses, truncates and zero-fills in one pass
__global__ void reverse_kernel(const u64* __restrict__ src, size_t last, size_t n, u64* __restrict__ dst, size_t dst_len) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < dst_len; i += stride)
    dst[i] = (i < n) ? src[last - i] : 0ULL;
}

// One Newton step point-wise in the transform domain: G[k] ← G[k]·(2 - H[k]·G[k])
template <class F>
__global__ void divrem_newton_step_kernel(const F f, u64* __restrict__ G, const u64* __restrict__ H, size_t n) {
  const u64 two = 2 % f.modulus();
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += stride) {
    const u64 g = G[k];
    G[k] = f.mul(g, f.sub(two, f.mul(H[k], g)));
  }
}

// dst[i] = Σ_j src[i + j·n] (the residue mod x^n - 1), i < dst_len ≤ n
template <class F>
__global__ void divrem_fold_kernel(const F f, const u64* __restrict__ src, size_t len, size_t n, u64* __restrict__ dst,
                                   size_t dst_len) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < dst_len; i += stride) {
    u64 acc = 0;
    for (size_t j = i; j < len; j += n) acc = f.add(acc, src[j]);
    dst[i] = acc;
  }
}

// Transform sizes (log2) of the plan: the quotient product (also the largest Newton step) and the remainder product.
// The remainder needs only b·q mod x^(db-1).  A quotient at least that long is cut to its low db - 1 words, like b,
// and the product runs without wrap (2(db-1) - 1 points); a shorter one keeps every word and the product is taken mod
// x^N - 1 with N ≥ db - 1, folding the operands longer than N (dividend, and b when db - 1 = N).
static void divrem_newton_sizes(size_t da, size_t db, u32* log_q, u32* log_r) {
  const size_t L = da - db + 1, rw = db - 1;  // L ≥ 1; rw = 0 (a constant divisor): no remainder product
  *log_q = std::max<u32>(1, log2_ceil(2 * L - 1));
  *log_r = rw == 0 ? 1 : std::max<u32>(1, L >= rw ? log2_ceil(2 * rw - 1) : log2_ceil(rw));
}

bool divrem_newton_fits(u64 p, u64 g, size_t da, size_t db) {
  if (g == 0 || da < db || db == 0) return false;
  u32 lq, lr;
  divrem_newton_sizes(da, db, &lq, &lr);
  const u32 lmax = std::max(lq, lr);
  return pow2_fits(p, lmax);
}

template <class F>
static int fold(ronk_ctx* ctx, const F& f, const u64* src, size_t len, size_t n, u64* dst, size_t dst_len) {
  return launch(ctx, "divrem_fold", divrem_fold_kernel<F>, grid_for(ctx, dst_len, 256), 256, 0, false, f, src, len, n, dst,
                dst_len);
}

int reverse_words(ronk_ctx* ctx, const char* name, const u64* src, size_t last, size_t n, u64* dst, size_t dst_len) {
  return launch(ctx, name, reverse_kernel, grid_for(ctx, dst_len, 256), 256, 0, false, src, last, n, dst, dst_len);
}

// G = hr^-1 mod x^L by Newton doubling, hr of hl ≤ L words with hr[0]^-1 = g1: g_2t = g_t·(2 - hr·g_t) mod x^2t on
// transforms of 4t points.  X and Y hold the largest of them: 2^⌈log2(2L - 1)⌉ words each.
template <class F>
static int newton_inverse(ronk_ctx* ctx, const F& f, u64 p, u64 g, const u64* HR, size_t hl, size_t L, u64 g1, u64* G,
                          u64* X, u64* Y) {
  // g_1 (pageable source: the copy is staged before cudaMemcpyAsync returns)
  RONK_CUDA(ctx, cudaMemcpyAsync(G, &g1, sizeof(u64), cudaMemcpyHostToDevice, ctx->stream));
  for (size_t t = 1; t < L; t *= 2) {
    // g_t·(2 - hr·g_t) has degree < 4t - 2: the 4t-point cyclic product is exact; keep its first m words
    const size_t m = std::min(2 * t, L);
    const u32 ln = log2_ceil(4 * t);
    RONK_TRY(ntt_device_bounded(ctx, p, g, HR, std::min(hl, m), Y, (u64)1 << ln, nullptr, ln, 0));  // Ĥ of hr mod x^m
    RONK_TRY(ntt_device_bounded(ctx, p, g, G, t, X, (u64)1 << ln, nullptr, ln, 0));                 // Ĝ of g_t
    RONK_TRY(launch(ctx, "divrem_newton_step", divrem_newton_step_kernel<F>, grid_for(ctx, (size_t)1 << ln, 256), 256, 0, false,
                    f, X, (const u64*)Y, (size_t)1 << ln));
    RONK_TRY(ntt_device_bounded(ctx, p, g, X, (u64)1 << ln, G, m, nullptr, ln, 1));  // g_2t mod x^m
  }
  return RONK_OK;
}

int newton_inverse_device(ronk_ctx* ctx, u64 p, u64 g, const u64* hr, size_t hl, size_t L, u64 g1, u64* G, u64* X, u64* Y) {
  return with_field(ctx, p, 0, false, [&](const auto& f) { return newton_inverse(ctx, f, p, g, hr, hl, L, g1, G, X, Y); });
}

template <class F>
static int divrem_newton_with_field(ronk_ctx* ctx, const F& f, u64 p, u64 g, const u64* a, size_t da, const u64* b, size_t db,
                                    u64 top, u64* q, u64* r) {
  const size_t L = da - db + 1, hl = std::min(db, L);
  u32 lq, lr;
  divrem_newton_sizes(da, db, &lq, &lr);
  const size_t nq = (size_t)1 << lq, nr = (size_t)1 << lr, nx = std::max(nq, nr);
  // X, Y transform buffers | G = inv | AR | HR
  Frame fr(ctx);
  u64* X = nullptr;
  RONK_TRY(fr.take(&X, 2 * nx + 2 * L + hl));
  u64* Y = X + nx;
  u64* G = Y + nx;
  u64* AR = G + L;
  u64* HR = AR + L;
  RONK_TRY(reverse_words(ctx, "divrem_reverse", a, da - 1, L, AR, L));
  RONK_TRY(reverse_words(ctx, "divrem_reverse", b, db - 1, hl, HR, hl));
  RONK_TRY(newton_inverse(ctx, f, p, g, HR, hl, L, h_powmod(top, p - 2, p), G, X, Y));  // g_1 = b[db-1]^-1
  // rev(q) = ar·inv mod x^L (nq ≥ 2L - 1: no wrap into the low L words), into AR, then reversed into q
  RONK_TRY(product_bounded(ctx, p, g, AR, L, G, L, lq, X, Y, AR, L));
  RONK_TRY(reverse_words(ctx, "divrem_reverse", AR, L - 1, L, q, da));
  const size_t rw = db - 1;  // remainder words
  if (rw == 0) {
    RONK_CUDA(ctx, cudaMemsetAsync(r, 0, da * sizeof(u64), ctx->stream));
    return RONK_OK;
  }
  const u64* A = a;
  if (L >= rw) {  // low product: (b mod x^rw)·(q mod x^rw), nr ≥ 2·rw - 1
    RONK_TRY(product_bounded(ctx, p, g, b, rw, q, rw, lr, X, Y, Y, rw));
  } else {  // b·q mod x^nr - 1, nr ≥ rw > L (q needs no fold; da < 2·rw, so every fold adds at most two terms)
    if (db > nr) {
      RONK_TRY(fold(ctx, f, b, db, nr, X, nr));
      RONK_TRY(product_bounded(ctx, p, g, X, nr, q, L, lr, X, Y, Y, rw));
    } else {
      RONK_TRY(product_bounded(ctx, p, g, b, db, q, L, lr, X, Y, Y, rw));
    }
    if (da > nr) {
      RONK_TRY(fold(ctx, f, a, da, nr, X, rw));
      A = X;
    }
  }
  RONK_TRY(ronk_poly_sub_u64(ctx, p, (const uint64_t*)A, rw, (const uint64_t*)Y, rw, (uint64_t*)r));
  if (da > rw) RONK_CUDA(ctx, cudaMemsetAsync(r + rw, 0, (da - rw) * sizeof(u64), ctx->stream));
  return RONK_OK;
}

// a / b with b[db-1] = top != 0 and divrem_newton_fits(p, g, da, db); q and r have da words.  Arguments are checked by
// the caller.  Stream-ordered; the caller synchronises.
int divrem_newton_device(ronk_ctx* ctx, u64 p, u64 g, const u64* a, size_t da, const u64* b, size_t db, u64 top, u64* q,
                         u64* r) {
  return with_field(ctx, p, 0, false, [&](const auto& f) {
    return divrem_newton_with_field(ctx, f, p, g, a, da, b, db, top, q, r);
  });
}

// ---- batches of rows (ronk_poly_divrem_batch_u64, poly.cu) ---------------------------------------------------------
// out[y·os] = top_y^-1 and, with_z, out[y·os + 1] = z_y = -b_y[0]·top_y^-1, top_y = b_y[db - 1] != 0 (rows db apart)
template <class F>
__global__ void divrem_top_inv_kernel(const F f, const u64* __restrict__ b, size_t db, u32 batch, u64* __restrict__ out, size_t os,
                                      bool with_z) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t y = (size_t)blockIdx.x * blockDim.x + threadIdx.x; y < batch; y += stride) {
    const u64 inv = field_pow(f, b[y * db + db - 1], f.modulus() - 2);
    out[y * os] = inv;
    if (with_z) out[y * os + 1] = f.mul(f.sub(0, b[y * db]), inv);
  }
}

// dst[y·n + k] = Σ_j src[y·ss + k + j·n] over k + j·n < len, k < n (n = 2^log_n): the rows mod x^n - 1, zero-padded;
// total = rows·n
template <class F>
__global__ void divrem_rows_fold_kernel(const F f, const u64* __restrict__ src, size_t ss, size_t len, u32 log_n, u64 total,
                                        u64* __restrict__ dst) {
  const u64 step = (u64)gridDim.x * blockDim.x, n = (u64)1 << log_n;
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += step) {
    const u64* row = src + (i >> log_n) * ss;
    u64 acc = 0;
    for (u64 k = i & (n - 1); k < len; k += n) acc = f.add(acc, row[k]);
    dst[i] = acc;
  }
}

// dst[y·ds + k] = src[y·ss + k], k < n; total = rows·n
__global__ void divrem_rows_copy_kernel(const u64* __restrict__ src, size_t ss, size_t n, u64* __restrict__ dst, size_t ds,
                                        u64 total) {
  const u64 step = (u64)gridDim.x * blockDim.x;
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += step) {
    const u64 y = i / n, k = i - y * n;
    dst[y * ds + k] = src[y * ss + k];
  }
}

// r[y·da + k] = k < rw ? Σ_j a[y·da + k + j·na] - P[y·np + k] : 0 (j over k + j·na < da), total = rows·da: the remainder
// from the low words of b·q, with the dividend taken mod x^na - 1 (na = da: not folded)
template <class F>
__global__ void divrem_rows_rem_kernel(const F f, const u64* __restrict__ a, size_t da, size_t na, const u64* __restrict__ P,
                                       size_t np, size_t rw, u64 total, u64* __restrict__ r) {
  const u64 step = (u64)gridDim.x * blockDim.x;
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += step) {
    const u64 y = i / da, k = i - y * da;
    if (k >= rw) {
      r[i] = 0;
      continue;
    }
    u64 acc = 0;
    for (u64 j = k; j < da; j += na) acc = f.add(acc, a[y * da + j]);
    r[i] = f.sub(acc, P[y * np + k]);
  }
}

template <class F>
static int rows_fold(ronk_ctx* ctx, const F& f, const u64* src, size_t ss, size_t len, u32 log_n, u32 rows, u64* dst) {
  const u64 total = (u64)rows << log_n;
  return launch(ctx, "divrem_rows_fold", divrem_rows_fold_kernel<F>, grid_for(ctx, total, 256), 256, 0, false, f, src, ss, len,
                log_n, total, dst);
}

// The cyclic products of X's batch rows (2^log_n words each, zero-padded, untransformed) by B's rows (one shared row, or
// batch): returns the buffer that holds them.
static u64* rows_product(ronk_ctx* ctx, u64 p, u64 g, u64* X, u64* B, u32 log_n, u32 batch, bool shared, int* rc) {
  if (shared) {
    if ((*rc = ntt_device(ctx, p, g, B, nullptr, log_n, 1, 0)) != RONK_OK) return nullptr;
    if ((*rc = ntt_device_shared_mul(ctx, p, g, X, X, B, log_n, batch)) != RONK_OK) return nullptr;
    *rc = ntt_device(ctx, p, g, X, nullptr, log_n, batch, 1);
    return X;
  }
  if ((*rc = ntt_device(ctx, p, g, X, nullptr, log_n, batch, 0)) != RONK_OK) return nullptr;
  if ((*rc = ntt_device(ctx, p, g, B, X, log_n, batch, 0)) != RONK_OK) return nullptr;  // B̂ ⊙ X̂ fused into the last pass
  *rc = ntt_device(ctx, p, g, B, nullptr, log_n, batch, 1);
  return B;
}

// The regions of the batched plan: G (the inverses, rows L apart) | HR (rev(b) cut to hl words) | X (batch rows of nx) |
// B (the other operand's rows of nx: one shared row, or batch).
struct DivremRows {
  size_t L, hl, rw, nq, nr, nx;
  u32 lq, lr;
  u32 rows_b;
};

static DivremRows divrem_rows_plan(size_t da, size_t db, bool b_shared, u32 batch) {
  DivremRows d;
  d.L = da - db + 1;
  d.hl = std::min(db, d.L);
  d.rw = db - 1;
  divrem_newton_sizes(da, db, &d.lq, &d.lr);
  d.nq = (size_t)1 << d.lq;
  d.nr = (size_t)1 << d.lr;
  d.nx = std::max(d.nq, d.nr);
  d.rows_b = b_shared ? 1 : batch;
  return d;
}

u64 divrem_newton_rows_transform_words(size_t da, size_t db, u32 batch) {
  u32 lq, lr;
  divrem_newton_sizes(da, db, &lq, &lr);
  return (u64)batch << std::max(lq, lr);
}

size_t divrem_newton_rows_scratch(size_t da, size_t db, bool b_shared, u32 batch) {
  const DivremRows d = divrem_rows_plan(da, db, b_shared, batch);
  const size_t words = d.rows_b * (d.L + d.hl + d.nx) + (size_t)batch * d.nx;
  return words + ntt_workspace_words(std::max(d.lq, d.lr), batch) + 8 * Frame::kAlign / 8;
}

template <class F>
static int divrem_newton_rows_with_field(ronk_ctx* ctx, const F& f, u64 p, u64 g, const u64* a, size_t da, const u64* b, size_t db,
                                         bool b_shared, u32 batch, u64 top, u64* q, u64* r) {
  const DivremRows d = divrem_rows_plan(da, db, b_shared, batch);
  const size_t L = d.L, hl = d.hl, rw = d.rw, nq = d.nq, nr = d.nr;
  Frame fr(ctx);
  u64 *G = nullptr, *HR = nullptr, *X = nullptr, *B = nullptr;
  RONK_TRY(fr.take(&G, d.rows_b * L));
  RONK_TRY(fr.take(&HR, d.rows_b * hl));
  RONK_TRY(fr.take(&X, (size_t)batch * d.nx));
  RONK_TRY(fr.take(&B, d.rows_b * d.nx));
  // (1) the inverses of rev(b) mod x^L
  RONK_TRY(reverse_rows(ctx, b, db, db - 1, hl, HR, hl, hl, d.rows_b));
  if (b_shared) {
    RONK_TRY(newton_inverse(ctx, f, p, g, HR, hl, L, h_powmod(top, p - 2, p), G, X, X + nq));  // batch ≥ 2: 2·nq ≤ batch·nx
  } else {  // the doubling steps of newton_inverse on batched transforms of every row
    RONK_TRY(launch(ctx, "divrem_top_inv", divrem_top_inv_kernel<F>, grid_for(ctx, batch, 256), 256, 0, false, f, b, db, batch, G,
                    L, false));
    for (size_t t = 1; t < L; t *= 2) {
      const size_t m = std::min(2 * t, L);
      const u32 ln = log2_ceil(4 * t);
      const u64 total = (u64)batch << ln;
      const int grid = grid_for(ctx, total, PAD_THREADS);
      RONK_TRY(launch(ctx, "poly_rows_pad", poly_rows_pad_kernel, grid, PAD_THREADS, 0, false, HR, (u32)std::min(hl, m), (u64)hl, ln,
                      total, B));
      RONK_TRY(launch(ctx, "poly_rows_pad", poly_rows_pad_kernel, grid, PAD_THREADS, 0, false, G, (u32)t, (u64)L, ln, total, X));
      RONK_TRY(ntt_device(ctx, p, g, B, nullptr, ln, batch, 0));
      RONK_TRY(ntt_device(ctx, p, g, X, nullptr, ln, batch, 0));
      RONK_TRY(launch(ctx, "divrem_newton_step", divrem_newton_step_kernel<F>, grid_for(ctx, total, 256), 256, 0, false, f, X,
                      (const u64*)B, (size_t)total));
      RONK_TRY(ntt_device(ctx, p, g, X, nullptr, ln, batch, 1));
      const u64 copied = (u64)batch * m;
      RONK_TRY(launch(ctx, "divrem_rows_copy", divrem_rows_copy_kernel, grid_for(ctx, copied, 256), 256, 0, false, (const u64*)X,
                      (size_t)1 << ln, m, G, L, copied));
    }
  }
  // (2) rev(q) = rev(a)·inv mod x^L (nq ≥ 2L - 1: no wrap into the low L words), reversed into q
  int rc = RONK_OK;
  RONK_TRY(reverse_rows(ctx, a, da, da - 1, L, X, nq, nq, batch));
  RONK_TRY(rows_fold(ctx, f, G, L, L, d.lq, d.rows_b, B));
  const u64* QR = rows_product(ctx, p, g, X, B, d.lq, batch, b_shared, &rc);
  RONK_TRY(rc);
  RONK_TRY(reverse_rows(ctx, QR, nq, L - 1, L, q, da, da, batch));
  if (rw == 0) {
    RONK_CUDA(ctx, cudaMemsetAsync(r, 0, (size_t)batch * da * sizeof(u64), ctx->stream));
    return RONK_OK;
  }
  // (3) r = a - b·q on its low rw words: (b mod x^rw)·(q mod x^rw) when L ≥ rw (nr ≥ 2·rw - 1, no wrap), else b·q and a
  // mod x^nr - 1 (nr ≥ rw > L), the cyclic difference being r itself
  const u64 total = (u64)batch * nr;
  RONK_TRY(launch(ctx, "poly_rows_pad", poly_rows_pad_kernel, grid_for(ctx, total, PAD_THREADS), PAD_THREADS, 0, false, (const u64*)q,
                  (u32)std::min(L, rw), (u64)da, d.lr, total, X));
  RONK_TRY(rows_fold(ctx, f, b, db, L >= rw ? rw : db, d.lr, d.rows_b, B));
  const u64* P = rows_product(ctx, p, g, X, B, d.lr, batch, b_shared, &rc);
  RONK_TRY(rc);
  const u64 words = (u64)batch * da;
  return launch(ctx, "divrem_rows_rem", divrem_rows_rem_kernel<F>, grid_for(ctx, words, 256), 256, 0, false, f, a, da,
                L >= rw ? da : nr, P, nr, rw, words, r);
}

int divrem_newton_rows(ronk_ctx* ctx, u64 p, u64 g, const u64* a, size_t da, const u64* b, size_t db, bool b_shared, u32 batch,
                       u64 top, u64* q, u64* r) {
  return with_field(ctx, p, 0, false, [&](const auto& f) {
    return divrem_newton_rows_with_field(ctx, f, p, g, a, da, b, db, b_shared, batch, top, q, r);
  });
}

int divrem_top_inverses(ronk_ctx* ctx, u64 p, const u64* b, size_t db, u32 batch, u64* out) {
  return with_field(ctx, p, 0, false, [&](const auto& f) {
    return launch(ctx, "divrem_top_inv", divrem_top_inv_kernel<std::decay_t<decltype(f)>>, grid_for(ctx, batch, 256), 256, 0, false,
                  f, b, db, batch, out, (size_t)2, true);
  });
}

}  // namespace ronk
