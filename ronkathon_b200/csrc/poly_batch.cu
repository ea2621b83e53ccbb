// poly_batch.cu — Polynomial::mul (src/polynomial/arithmetic.rs:97-119) of many row pairs in one call
// (ronk_poly_mul_batch_u64).  Every row holds the words ronk_poly_mul_u64 gives for its pair.  The path is chosen once per
// call from (p, g, da, db):
//   fused      N = 2^⌈log2 L⌉ ≤ 2^kFusedMaxLog divides p - 1: one launch of polymul_fused_kernel for the whole batch;
//   long       a larger N (≤ 2^26) divides p - 1: pad kernel, batched forward transforms (the second with the point-wise
//              product fused in), batched inverse, clip kernel;
//   crt        no power of two ≥ L divides p - 1: crt_reduce, the two paths above over each auxiliary prime, crt_combine
//              (poly_crt.cu);
//   schoolbook g = 0, L > 2^26, or below the crossovers: poly_mul_schoolbook_kernel over batch·L outputs (poly.cu).
#include <algorithm>
#include <type_traits>

#include "crt.cuh"
#include "polymul_kernel.cuh"
#include "ronk_internal.h"

namespace ronk {

// The crossovers, in da·db per N·log2 N (the schoolbook kernel's work against the size of the transforms): the transform
// path runs from da·db ≥ this·N·log2 N.  tools/poly_mul_batch_timing.py on an H100 80GB HBM3 at 700 W (DESIGN.md §5), at
// da = db and 2^22 output words per call; each constant is da·db / (N·log2 N) of the smallest da from which the transform
// path won at every larger da measured.
// Goldilocks policy: fused from da = 8 (0.107 vs 0.137 ms; da = 4: 0.110 vs 0.091).  Montgomery policy (BabyBear): from
// da = 4 (0.141 vs 0.212 ms; da = 2: 0.131 vs 0.118).  Multi-modular, k = 1 (p = 101) and k = 2 (2^31 - 1): from da = 8,
// the smallest da timed (0.127 vs 0.281 and 0.277 vs 0.283 ms); k = 3 (2^64 - 279): from da = 32 (0.609 vs 0.658 ms;
// da = 16: 0.583 vs 0.434), so between 1.6 and 2.67.
constexpr double kBatchSchoolPerPointGl = 1.0, kBatchSchoolPerPointMont = 0.6;
constexpr double kBatchCrtSchoolPerPoint[kCrtPrimes] = {1.0, 1.0, 2.0};
// Fused up to 2^11 points (its shared-memory cap), the batched transforms above: the fused kernel won at every L it
// covers, 2^8 … 2^11 (Goldilocks 0.135 … 0.192 ms against 0.270 … 0.296 ms for the batched transforms; BabyBear 0.229 …
// 0.273 against 0.319 … 0.378 ms).
constexpr u32 kFusedMaxLog = PM_MAX_LOG;

// Envelope (RONK_EUNSUPPORTED outside): da, db ≤ 2^32; batch·da, batch·db and batch·L ≤ 2^40 words; batch·N ≤ 2^32
// words wherever the batched transforms run.
constexpr u64 kBatchMaxWords = (u64)1 << 40, kBatchMaxTransformWords = (u64)1 << 32;

// dst[r·N + k] = k < d ? src[r·stride + k] : 0, over total = rows·N words.
__global__ void __launch_bounds__(PAD_THREADS)
poly_rows_pad_kernel(const u64* __restrict__ src, u32 d, u64 stride, u32 log_n, u64 total, u64* __restrict__ dst) {
  const u64 step = (u64)gridDim.x * blockDim.x, M = ((u64)1 << log_n) - 1;
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += step) {
    const u64 k = i & M;
    dst[i] = k < d ? src[(i >> log_n) * stride + k] : 0ULL;
  }
}

// dst[r·L + k] = src[r·N + k], k < L, over total = rows·L words.
__global__ void __launch_bounds__(PAD_THREADS)
poly_rows_clip_kernel(const u64* __restrict__ src, u32 log_n, u64 L, u64 total, u64* __restrict__ dst) {
  const u64 step = (u64)gridDim.x * blockDim.x;
  for (u64 o = (u64)blockIdx.x * blockDim.x + threadIdx.x; o < total; o += step) {
    const u64 r = o / L;
    dst[o] = src[(r << log_n) + (o - r * L)];
  }
}

static bool fused_fits(const ronk_ctx* ctx, u32 log_n) {
  return log_n >= 1 && log_n <= kFusedMaxLog && ctx->tune.poly_batch_path != 3;
}

size_t poly_mul_rows_pow2_scratch(const ronk_ctx* ctx, size_t da, size_t db, bool b_shared, u32 batch) {
  const u32 log_n = log2_ceil(da + db - 1);
  if (fused_fits(ctx, log_n)) return 0;
  const size_t n = (size_t)1 << log_n, rows = (size_t)batch << log_n;
  return 2 * rows + (b_shared ? n : rows) + 3 * Frame::kAlign / 8;  // A, B, and the transforms' workspace
}

static int rows_fused(ronk_ctx* ctx, u64 q, u64 g, const u64* a, size_t da, const u64* b, size_t db, bool b_shared, u32 batch,
                      u64* c, u32 log_n) {
  const u64 *twf = nullptr, *twi = nullptr;
  u64 scale = 0, tiles = 0;
  RONK_TRY(ntt_single_tables(ctx, q, g, log_n, &twf, &twi, &scale));
  const PolyMulArgs A = polymul_args(a, (u32)da, b, (u32)db, b_shared, batch, c, log_n, twf, twi, scale, &tiles);
  const size_t smem = ((size_t)2 << PM_TILE_LOG) * sizeof(u64) + (size_t)2 * A.R.tw_words * sizeof(u64) + 16;
  u32 off[4];
  const size_t smem_max = ((size_t)2 << PM_TILE_LOG) * sizeof(u64) + (size_t)2 * ntt_tw2d_layout(PM_MAX_LOG, off) * sizeof(u64) + 16;
  return with_field(ctx, q, g, false, [&](const auto& ff) {
    using F = std::decay_t<decltype(ff)>;
    F fi = ff;
    if constexpr (std::is_same<F, MontField>::value) RONK_TRY(make_mont_field(ctx, q, g, true, &fi));
    RONK_TRY(ensure_smem_attr(ctx, polymul_fused_kernel<F>, (int)smem_max));
    return launch(ctx, "poly_mul_fused", polymul_fused_kernel<F>, (u32)tiles, PM_THREADS, smem, false, ff, fi, A);
  });
}

static int rows_long(ronk_ctx* ctx, u64 q, u64 g, const u64* a, size_t da, const u64* b, size_t db, bool b_shared, u32 batch,
                     u64* c, u32 log_n) {
  const size_t n = (size_t)1 << log_n, rows = (size_t)batch << log_n, L = da + db - 1;
  Frame fr(ctx);
  u64 *A = nullptr, *B = nullptr;
  RONK_TRY(fr.take(&A, rows));
  RONK_TRY(fr.take(&B, b_shared ? n : rows));
  const int pad_grid = grid_for(ctx, rows, PAD_THREADS);
  RONK_TRY(launch(ctx, "poly_rows_pad", poly_rows_pad_kernel, pad_grid, PAD_THREADS, 0, false, a, (u32)da, (u64)da, log_n,
                  (u64)rows, A));
  u64* prod = A;
  if (b_shared) {
    RONK_TRY(ntt_device_bounded(ctx, q, g, b, db, B, n, nullptr, log_n, 0));  // b̂, once
    RONK_TRY(ntt_device_shared_mul(ctx, q, g, A, A, B, log_n, batch));       // â[r] ⊙ b̂ with the n-word mask
  } else {
    RONK_TRY(launch(ctx, "poly_rows_pad", poly_rows_pad_kernel, pad_grid, PAD_THREADS, 0, false, b, (u32)db, (u64)db, log_n,
                    (u64)rows, B));
    RONK_TRY(ntt_device(ctx, q, g, A, nullptr, log_n, batch, 0));  // â
    RONK_TRY(ntt_device(ctx, q, g, B, A, log_n, batch, 0));        // b̂ ⊙ â fused into the last pass
    prod = B;
  }
  RONK_TRY(ntt_device(ctx, q, g, prod, nullptr, log_n, batch, 1));
  const u64 total = (u64)batch * L;
  return launch(ctx, "poly_rows_clip", poly_rows_clip_kernel, grid_for(ctx, total, PAD_THREADS), PAD_THREADS, 0, false, prod,
                log_n, (u64)L, total, c);
}

int poly_mul_rows_pow2(ronk_ctx* ctx, u64 q, u64 g, const u64* a, size_t da, const u64* b, size_t db, bool b_shared,
                       u32 batch, u64* c) {
  const u32 log_n = log2_ceil(da + db - 1);
  if (fused_fits(ctx, log_n)) return rows_fused(ctx, q, g, a, da, b, db, b_shared, batch, c, log_n);
  return rows_long(ctx, q, g, a, da, b, db, b_shared, batch, c, log_n);
}

enum BatchPath { BP_SCHOOL, BP_POW2, BP_CRT };

static BatchPath batch_path(const ronk_ctx* ctx, u64 p, u64 g, size_t da, size_t db) {
  const size_t L = da + db - 1;
  const u32 log_n = log2_ceil(L);
  const bool fits = g != 0 && log_n >= 1 && L <= kCrtMulMaxLen;
  const bool pow2 = fits && pow2_fits(p, log_n);
  if (!fits) return BP_SCHOOL;
  const int forced = ctx->tune.poly_batch_path;
  if (forced == 1) return BP_SCHOOL;
  if (forced >= 2) return pow2 ? BP_POW2 : BP_CRT;
  const double work = (double)da * (double)db, size = (double)((u64)1 << log_n) * (double)log_n;
  if (pow2) {
    const double per_point = p == GL_P && g == 7 ? kBatchSchoolPerPointGl : kBatchSchoolPerPointMont;  // with_field's choice
    return work >= per_point * size ? BP_POW2 : BP_SCHOOL;
  }
  const int k = crt_prime_count(p, std::min(da, db));
  return work >= kBatchCrtSchoolPerPoint[k - 1] * size ? BP_CRT : BP_SCHOOL;
}

static int poly_mul_batch_device(ronk_ctx* ctx, u64 p, u64 g, const u64* a, size_t da, const u64* b, size_t db, bool b_shared,
                                 u32 batch, u64* c) {
  if (!ctx || !a || !b || !c) return set_err(ctx, RONK_EINVAL, "null argument");
  if (da == 0 || db == 0) return set_err(ctx, RONK_EINVAL, "empty polynomial (D + D2 - 1 underflows)");
  RONK_TRY(validate_modulus(ctx, p));
  if (g >= p) return set_err(ctx, RONK_EINVAL, "generator out of range");
  if (da > ((u64)1 << 32) || db > ((u64)1 << 32)) return set_err(ctx, RONK_EUNSUPPORTED, "rows longer than 2^32 words");
  const u64 L = da + db - 1, na = (u64)batch * da, nb = b_shared ? db : (u64)batch * db, total = (u64)batch * L;
  if (na > kBatchMaxWords || nb > kBatchMaxWords || total > kBatchMaxWords)
    return set_err(ctx, RONK_EUNSUPPORTED, "more than 2^40 words in one operand or in the product");
  const BatchPath path = batch_path(ctx, p, g, da, db);
  const u32 log_n = log2_ceil(L);
  if (path != BP_SCHOOL && !fused_fits(ctx, log_n) && ((u64)batch << log_n) > kBatchMaxTransformWords)
    return set_err(ctx, RONK_EUNSUPPORTED, "more than 2^32 words of batched transforms");
  if (overlaps(c, total, a, na) || overlaps(c, total, b, nb)) return set_err(ctx, RONK_EINVAL, "c may not overlap a or b");
  if (batch == 0) return RONK_OK;
  if (path == BP_SCHOOL) return poly_mul_schoolbook_rows(ctx, p, a, da, b, db, b_shared ? 0 : db, batch, c);
  {  // all the call's scratch, before anything is enqueued: the takes below then fit the blocks this one leaves
    Frame fr(ctx);
    u64* all = nullptr;
    const size_t words = path == BP_POW2 ? poly_mul_rows_pow2_scratch(ctx, da, db, b_shared, batch)
                                         : crt_mul_rows_scratch(ctx, p, da, db, b_shared, batch);
    if (words) RONK_TRY(fr.take(&all, words));
  }
  if (path == BP_POW2) return poly_mul_rows_pow2(ctx, p, g, a, da, b, db, b_shared, batch, c);
  return crt_mul_rows_device(ctx, p, a, da, b, db, b_shared, batch, c);
}

}  // namespace ronk

using namespace ronk;

extern "C" {

int ronk_poly_mul_batch_u64(ronk_ctx* ctx, uint64_t p, uint64_t g, const uint64_t* a, size_t da, const uint64_t* b, size_t db,
                            int b_shared, uint32_t batch, uint64_t* c) {
  ronk::DeviceGuard _dg(ctx);
  return poly_mul_batch_device(ctx, p, g, (const u64*)a, da, (const u64*)b, db, b_shared != 0, batch, (u64*)c);
}

// Host pointers: the device function's checks that staging needs come first (a null argument cannot be uploaded, an
// oversized one is refused before it is copied).
int ronk_poly_mul_batch_u64_host(ronk_ctx* ctx, uint64_t p, uint64_t g, const uint64_t* a, size_t da, const uint64_t* b,
                                 size_t db, int b_shared, uint32_t batch, uint64_t* c) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx || !a || !b || !c) return set_err(ctx, RONK_EINVAL, "null argument");
  if (da == 0 || db == 0) return set_err(ctx, RONK_EINVAL, "empty polynomial (D + D2 - 1 underflows)");
  if (da > ((u64)1 << 32) || db > ((u64)1 << 32)) return set_err(ctx, RONK_EUNSUPPORTED, "rows longer than 2^32 words");
  const u64 na = (u64)batch * da, nb = b_shared ? db : (u64)batch * db, total = (u64)batch * (da + db - 1);
  if (na > kBatchMaxWords || nb > kBatchMaxWords || total > kBatchMaxWords)
    return set_err(ctx, RONK_EUNSUPPORTED, "more than 2^40 words in one operand or in the product");
  if (batch == 0) {
    RONK_TRY(validate_modulus(ctx, p));
    return g >= p ? set_err(ctx, RONK_EINVAL, "generator out of range") : RONK_OK;
  }
  Staged s[] = {{na * 8, a}, {nb * 8, b}, {total * 8, nullptr, c}};
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  return stage_out(ctx, poly_mul_batch_device(ctx, p, g, s[0].dev, da, s[1].dev, db, b_shared != 0, batch, s[2].dev), s);
}

}  // extern "C"
