// poly_crt.cu — Polynomial::mul over a prime without power-of-two roots of the product's length
// (src/polynomial/arithmetic.rs:97-119): the operands' integer coefficients are convolved modulo k ≤ 3 auxiliary NTT
// primes on the power-of-two transforms, and each coefficient is rebuilt by the Chinese remainder theorem and reduced
// mod p (crt.cuh).  The words are those of the schoolbook kernel, in O(n log n).
#include <algorithm>

#include "crt.cuh"
#include "ronk_internal.h"

namespace ronk {

constexpr int CRT_THREADS = 256;

// The operands' copies modulo an auxiliary prime q below p: ra[0, da) = a mod q, rb[0, db) = b mod q.
__global__ void __launch_bounds__(CRT_THREADS)
crt_reduce_kernel(u64 q, const u64* __restrict__ a, size_t da, u64* __restrict__ ra, const u64* __restrict__ b, size_t db,
                  u64* __restrict__ rb) {
  const size_t n = da > db ? da : db, stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    if (i < da) ra[i] = crt_below(a[i], q);
    if (i < db) rb[i] = crt_below(b[i], q);
  }
}

// c[i] = the coefficient whose residues are C[i], C[L + i], C[2L + i] (K of them), mod p.
template <class F, int K>
__global__ void __launch_bounds__(CRT_THREADS)
crt_combine_kernel(const F f, const CrtConsts k, const u64* __restrict__ C, size_t L, u64* __restrict__ c) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < L; i += stride) {
    const u64 c2 = K >= 2 ? C[L + i] : 0ULL, c3 = K >= 3 ? C[2 * L + i] : 0ULL;
    c[i] = crt_garner<K>(f, k, C[i], c2, c3);
  }
}

// The measured crossovers, per prime count: tools/crt_mul_timing.py on an H100 80GB HBM3 at 700 W (DESIGN.md §5).
// kCrtMulMin: at da = db = 2^6 … 2^16, the smallest da·db from which the multi-modular path won over the schoolbook kernel
// at every larger size (k = 1, p = 101: 2^8 × 2^8, 0.048 vs 0.060 ms; k = 2, p = 2^31 - 1: 2^10 × 2^10, 0.082 vs 0.178
// ms; k = 3, p = 2^64 - 279: 2^10 × 2^10, 0.142 vs 0.191 ms).
// kCrtMulShortMin: the schoolbook kernel does min(da, db) multiplies per coefficient, the multi-modular path about
// k·log2(L) whatever the shape, so a short operand keeps the schoolbook kernel ahead at any length (2 × 2^20 over
// 2^64 - 279: 0.035 vs 0.84 ms).  At da = 2^0 … 2^12 against db = 2^16, 2^20 and 2^24, the smallest da from which the
// multi-modular path won at every larger da, for every db (k = 1: 256 at db = 2^16; k = 2: 512 at 2^16; k = 3: 1024 at
// 2^16).  RONK_CRT_MUL_MIN replaces both.
constexpr u64 kCrtMulMin[kCrtPrimes] = {(u64)1 << 16, (u64)1 << 20, (u64)1 << 20};
constexpr size_t kCrtMulShortMin[kCrtPrimes] = {256, 512, 1024};

bool crt_mul_fits(const ronk_ctx* ctx, u64 p, u64 g, size_t da, size_t db) {
  const size_t L = da + db - 1;
  if (g == 0 || L > kCrtMulMaxLen) return false;
  if (pow2_fits(p, log2_ceil(L))) return false;  // the direct transform fits
  const u64 work = (u64)da * (u64)db;             // da, db ≤ L ≤ 2^26: no overflow
  const long long forced = ctx->tune.crt_mul_min;
  if (forced >= 0) return work >= (u64)forced;
  const size_t m = std::min(da, db);
  const int k = crt_prime_count(p, m);
  return work >= kCrtMulMin[k - 1] && m >= kCrtMulShortMin[k - 1];
}

static int crt_reduce(ronk_ctx* ctx, u64 q, const u64* a, size_t na, u64* ra, const u64* b, size_t nb, u64* rb) {
  return launch(ctx, "crt_reduce", crt_reduce_kernel, grid_for(ctx, std::max(na, nb), CRT_THREADS), CRT_THREADS, 0, false, q,
                a, na, ra, b, nb, rb);
}

// c[0, len) mod p from the K residue vectors C[i·len, (i + 1)·len), i < K.
static int crt_combine(ronk_ctx* ctx, u64 p, int K, const u64* C, size_t len, u64* c) {
  return with_field(ctx, p, 0, false, [&](const auto& f) {
    using F = std::decay_t<decltype(f)>;
    const CrtConsts k = crt_consts(f);
    const int grid = grid_for(ctx, len, CRT_THREADS);
    switch (K) {
      case 1: return launch(ctx, "crt_combine", crt_combine_kernel<F, 1>, grid, CRT_THREADS, 0, false, f, k, C, len, c);
      case 2: return launch(ctx, "crt_combine", crt_combine_kernel<F, 2>, grid, CRT_THREADS, 0, false, f, k, C, len, c);
      default: return launch(ctx, "crt_combine", crt_combine_kernel<F, 3>, grid, CRT_THREADS, 0, false, f, k, C, len, c);
    }
  });
}

// Per auxiliary prime q_i: [reduce a into B and b into C_i when q_i < p], Â into A, B̂ ⊙ Â into B, the inverse into C_i
// (L words).  Then crt_combine writes c.  a and b are read only before it, so c may alias them, as on the direct path.
int crt_mul_device(ronk_ctx* ctx, u64 p, const u64* a, size_t da, const u64* b, size_t db, u64* c) {
  const size_t L = da + db - 1;
  const u32 log_n = log2_ceil(L);
  const size_t n = (size_t)1 << log_n;
  const int K = crt_prime_count(p, std::min(da, db));
  Frame fr(ctx);
  u64* A = nullptr;
  RONK_TRY(fr.take(&A, 2 * n + (size_t)K * L));
  u64* B = A + n;
  u64* C = B + n;
  for (int i = 0; i < K; i++) {
    const u64 q = kCrtQ[i];
    u64* Ci = C + (size_t)i * L;
    const u64 *sa = a, *sb = b;
    if (q < p) {
      RONK_TRY(crt_reduce(ctx, q, a, da, B, b, db, Ci));
      sa = B;
      sb = Ci;
    }
    RONK_TRY(product_bounded(ctx, q, kCrtG[i], sa, da, sb, db, log_n, A, B, Ci, L));  // residues mod q_i, L of them
  }
  return crt_combine(ctx, p, K, C, L, c);
}

// The same path over `batch` contiguous rows (ronk_poly_mul_batch_u64): one crt_reduce over the flat batch·da and
// batch·db (db when shared) words where q_i < p, the batched product over q_i into C_i (batch·L words), one crt_combine
// over batch·L words.
size_t crt_mul_rows_scratch(const ronk_ctx* ctx, u64 p, size_t da, size_t db, bool b_shared, u32 batch) {
  const size_t L = da + db - 1, nb = b_shared ? db : (size_t)batch * db;
  const int K = crt_prime_count(p, std::min(da, db));
  size_t w = (size_t)K * batch * L;
  bool reduce = false;
  for (int i = 0; i < K; i++) reduce = reduce || kCrtQ[i] < p;
  if (reduce) w += (size_t)batch * da + nb;
  return w + poly_mul_rows_pow2_scratch(ctx, da, db, b_shared, batch) + 3 * Frame::kAlign / 8;
}

int crt_mul_rows_device(ronk_ctx* ctx, u64 p, const u64* a, size_t da, const u64* b, size_t db, bool b_shared, u32 batch,
                        u64* c) {
  const size_t L = da + db - 1, na = (size_t)batch * da, nb = b_shared ? db : (size_t)batch * db, total = (size_t)batch * L;
  const int K = crt_prime_count(p, std::min(da, db));
  Frame fr(ctx);
  u64* C = nullptr;
  RONK_TRY(fr.take(&C, (size_t)K * total));
  u64 *ra = nullptr, *rb = nullptr;
  for (int i = 0; i < K; i++) {
    const u64 q = kCrtQ[i], g = kCrtG[i];
    const u64 *sa = a, *sb = b;
    if (q < p) {
      if (!ra) {
        RONK_TRY(fr.take(&ra, na));
        RONK_TRY(fr.take(&rb, nb));
      }
      RONK_TRY(crt_reduce(ctx, q, a, na, ra, b, nb, rb));
      sa = ra;
      sb = rb;
    }
    RONK_TRY(poly_mul_rows_pow2(ctx, q, g, sa, da, sb, db, b_shared, batch, C + (size_t)i * total));
  }
  return crt_combine(ctx, p, K, C, total, c);
}

}  // namespace ronk
