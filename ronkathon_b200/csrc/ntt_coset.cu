// ntt_coset.cu — transforms on a coset s·H_n of the power-of-two subgroup H_n = {ω_n^k}, and the low-degree extension
// built on them (ronk_ntt_coset_u64, ronk_poly_lde_u64 and their _host twins, include/ronk_b200.h).
//   forward  X[k] = Σ_j a_j (s·ω_n^k)^j           = NTT(a ⊙ s^j)
//   inverse  a_j  = s^-j · n^-1 Σ_k X_k ω_n^(-jk)  = INTT(X) ⊙ s^-j
// The factor s^±j rides on the load of the transform's first pass or the store of its last (ntt.cu, run_ntt), so a coset
// transform moves the same bytes as the plain one; its only extra launch builds the two O(√n)-word factor tables.
#include "ronk_internal.h"

namespace ronk {

// batch·N bound of the LDE, as for the batched transforms of ronk_poly_mul_batch_u64
constexpr u64 kLdeMaxWords = (u64)1 << 32;

// The checks of ronk_ntt_u64 (same codes, same order), then the shift.
static int coset_args(ronk_ctx* ctx, u64 p, u64 g, const void* data, u32 log_n, u64 shift) {
  if (!ctx || !data) return set_err(ctx, RONK_EINVAL, "null argument");
  RONK_TRY(validate_modulus(ctx, p));
  if (g == 0 || g >= p) return set_err(ctx, RONK_EINVAL, "generator out of range");
  if (log_n >= 64 || (p - 1) % ((u64)1 << log_n) != 0)
    return set_err(ctx, RONK_EINVAL, "n must divide p - 1 (no primitive n-th root of unity)");
  if (log_n > 26) return set_err(ctx, RONK_EUNSUPPORTED, "log_n > 26 not supported");
  if (shift == 0 || shift >= p) return set_err(ctx, RONK_EINVAL, "shift must be in [1, p)");
  return RONK_OK;
}

// Every word a coset transform of batch × 2^log_n takes from the scratch (the factor tables and the transform's workspace),
// taken once and given back, so that the takes of the call fit the blocks it leaves and nothing is enqueued before a
// failed allocation.
static int reserve_scratch(ronk_ctx* ctx, u32 log_n, u32 batch, u64 shift) {
  const u32 h = (log_n + 1) / 2;
  const size_t tables = shift == 1 ? 0 : ((size_t)1 << h) + ((size_t)1 << (log_n - h));
  Frame fr(ctx);
  u64* all = nullptr;
  return fr.take(&all, tables + ntt_workspace_words(log_n, batch) + 2 * Frame::kAlign / 8);
}

static int ntt_coset_device(ronk_ctx* ctx, u64 p, u64 g, u64* data, u32 log_n, u32 batch, u64 shift, int inverse) {
  RONK_TRY(coset_args(ctx, p, g, data, log_n, shift));
  if (batch == 0 || log_n == 0) return RONK_OK;
  if (shift == 1) return ntt_device(ctx, p, g, data, nullptr, log_n, batch, inverse);
  RONK_TRY(reserve_scratch(ctx, log_n, batch, shift));
  return ntt_device_coset(ctx, p, g, data, log_n, batch, shift, inverse);
}

// The LDE's checks, in the order the header states; `out` stands for the data pointer of coset_args.
static int lde_args(ronk_ctx* ctx, u64 p, u64 g, const void* coeffs, size_t d, u32 log_n, u64 shift, u32 batch,
                    const void* out) {
  if (!ctx || !coeffs || !out) return set_err(ctx, RONK_EINVAL, "null argument");
  RONK_TRY(coset_args(ctx, p, g, out, log_n, shift));
  if (d == 0 || d > ((u64)1 << log_n)) return set_err(ctx, RONK_EINVAL, "d must be in [1, 2^log_n]");
  if (((u64)batch << log_n) > kLdeMaxWords) return set_err(ctx, RONK_EUNSUPPORTED, "more than 2^32 words of output");
  if (overlaps((const u64*)out, (size_t)batch << log_n, (const u64*)coeffs, (size_t)batch * d))
    return set_err(ctx, RONK_EINVAL, "out may not overlap coeffs");
  return RONK_OK;
}

static int lde_device(ronk_ctx* ctx, u64 p, u64 g, const u64* coeffs, size_t d, u32 log_n, u64 shift, u32 batch, u64* out) {
  RONK_TRY(lde_args(ctx, p, g, coeffs, d, log_n, shift, batch, out));
  if (batch == 0) return RONK_OK;
  RONK_TRY(reserve_scratch(ctx, log_n, batch, shift));
  const u64 total = (u64)batch << log_n;
  RONK_TRY(launch(ctx, "lde_pad", poly_rows_pad_kernel, grid_for(ctx, total, PAD_THREADS), PAD_THREADS, 0, false, coeffs,
                  (u32)d, (u64)d, log_n, total, out));
  if (log_n == 0) return RONK_OK;
  if (shift == 1) return ntt_device(ctx, p, g, out, nullptr, log_n, batch, 0);
  return ntt_device_coset(ctx, p, g, out, log_n, batch, shift, 0);
}

}  // namespace ronk

using namespace ronk;

extern "C" {

int ronk_ntt_coset_u64(ronk_ctx* ctx, uint64_t p, uint64_t g, uint64_t* data, uint32_t log_n, uint32_t batch,
                       uint64_t shift, int inverse) {
  ronk::DeviceGuard _dg(ctx);
  return ntt_coset_device(ctx, p, g, (u64*)data, log_n, batch, shift, inverse);
}

int ronk_ntt_coset_u64_host(ronk_ctx* ctx, uint64_t p, uint64_t g, uint64_t* host_data, uint32_t log_n, uint32_t batch,
                            uint64_t shift, int inverse) {
  ronk::DeviceGuard _dg(ctx);
  RONK_TRY(coset_args(ctx, p, g, host_data, log_n, shift));  // before staging: a refused call copies nothing
  if (batch == 0) return RONK_OK;
  Staged s[] = {{((size_t)batch << log_n) * 8, host_data, host_data}};
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  return stage_out(ctx, ntt_coset_device(ctx, p, g, s[0].dev, log_n, batch, shift, inverse), s);
}

int ronk_poly_lde_u64(ronk_ctx* ctx, uint64_t p, uint64_t g, const uint64_t* coeffs, size_t d, uint32_t log_n, uint64_t shift,
                      uint32_t batch, uint64_t* out) {
  ronk::DeviceGuard _dg(ctx);
  return lde_device(ctx, p, g, (const u64*)coeffs, d, log_n, shift, batch, (u64*)out);
}

int ronk_poly_lde_u64_host(ronk_ctx* ctx, uint64_t p, uint64_t g, const uint64_t* coeffs, size_t d, uint32_t log_n,
                           uint64_t shift, uint32_t batch, uint64_t* out) {
  ronk::DeviceGuard _dg(ctx);
  RONK_TRY(lde_args(ctx, p, g, coeffs, d, log_n, shift, batch, out));  // the host buffers, before staging
  if (batch == 0) return RONK_OK;
  Staged s[] = {{(size_t)batch * d * 8, coeffs}, {((size_t)batch << log_n) * 8, nullptr, out}};
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  return stage_out(ctx, lde_device(ctx, p, g, s[0].dev, d, log_n, shift, batch, s[1].dev), s);
}

}  // extern "C"
