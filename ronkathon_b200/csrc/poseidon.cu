// poseidon.cu — batches of the reference's Poseidon permutation and sponge (src/hashes/poseidon/{mod,sponge}.rs):
// ronk_poseidon_permute_u64, ronk_poseidon_sponge_u64 and their _host twins (include/ronk_b200.h).
//
// poseidon_rows_kernel<F, T>, one launch per call: one thread per row, grid-stride.  Each CTA first copies the round
// constants and the MDS matrix into shared memory in the policy's twiddle form (poseidon.cuh); every thread of a warp
// then reads the same constant at the same time, which shared memory broadcasts.  The constants travel as kernel
// arguments and device buffers, never through a __constant__ symbol, so concurrent contexts and streams never share
// them.  Widths 2 … 16 × the two field policies are the 30 instantiations.  A permutation is the sponge row of rate =
// width that absorbs and squeezes the row's width words in place (poseidon.cuh), so both entries run the same kernel.
#include "poseidon.cuh"
#include "ronk_internal.h"

namespace ronk {

constexpr int POS_THREADS = 128;
constexpr u64 POS_MAX_WORDS = (u64)1 << 40;

template <class F, int T>
__global__ void __launch_bounds__(POS_THREADS)
poseidon_rows_kernel(F f, PosRounds r, const u64* __restrict__ rc_g, const u64* __restrict__ mds_g, u32 rate,
                     const u64* in, u64 len, u64* out, u64 n_out, u64 batch) {
  extern __shared__ u64 pos_smem[];
  u64* mds = pos_smem;              // [T²]
  u64* rc = pos_smem + T * T;       // [R·T]
  const u32 n_rc = r.rounds * T, n_mds = r.rounds ? T * T : 0;  // zero rounds read neither table
  for (u32 i = threadIdx.x; i < n_mds; i += POS_THREADS) mds[i] = f.to_tw(mds_g[i]);
  for (u32 i = threadIdx.x; i < n_rc; i += POS_THREADS) rc[i] = f.to_tw(rc_g[i]);
  __syncthreads();
  const u64 stride = (u64)gridDim.x * POS_THREADS;
  for (u64 y = (u64)blockIdx.x * POS_THREADS + threadIdx.x; y < batch; y += stride) {
    pos_sponge_row<F, T>(f, r, rc, mds, rate, in + y * len, len, out + y * n_out, n_out);
  }
}

// Step (1) of both entries' errors, which reads no pointer; on RONK_OK *r holds the round structure.  sponge: rate, in,
// len, out and n_out are the sponge's; otherwise out holds the states and rate, in, len, n_out are unused.
static int poseidon_args(ronk_ctx* ctx, u64 p, u32 width, u64 alpha, u32 num_f, u32 num_p, const u64* rc, const u64* mds,
                         bool sponge, u32 rate, const u64* in, u64 len, const u64* out, u64 n_out, u64 batch, PosRounds* r) {
  if (!ctx) return RONK_EINVAL;
  const u64 rounds = (u64)num_f + num_p;
  const bool null_arg = sponge ? (batch && len && !in) || (batch && n_out && !out) : (batch && !out);
  if (null_arg || (batch && rounds && (!rc || !mds))) return set_err(ctx, RONK_EINVAL, "null argument");
  RONK_TRY(validate_modulus(ctx, p));
  if (width < (u32)POS_MIN_WIDTH) return set_err(ctx, RONK_EINVAL, "hash width should be greater than 1 (poseidon/mod.rs:47)");
  if (sponge && (rate == 0 || rate > width)) return set_err(ctx, RONK_EINVAL, "rate must be in [1, width]");
  if (width > (u32)POS_MAX_WIDTH) return set_err(ctx, RONK_EUNSUPPORTED, "width above 16");
  if (rounds * width + (u64)width * width > POS_MAX_CONST_WORDS)
    return set_err(ctx, RONK_EUNSUPPORTED, "(num_f + num_p)·width + width² above 6144 words of constants");
  const unsigned __int128 b = batch;
  if (b * width > POS_MAX_WORDS || (sponge && (b * len > POS_MAX_WORDS || b * n_out > POS_MAX_WORDS)))
    return set_err(ctx, RONK_EUNSUPPORTED, "more than 2^40 words in a buffer");
  r->rounds = (u32)rounds;
  r->full_lo = num_f / 2;
  r->full_hi = num_p + num_f / 2;
  r->alpha = alpha;
  return RONK_OK;
}

// Step (2): the output may not overlap the constants or (sponge) the input.
static int poseidon_overlap(ronk_ctx* ctx, u32 width, const PosRounds& r, const u64* rc, const u64* mds, const u64* in,
                            u64 in_words, const u64* out, u64 out_words) {
  const size_t n_mds = r.rounds ? (size_t)width * width : 0;
  if (overlaps(out, out_words, rc, (size_t)r.rounds * width) || overlaps(out, out_words, mds, n_mds) ||
      overlaps(out, out_words, in, in_words))
    return set_err(ctx, RONK_EINVAL, "the output may not overlap rc, mds or the input");
  return RONK_OK;
}

static int poseidon_launch(ronk_ctx* ctx, const char* name, u64 p, u32 width, const PosRounds& r, const u64* rc,
                           const u64* mds, u32 rate, const u64* in, u64 len, u64* out, u64 n_out, u64 batch) {
  const size_t smem = ((size_t)r.rounds * width + (size_t)width * width) * sizeof(u64);
  const int grid = grid_for(ctx, batch, POS_THREADS);
  return with_field(ctx, p, 0, false, [&](const auto& f) {
    using F = std::decay_t<decltype(f)>;
    auto go = [&](auto kernel) {
      return launch(ctx, name, kernel, grid, POS_THREADS, smem, false, f, r, rc, mds, rate, in, len, out, n_out, batch);
    };
    switch (width) {
      case 2: return go(poseidon_rows_kernel<F, 2>);
      case 3: return go(poseidon_rows_kernel<F, 3>);
      case 4: return go(poseidon_rows_kernel<F, 4>);
      case 5: return go(poseidon_rows_kernel<F, 5>);
      case 6: return go(poseidon_rows_kernel<F, 6>);
      case 7: return go(poseidon_rows_kernel<F, 7>);
      case 8: return go(poseidon_rows_kernel<F, 8>);
      case 9: return go(poseidon_rows_kernel<F, 9>);
      case 10: return go(poseidon_rows_kernel<F, 10>);
      case 11: return go(poseidon_rows_kernel<F, 11>);
      case 12: return go(poseidon_rows_kernel<F, 12>);
      case 13: return go(poseidon_rows_kernel<F, 13>);
      case 14: return go(poseidon_rows_kernel<F, 14>);
      case 15: return go(poseidon_rows_kernel<F, 15>);
      default: return go(poseidon_rows_kernel<F, 16>);
    }
  });
}

// Whether every one of the n words at x is below p.
static bool canonical(const u64* x, u64 n, u64 p) {
  for (u64 i = 0; i < n; i++)
    if (x[i] >= p) return false;
  return true;
}

}  // namespace ronk

using namespace ronk;

extern "C" {

int ronk_poseidon_permute_u64(ronk_ctx* ctx, uint64_t p, uint32_t width, uint64_t alpha, uint32_t num_f, uint32_t num_p,
                              const uint64_t* rc, const uint64_t* mds, uint64_t* states, size_t batch) {
  ronk::DeviceGuard _dg(ctx);
  PosRounds r;
  RONK_TRY(poseidon_args(ctx, p, width, alpha, num_f, num_p, rc, mds, false, 0, nullptr, 0, states, 0, batch, &r));
  RONK_TRY(poseidon_overlap(ctx, width, r, rc, mds, nullptr, 0, states, (u64)batch * width));
  if (batch == 0) return RONK_OK;
  return poseidon_launch(ctx, "poseidon_permute", p, width, r, rc, mds, width, states, width, states, width, batch);
}

int ronk_poseidon_sponge_u64(ronk_ctx* ctx, uint64_t p, uint32_t width, uint64_t alpha, uint32_t num_f, uint32_t num_p,
                             const uint64_t* rc, const uint64_t* mds, uint32_t rate, const uint64_t* in, size_t len,
                             size_t batch, uint64_t* out, size_t n_out) {
  ronk::DeviceGuard _dg(ctx);
  PosRounds r;
  RONK_TRY(poseidon_args(ctx, p, width, alpha, num_f, num_p, rc, mds, true, rate, in, len, out, n_out, batch, &r));
  RONK_TRY(poseidon_overlap(ctx, width, r, rc, mds, in, (u64)batch * len, out, (u64)batch * n_out));
  if (batch == 0 || n_out == 0) return RONK_OK;
  return poseidon_launch(ctx, "poseidon_sponge", p, width, r, rc, mds, rate, in, len, out, n_out, batch);
}

int ronk_poseidon_permute_u64_host(ronk_ctx* ctx, uint64_t p, uint32_t width, uint64_t alpha, uint32_t num_f,
                                   uint32_t num_p, const uint64_t* rc, const uint64_t* mds, uint64_t* states, size_t batch) {
  ronk::DeviceGuard _dg(ctx);
  PosRounds r;
  RONK_TRY(poseidon_args(ctx, p, width, alpha, num_f, num_p, rc, mds, false, 0, nullptr, 0, states, 0, batch, &r));
  if (batch == 0) return RONK_OK;
  const u64 n_rc = (u64)r.rounds * width, n_mds = r.rounds ? (u64)width * width : 0, words = (u64)batch * width;
  if (!canonical(rc, n_rc, p) || !canonical(mds, n_mds, p) || !canonical(states, words, p))
    return set_err(ctx, RONK_EINVAL, "non-canonical residue");
  Staged s[] = {{n_rc * 8, rc}, {n_mds * 8, mds}, {words * 8, states, states}};
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  return stage_out(ctx, ronk_poseidon_permute_u64(ctx, p, width, alpha, num_f, num_p, s[0].dev, s[1].dev, s[2].dev, batch), s);
}

int ronk_poseidon_sponge_u64_host(ronk_ctx* ctx, uint64_t p, uint32_t width, uint64_t alpha, uint32_t num_f, uint32_t num_p,
                                  const uint64_t* rc, const uint64_t* mds, uint32_t rate, const uint64_t* in, size_t len,
                                  size_t batch, uint64_t* out, size_t n_out) {
  ronk::DeviceGuard _dg(ctx);
  PosRounds r;
  RONK_TRY(poseidon_args(ctx, p, width, alpha, num_f, num_p, rc, mds, true, rate, in, len, out, n_out, batch, &r));
  if (batch == 0) return RONK_OK;
  const u64 n_rc = (u64)r.rounds * width, n_mds = r.rounds ? (u64)width * width : 0, n_in = (u64)batch * len;
  if (!canonical(rc, n_rc, p) || !canonical(mds, n_mds, p) || !canonical(in, n_in, p))
    return set_err(ctx, RONK_EINVAL, "non-canonical residue");
  if (n_out == 0) return RONK_OK;
  Staged s[] = {{n_rc * 8, rc}, {n_mds * 8, mds}, {n_in * 8, in}, {(u64)batch * n_out * 8, nullptr, out}};
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  return stage_out(ctx,
                   ronk_poseidon_sponge_u64(ctx, p, width, alpha, num_f, num_p, s[0].dev, s[1].dev, rate, s[2].dev, len, batch,
                                            s[3].dev, n_out),
                   s);
}

}  // extern "C"
