// ntt.cu — plans (twiddle tables) and launches for the tiled NTT kernel.
// Public entry points: ronk_ntt_u64, ronk_ntt_mul_u64, ronk_ntt_u64_host (include/ronk_b200.h),
// replacing Polynomial::fft / ifft (src/polynomial/mod.rs:273-323, :430-484).
#include <cstdlib>

#include <type_traits>

#include "ntt12_kernel.cuh"
#include "ntt3_kernel.cuh"
#include "ntt_kernel.cuh"
#include "ronk_internal.h"

namespace ronk {

int make_mont_field(ronk_ctx* ctx, u64 p, u64 g, bool inverse, MontField* out) {
  if (!(p & 1) || p < 3) return set_err(ctx, RONK_EUNSUPPORTED, "modulus must be an odd prime");
  MontField f = h_mont_field(p);
  const u64 r1 = f.w16t[0];  // R mod p
  if (g) {
    u32 k = 0;
    while (k < 4 && ((p - 1) >> k) % 2 == 0) k++;
    if (k) {
      u64 w = h_powmod(g, (p - 1) >> k, p);                  // primitive 2^k-th root
      if (inverse) w = h_powmod(w, ((u64)1 << k) - 1, p);    // its inverse
      const int stride = 16 >> k;
      for (int e = 0; e < 8; e++)
        if (e % stride == 0) f.w16t[e] = h_mulmod(h_powmod(w, e / stride, p), r1, p);
    }
  }
  *out = f;
  return RONK_OK;
}

template <class F>
static int build_pow_table(ronk_ctx* ctx, const F& f, u64 w, u64 s, DevBuf<u64>* tab, u32 count) {
  RONK_TRY(tab->alloc(ctx, count));
  return launch(ctx, "pow_table", pow_table_kernel<F>, (count + 255) / 256, 256, 0, false, f, w, s, tab->get(), count);
}

static int build_tw2d(ronk_ctx* ctx, const u64* tw1d, u32 log_m, DevBuf<u64> out2d[2]) {
  u32 off[4];
  const u32 words = ntt_tw2d_layout(log_m, off);
  for (int d = 0; d < 2; d++) {
    RONK_TRY(out2d[d].alloc(ctx, words ? words : 2));
    if (!words) continue;
    RONK_TRY(launch(ctx, "tw2d_gather", tw2d_gather_kernel, (words + 255) / 256, 256, 0, false, tw1d, log_m, d, out2d[d].get(), words));
  }
  return RONK_OK;
}

template <class F>
static int build_plan(ronk_ctx* ctx, const F& f, u64 p, u64 g, u32 log_n, NttPlan* plan) {
  const u64 n = (u64)1 << log_n;
  const u64 w = h_powmod(g, (p - 1) / n, p);
  const u64 ninv = h_powmod(n % p, p - 2, p);
  plan->p = p;
  plan->g = g;
  plan->log_n = log_n;
  const NttShape sh = ntt_shape(log_n);
  if (!sh.two_pass) {
    plan->two_pass = false;
    RONK_TRY(build_pow_table(ctx, f, w, 1, &plan->tw1, (u32)n));
    RONK_TRY(build_tw2d(ctx, plan->tw1.get(), log_n, plan->tw1_2d));
  } else {
    plan->two_pass = true;
    plan->log_n1 = sh.log_n1;
    plan->log_n2 = sh.log_n2;
    const u64 n1 = (u64)1 << plan->log_n1, n2 = (u64)1 << plan->log_n2;
    RONK_TRY(build_pow_table(ctx, f, h_powmod(w, n2, p), 1, &plan->tw1, (u32)n1));
    RONK_TRY(build_pow_table(ctx, f, h_powmod(w, n1, p), 1, &plan->tw2, (u32)n2));
    RONK_TRY(build_pow_table(ctx, f, w, 1, &plan->tw_lo, (u32)n1));
    RONK_TRY(build_pow_table(ctx, f, h_powmod(w, n1, p), ninv, &plan->tw_hi_inv, (u32)n2));
    RONK_TRY(build_tw2d(ctx, plan->tw1.get(), plan->log_n1, plan->tw1_2d));
    RONK_TRY(build_tw2d(ctx, plan->tw2.get(), plan->log_n2, plan->tw2_2d));
  }
  // n^-1 in twiddle form: Goldilocks → plain; Montgomery → ninv·R mod p
  if (p == GL_P && g == 7) plan->scale_inv = ninv;
  else plan->scale_inv = h_mulmod(ninv, (u64)((((unsigned __int128)1) << 64) % p), p);
  return RONK_OK;
}

// n-word table of the inter-pass twiddles for one direction and one workspace layout (log2 C2), built on first use.
// The table is cached in the plan; *out = nullptr where there is no memory for it: the stepped form needs none.
template <class F>
static int interpass_table(ronk_ctx* ctx, const F& f, NttPlan& pl, bool inverse, u32 log_c2, const u64* tw_lo,
                           const u64* tw_hi, const u64** out) {
  DevBuf<u64>& tab = pl.tw_full[inverse ? 1 : 0][log_c2];  // empty until built
  const u64 n = (u64)1 << pl.log_n;
  if (!tab) RONK_TRY(build_table(ctx, &tab, n, [&](u64* t) {
    return launch(ctx, "interpass_table", interpass_table_kernel<F>, (unsigned)((n + 255) / 256), 256, 0, false, f, tw_lo, tw_hi,
                  pl.log_n, pl.log_n1, pl.log_n2, log_c2, pl.log_n1, inverse ? 1 : 0, t);
  }, true));
  *out = tab.get();
  return RONK_OK;
}

template <class F, int MODE, bool INV, int NTHR, int MINB, bool BOUNDED, bool FMUL, bool COSET = false>
static int launch_tile_nb(ronk_ctx* ctx, const F& f, const NttTileArgs& A0, u32 tiles, const char* name) {
  NttTileArgs A = A0;
  if (MODE == MODE_PASS1) A.prefetch_dist = (u32)ctx->tune.pf_dist * (u32)ctx->sm_count * (u32)MINB;
  const size_t smem = ((size_t)1 << A.tile_log) * sizeof(u64) + (size_t)A.tw_words * sizeof(u64) + 16;
  // the attribute is per device: set once per (context, instantiation)
  RONK_TRY(ensure_smem_attr(ctx, ntt_tile_kernel<F, MODE, INV, NTHR, MINB, BOUNDED, FMUL, COSET>, 226 * 1024));
  // pass 2 directly follows its pass 1 on the stream and may start early.  That helps launch-bound jobs (2^14…2^18) and
  // hurts a 2^24 transform (the waiting CTAs start in lockstep), so only small jobs take it
  const bool pdl = MODE == MODE_PASS2 && ctx->tune.pdl && (((u64)tiles << A.tile_log) <= ((u64)1 << 21));
  return launch(ctx, name, ntt_tile_kernel<F, MODE, INV, NTHR, MINB, BOUNDED, FMUL, COSET>, tiles, NTHR, smem, pdl, f, A);
}

// The bounded instantiation exists only where poly_mul needs it: a zero-padded SOURCE enters through
// pass 1 / a single-pass tile, a clipped DESTINATION leaves through pass 2 / a single-pass tile.
template <class F, int MODE, bool INV, int NTHR, int MINB>
static int launch_tile_n(ronk_ctx* ctx, const F& f, const NttTileArgs& A, u32 tiles, const char* name) {
  // a coset transform's hooked pass (forward: the first, inverse: the last) has an instantiation of its own; the other
  // pass is the plain one
  constexpr bool can_coset = MODE == MODE_SINGLE || (MODE == MODE_PASS1) != INV;
  if constexpr (can_coset) {
    if (A.coset_lo) return launch_tile_nb<F, MODE, INV, NTHR, MINB, false, false, true>(ctx, f, A, tiles, name);
  }
  const bool bounded = (MODE != MODE_PASS2 && A.src_len != NTT_UNBOUNDED) || (MODE != MODE_PASS1 && A.dst_len != NTT_UNBOUNDED);
  // the fused point-wise multiply of pass 2 (forward transforms of poly_mul) has its own instantiation too
  constexpr bool can_fmul = MODE == MODE_PASS2 && !INV && ((RONK_STORE_V0_MASK >> MODE_PASS2) & 1);
  const bool fmul = can_fmul && (A.flags & NTT_FLAG_MUL);
  if (can_fmul && fmul) {
    if (bounded) return launch_tile_nb<F, MODE, INV, NTHR, MINB, true, can_fmul>(ctx, f, A, tiles, name);
    return launch_tile_nb<F, MODE, INV, NTHR, MINB, false, can_fmul>(ctx, f, A, tiles, name);
  }
  if (bounded) return launch_tile_nb<F, MODE, INV, NTHR, MINB, true, false>(ctx, f, A, tiles, name);
  return launch_tile_nb<F, MODE, INV, NTHR, MINB, false, false>(ctx, f, A, tiles, name);
}

// The specialised 4096-point-per-tile kernel (ntt12_kernel.cuh): Goldilocks, unbounded, log_m = 12, the default
// tile shapes (pass 1: 4 columns, pass 2: 2 columns).
template <int MODE, bool INV, int LC, bool FMUL>
static int launch12_one(ronk_ctx* ctx, const GoldilocksField& f, const NttTileArgs& A0, u32 tiles, const char* name) {
  using L = N12<LC, MODE>;
  NttTileArgs A = A0;
  if (MODE == MODE_PASS1) A.prefetch_dist = (u32)ctx->tune.pf_dist * (u32)ctx->sm_count * (L::NTHR >= 512 ? 1u : 2u);
  if (MODE == MODE_PASS2) A.prefetch_dist = (u32)ctx->tune.pf_dist2 * (u32)ctx->sm_count * (L::NTHR >= 512 ? 1u : 2u);
  const size_t smem = (size_t)L::TILE_SLOTS * 16 + (size_t)L::TW_WORDS * sizeof(u64) + 16;
  RONK_TRY(ensure_smem_attr(ctx, ntt12_kernel<GoldilocksField, MODE, INV, LC, FMUL>, (int)smem));
  return launch(ctx, name, ntt12_kernel<GoldilocksField, MODE, INV, LC, FMUL>, tiles, L::NTHR, smem, false, f, A);
}
template <int MODE, bool INV>
static int launch12(ronk_ctx* ctx, const GoldilocksField& f, const NttTileArgs& A, u32 tiles, const char* name) {
  if constexpr (MODE == MODE_PASS1) {
    return launch12_one<MODE, INV, 2, false>(ctx, f, A, tiles, name);
  } else {
    if (!INV && (A.flags & NTT_FLAG_MUL)) return launch12_one<MODE, INV, 1, !INV>(ctx, f, A, tiles, name);
    return launch12_one<MODE, INV, 1, false>(ctx, f, A, tiles, name);
  }
}

// CTA shape: every thread owns 32 tile elements per round (two radix-16 groups, ≤128 registers, no
// spills).  A 2^14 tile is one 512-thread CTA per SM; a 2^13 tile is a 256-thread CTA and two of
// them share an SM, so one CTA's load/store phases overlap the other's butterflies.
template <class F, int MODE, bool INV>
static int launch_tile(ronk_ctx* ctx, const F& f, const NttTileArgs& A, u32 tiles, const char* name) {
  if constexpr (std::is_same<F, GoldilocksField>::value && MODE != MODE_SINGLE) {
    if (ctx->tune.fast12 && !A.coset_lo && ntt12_applicable(A, MODE) && !(INV && (A.flags & NTT_FLAG_MUL)))
      return launch12<MODE, INV>(ctx, f, A, tiles, name);
  }
  const u32 groups = (1u << A.tile_log) / 16;
  if (groups >= 1024) return launch_tile_n<F, MODE, INV, 512, 1>(ctx, f, A, tiles, name);
  if (groups >= 512) return launch_tile_n<F, MODE, INV, 256, 2>(ctx, f, A, tiles, name);
  if (groups >= 128) return launch_tile_n<F, MODE, INV, 128, 2>(ctx, f, A, tiles, name);
  return launch_tile_n<F, MODE, INV, 32, 2>(ctx, f, A, tiles, name);
}

// ---- transforms as passes of 256-point tiles (ntt3_kernel.cuh): n = 2^24 (three passes) and n = 2^16 (two) -------
template <class F, int PASS, bool INV, int LOGN, bool BOUNDED, int NG, int LI = 0, bool COSET = false>
static int launch3_ng(ronk_ctx* ctx, const F& f, const Ntt3Args& A, const char* name, bool dependent, unsigned tiles) {
  return launch(ctx, name, ntt3_kernel<F, PASS, INV, LOGN, BOUNDED, NG, LI, COSET>, tiles, N3_THREADS * (2 / NG), 0,
                dependent && ctx->tune.ntt3_pdl, f, A);
}
template <class F, int PASS, bool INV, int LOGN, bool BOUNDED, int LI = 0, bool COSET = false>
static int launch3(ronk_ctx* ctx, const F& f, const Ntt3Args& A, const char* name, bool dependent) {
  const unsigned tiles = A.batch * (LOGN >= 21 ? (1u << (LOGN - 12)) : LOGN == 20 ? 256u : 16u);
  // a grid that leaves most warp slots empty runs one radix-16 group per thread (256 threads per tile): a single
  // 2^16- or 2^20-point transform is a chain of dependent carry chains per warp, and twice the warps halve it
  if constexpr ((LOGN == 16 || LOGN == 20) && !BOUNDED) {
    if (tiles < (unsigned)ctx->tune.ntt3_ng1_tiles * (unsigned)ctx->sm_count)
      return launch3_ng<F, PASS, INV, LOGN, BOUNDED, 1, LI>(ctx, f, A, name, dependent, tiles);
  }
  return launch3_ng<F, PASS, INV, LOGN, BOUNDED, 2, LI, COSET>(ctx, f, A, name, dependent, tiles);
}

// pass C of the 2^20-point transform (ntt3c_kernel): one thread per (transform, k2)
template <class F, bool INV>
static int launch3c(ronk_ctx* ctx, const F& f, const Ntt3Args& A, const char* name) {
  const unsigned blocks = (unsigned)((((u64)A.batch << 16) + N3C_THREADS - 1) / N3C_THREADS);
  return launch(ctx, name, ntt3c_kernel<F, INV>, blocks, N3C_THREADS, 0, ctx->tune.ntt3_pdl, f, A);
}

// first pass of a split transform (ntt3p_kernel): radix 2^LI over the elements n' apart, twiddle, in place
template <class F, bool INV, int LI>
static int launch3p(ronk_ctx* ctx, const F& f, const Ntt3Args& A, u32 log_np, u32 log_lo, const char* name) {
  const u64 threads = (u64)A.batch << (log_np - (4 - LI));
  const unsigned blocks = (unsigned)((threads + N3C_THREADS - 1) / N3C_THREADS);
  return launch(ctx, name, ntt3p_kernel<F, INV, LI>, blocks, N3C_THREADS, 0, false, f, A, log_np, log_lo);
}

// one-time tables of the 256-point-tile kernels for one direction: ω_256^x and the 64 Ki-entry ω_65536^(±k·j) [· n^-1]
template <class F, bool INV>
static int ntt3_tables(ronk_ctx* ctx, const F& f, NttPlan& pl, int log_n) {
  const int d = INV ? 1 : 0;
  if (pl.tw256[d]) return RONK_OK;
  const u64 p = pl.p, n = (u64)1 << log_n;
  u64 w = h_powmod(pl.g, (p - 1) / n, p);
  if (INV) w = h_powmod(w, p - 2, p);
  DevBuf<u64> tw256, t2;
  RONK_TRY(build_tables(ctx, [&] {
    RONK_TRY(build_pow_table(ctx, f, h_powmod(w, n >> 8, p), 1, &tw256, 256));
    RONK_TRY(t2.alloc(ctx, 65536));
    const u64 ninv = INV ? h_powmod(n % p, p - 2, p) : 1;
    return launch(ctx, "ntt3_t2", ntt3_t2_kernel<F>, 256, 256, 0, false, f, h_powmod(w, n >> 16, p), ninv, t2.get());
  }));
  pl.tw256[d] = std::move(tw256);
  pl.t2[d] = std::move(t2);
  return RONK_OK;
}

// Small batches of 2^16-point transforms in ONE launch: a 16-CTA thread-block cluster per transform, the pass-2 → pass-3
// exchange through distributed shared memory (ntt16c_kernel).  In place, no workspace.  Returns RONK_OK with *done = false
// when the device refuses the cluster shape (the caller then takes the two-launch path).
template <class F, bool INV>
static int run_ntt16_cluster(ronk_ctx* ctx, const F& f, NttPlan& pl, u64* data, const u64* src, const u64* mul, u32 batch,
                             bool* done, u64 mul_mask = ~0ULL) {
  *done = false;
  if (ctx->cluster16_state < 0) return RONK_OK;
  RONK_TRY((ntt3_tables<F, INV>(ctx, f, pl, 16)));
  constexpr size_t kSmem = (size_t)(N3_TILE_WORDS + N3_RECV_WORDS) * sizeof(u64);
  auto kern = ntt16c_kernel<F, INV>;
  const void* key = reinterpret_cast<const void*>(kern);
  if (!ctx->smem_attr_done.count(key)) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess) {
      cudaGetLastError();
      ctx->cluster16_state = -1;
      return RONK_OK;
    }
    RONK_TRY(ensure_smem_attr(ctx, kern, (int)kSmem));
  }
  const int d = INV ? 1 : 0;
  Ntt3Args A = {};
  A.tw256 = pl.tw256[d].get();
  A.t2 = pl.t2[d].get();
  A.batch = batch;
  A.src_len = A.dst_len = NTT_UNBOUNDED;
  A.src = src;
  A.dst = data;
  A.mul_src = mul;
  A.mul_mask = mul_mask;
  A.flags = mul ? NTT_FLAG_MUL : 0;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(16u * batch);
  cfg.blockDim = dim3(2 * N3_THREADS);
  cfg.dynamicSmemBytes = kSmem;
  cfg.stream = ctx->stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 16;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  if (ctx->cluster16_state == 0) {  // first use: can the device place a 16-CTA cluster of this footprint at all?
    int clusters = 0;
    if (cudaOccupancyMaxActiveClusters(&clusters, kern, &cfg) != cudaSuccess || clusters < 1) {
      cudaGetLastError();
      ctx->cluster16_state = -1;
      return RONK_OK;
    }
    ctx->cluster16_state = 1;
  }
  {
    LaunchScope ls(ctx, INV ? "intt16_cluster" : "ntt16_cluster");
    RONK_CUDA(ctx, cudaLaunchKernelEx(&cfg, kern, f, A));
  }
  RONK_TRY(check_launch(ctx, "ntt16c_kernel"));
  *done = true;
  return RONK_OK;
}

// data = NTT(src [zero-extended from src_len]) [⊙ mul], the first dst_len outputs stored.  Pass 1 src → workspace, pass 2
// in place in the workspace (its input and output views coincide), pass 3 workspace → data: src is only read, data only
// written by the last pass, so src == data (in place) and a short data buffer (dst_len words) are both fine.
// LI > 0: a SPLIT transform n = 2^LI·2^LOGN (2^17 … 2^19 over 2^16, 2^25 / 2^26 over 2^24): `outer` is the n-point plan (its
// two-level tables feed the first pass), pl the 2^LOGN-point plan of the 2^LI·batch sub-transforms; ntt3p_kernel runs
// first (src → data, in place when they coincide) and the last pass interleaves the sub-transforms' outputs.
// COSET (2^21 … 2^24, unbounded, no multiplier): `coset` holds the two coset tables of run_ntt; pass 1 (forward) or
// pass 3 (inverse) applies the factor, and every pass's profile name carries "_coset".
template <class F, bool INV, int LOGN, bool BOUNDED, int LI = 0, bool COSET = false>
static int run_ntt3(ronk_ctx* ctx, const F& f, NttPlan& pl, u64* data, const u64* src, const u64* mul, u32 batch,
                    u64 src_len, u64 dst_len, u64 mul_mask = ~0ULL, const NttPlan* outer = nullptr, const u64* coset = nullptr) {
  static_assert(LI == 0 || ((LOGN == 16 || LOGN == 24) && !BOUNDED), "split transforms: over 2^16 or 2^24, unbounded");
  static_assert(!COSET || (LI == 0 && !BOUNDED && LOGN >= 21), "coset transforms: 2^21 … 2^24, unbounded");
  const int d = INV ? 1 : 0;
  const u64 n = (u64)1 << LOGN;
  RONK_TRY((ntt3_tables<F, INV>(ctx, f, pl, LOGN)));
  if (LOGN >= 20 && LOGN <= ctx->tune.ntt3_t1 && !pl.t1[d]) {  // n-word table of the stepped twiddles: 8 MiB (2^20) … 128 MiB (2^24) per direction; no memory: stay stepped
    if (pl.log_n1 != (u32)(LOGN + 1) / 2 || !pl.tw_lo || !pl.tw2) return set_err(ctx, RONK_ECUDA, "internal: unexpected plan shape");
    RONK_TRY(build_table(ctx, &pl.t1[d], n, [&](u64* t1) {
      if (LOGN >= 21)
        return launch(ctx, "ntt3_t1", ntt3_t1_kernel<F>, (unsigned)(n / 256), 256, 0, false, f, pl.tw_lo.get(), pl.tw2.get(),
                      INV ? 1 : 0, t1, (u32)LOGN);
      return launch(ctx, "ntt3_t1", ntt3_t1_20_kernel<F>, (unsigned)(n / 256), 256, 0, false, f, pl.tw_lo.get(), pl.tw2.get(),
                    INV ? 1 : 0, t1);
    }, true));
  }
  if (LI > 0) {
    if (!outer || !outer->tw_lo || !outer->tw2 || batch > (0x7FFFFFFFu >> (12 + LI))) return set_err(ctx, RONK_EUNSUPPORTED, "batch too large");
    Ntt3Args P = {};
    P.src = src;
    P.dst = data;
    P.tw_lo = outer->tw_lo.get();
    P.tw_hi = outer->tw2.get();
    P.scale_tw = INV ? f.to_tw(h_powmod((u64)1 << LI, pl.p - 2, pl.p)) : 0;   // 2^-LI: the rest of n^-1 rides on the sub-transforms' tables
    P.batch = batch;
    RONK_TRY((launch3p<F, INV, LI>(ctx, f, P, (u32)LOGN, outer->log_n1, INV ? "intt3_split" : "ntt3_split")));
    src = data;
    batch <<= LI;
  }
  if (batch > (0x7FFFFFFFu >> 12)) return set_err(ctx, RONK_EUNSUPPORTED, "batch too large");
  Frame fr(ctx);
  u64* ws = nullptr;
  RONK_TRY(fr.take(&ws, (size_t)batch << LOGN));
  if (LOGN >= 20 && (pl.log_n1 != (u32)(LOGN + 1) / 2 || !pl.tw_lo || !pl.tw2)) return set_err(ctx, RONK_ECUDA, "internal: unexpected plan shape");
  Ntt3Args A = {};
  A.t1 = LOGN <= ctx->tune.ntt3_t1 ? pl.t1[d].get() : nullptr;
  A.tw256 = pl.tw256[d].get();
  A.tw_lo = pl.tw_lo.get();
  A.tw_hi = pl.tw2.get();   // ω_n^(4096 y), plain: the n^-1 of the inverse rides on the pass-2 table
  A.t2 = pl.t2[d].get();
  A.batch = batch;
  A.src_len = src_len;
  A.dst_len = dst_len;
  A.mul_mask = mul_mask;
  A.src = src;
  A.dst = ws;
  if constexpr (COSET) A.coset = coset;
  if constexpr (LOGN == 20) {
    // sixteen interleaved 2^16-point transforms + one radix-16 pass (ntt3_kernel.cuh): A1 src → data (identical views, so
    // src == data is fine), A2 data → workspace, C workspace → data.  A.tw_hi = ω_n^(1024 y): the plan's 10 / 10 split.
    A.dst = data;
    RONK_TRY((launch3<F, 2, INV, 20, false>(ctx, f, A, INV ? "intt3_a1" : "ntt3_a1", false)));
    A.src = data;
    A.dst = ws;
    RONK_TRY((launch3<F, 1, INV, 20, false>(ctx, f, A, INV ? "intt3_a2" : "ntt3_a2", true)));
    A.src = ws;
    A.dst = data;
    A.mul_src = mul;
    A.flags = mul ? NTT_FLAG_MUL : 0;
    return launch3c<F, INV>(ctx, f, A, INV ? "intt3_c" : "ntt3_c");
  } else {
    if constexpr (LOGN >= 21) {
      const char* name = COSET ? (INV ? "intt3_pass1_coset" : "ntt3_pass1_coset") : (INV ? "intt3_pass1" : "ntt3_pass1");
      RONK_TRY((launch3<F, 1, INV, LOGN, BOUNDED, 0, COSET && !INV>(ctx, f, A, name, false)));
      A.src = ws;
    }
    const char* name2 = COSET ? (INV ? "intt3_pass2_coset" : "ntt3_pass2_coset") : (INV ? "intt3_pass2" : "ntt3_pass2");
    RONK_TRY((launch3<F, 2, INV, LOGN, BOUNDED && LOGN == 16>(ctx, f, A, name2, LOGN >= 21)));
    A.src = ws;
    A.dst = data;
    A.mul_src = mul;
    A.flags = mul ? NTT_FLAG_MUL : 0;
    const char* name3 = COSET ? (INV ? "intt3_pass3_coset" : "ntt3_pass3_coset") : (INV ? "intt3_pass3" : "ntt3_pass3");
    return launch3<F, 3, INV, LOGN, BOUNDED, LI, COSET && INV>(ctx, f, A, name3, true);
  }
}

// the plan of (p, g, 2^log_n), built on first use (std::map: references to other plans stay valid)
template <class F>
static int plan_for(ronk_ctx* ctx, const F& f, u64 p, u64 g, u32 log_n, NttPlan** out) {
  auto key = std::make_tuple((uint64_t)p, (uint64_t)g, (uint32_t)log_n);
  auto it = ctx->plans.find(key);
  if (it == ctx->plans.end()) {
    NttPlan pl;
    RONK_TRY(build_tables(ctx, [&] { return build_plan(ctx, f, p, g, log_n, &pl); }));
    it = ctx->plans.emplace(key, std::move(pl)).first;
  }
  *out = &it->second;
  return RONK_OK;
}

// src == nullptr: in place.  Otherwise (batch == 1) the transform reads src[0, src_len) zero-extended to n
// words and writes data[0, dst_len): the zero padding of poly_mul's operands and the clipping of its
// result happen inside the load / store phases instead of in separate copy kernels.
// coset != nullptr: a coset transform, in place, unbounded, without multiplier.  `coset` holds c^i for i < 2^h, then
// c^(i·2^h) for i < 2^(log_n - h), twiddle form, h = ⌈log_n / 2⌉ (c = s forward, s^-1 inverse).  It takes the
// single-tile kernel or the generic pass pair, and the 256-point-tile passes at 2^21 … 2^24 for Goldilocks with g = 7,
// whatever the context's transform switches say; every launch's profile name carries "_coset".
template <class F, bool INV>
static int run_ntt(ronk_ctx* ctx, const F& f, NttPlan& pl, u64* data, const u64* mul, u32 batch,
                   const u64* src = nullptr, u64 src_len = NTT_UNBOUNDED, u64 dst_len = NTT_UNBOUNDED,
                   u64 mul_mask = ~0ULL, const u64* coset = nullptr) {
  const u32 log_n = pl.log_n;
  const u32 coset_h = (log_n + 1) / 2;
  u64 tiles = 0;
  if (!src) src = data;
  if (src_len >= ((u64)1 << log_n)) src_len = NTT_UNBOUNDED;
  if (dst_len >= ((u64)1 << log_n)) dst_len = NTT_UNBOUNDED;
  if (!pl.two_pass) {
    const u32 cap = (u32)ctx->tune.single_tile_log;
    NttTileArgs A =
        ntt_args_single(data, mul, pl.tw1_2d[INV ? 1 : 0].get(), pl.scale_inv, log_n, (u64)batch << log_n, INV, cap, &tiles);
    A.src = src;
    A.src_len = src_len;
    A.dst_len = dst_len;
    A.mul_mask = mul_mask;
    if (coset) {
      A.coset_lo = coset;
      A.coset_hi = coset + ((size_t)1 << coset_h);
      A.coset_h = coset_h;
    }
    if (tiles > 0x7FFFFFFFULL) return set_err(ctx, RONK_EUNSUPPORTED, "batch too large");
    const char* name = coset ? (INV ? "intt_single_coset" : "ntt_single_coset") : (INV ? "intt_single" : "ntt_single");
    return launch_tile<F, MODE_SINGLE, INV>(ctx, f, A, (u32)tiles, name);
  }
  if constexpr (std::is_same<F, GoldilocksField>::value) {
    if (coset) {
      switch (log_n) {
        case 21: return run_ntt3<F, INV, 21, false, 0, true>(ctx, f, pl, data, src, mul, batch, src_len, dst_len, mul_mask, nullptr, coset);
        case 22: return run_ntt3<F, INV, 22, false, 0, true>(ctx, f, pl, data, src, mul, batch, src_len, dst_len, mul_mask, nullptr, coset);
        case 23: return run_ntt3<F, INV, 23, false, 0, true>(ctx, f, pl, data, src, mul, batch, src_len, dst_len, mul_mask, nullptr, coset);
        case 24: return run_ntt3<F, INV, 24, false, 0, true>(ctx, f, pl, data, src, mul, batch, src_len, dst_len, mul_mask, nullptr, coset);
        default: break;
      }
    } else if (ctx->tune.ntt3 && !(INV && mul)) {   // mul_mask: one multiplier word per output (~0) or a shared n-word one (n - 1)
      const bool bounded = src_len != NTT_UNBOUNDED || dst_len != NTT_UNBOUNDED;  // only ever with batch == 1
      // 2^16: worth it once the grid fills the GPU (16 tiles per transform); single transforms stay launch-bound
      if (log_n == 24 && !bounded) return run_ntt3<F, INV, 24, false>(ctx, f, pl, data, src, mul, batch, src_len, dst_len, mul_mask);
      if (log_n == 24 && batch == 1) return run_ntt3<F, INV, 24, true>(ctx, f, pl, data, src, mul, batch, src_len, dst_len, mul_mask);
      if (!bounded && ctx->tune.ntt3_split && ((log_n >= 17 && log_n <= 19 && (batch << (log_n - 16)) >= (u32)ctx->tune.ntt3_split_min16) ||
                                               log_n == 25 || log_n == 26)) {
        // split transforms: a radix-2/4/8 register pass, then 2^16- or 2^24-point tile transforms whose last pass interleaves
        const u32 lsub = log_n >= 25 ? 24u : 16u;
        NttPlan* sub = nullptr;
        RONK_TRY(plan_for(ctx, f, pl.p, pl.g, lsub, &sub));
        switch (log_n) {
          case 17: return run_ntt3<F, INV, 16, false, 1>(ctx, f, *sub, data, src, mul, batch, src_len, dst_len, mul_mask, &pl);
          case 18: return run_ntt3<F, INV, 16, false, 2>(ctx, f, *sub, data, src, mul, batch, src_len, dst_len, mul_mask, &pl);
          case 19: return run_ntt3<F, INV, 16, false, 3>(ctx, f, *sub, data, src, mul, batch, src_len, dst_len, mul_mask, &pl);
          case 25: return run_ntt3<F, INV, 24, false, 1>(ctx, f, *sub, data, src, mul, batch, src_len, dst_len, mul_mask, &pl);
          default: return run_ntt3<F, INV, 24, false, 2>(ctx, f, *sub, data, src, mul, batch, src_len, dst_len, mul_mask, &pl);
        }
      }
      if (log_n >= 21 && log_n <= 23 && !bounded && ctx->tune.ntt3_mid) {   // 2^21 … 2^23: first pass of 32 / 64 / 128 points, then as 2^24
        if (log_n == 21) return run_ntt3<F, INV, 21, false>(ctx, f, pl, data, src, mul, batch, src_len, dst_len, mul_mask);
        if (log_n == 22) return run_ntt3<F, INV, 22, false>(ctx, f, pl, data, src, mul, batch, src_len, dst_len, mul_mask);
        return run_ntt3<F, INV, 23, false>(ctx, f, pl, data, src, mul, batch, src_len, dst_len, mul_mask);
      }
      if (log_n >= 21 && log_n <= 23 && bounded && batch == 1 && ctx->tune.ntt3_mid) {   // zero-padded source / clipped destination (poly_mul)
        if (log_n == 21) return run_ntt3<F, INV, 21, true>(ctx, f, pl, data, src, mul, batch, src_len, dst_len, mul_mask);
        if (log_n == 22) return run_ntt3<F, INV, 22, true>(ctx, f, pl, data, src, mul, batch, src_len, dst_len, mul_mask);
        return run_ntt3<F, INV, 23, true>(ctx, f, pl, data, src, mul, batch, src_len, dst_len, mul_mask);
      }
      if (log_n == 20 && !bounded && ctx->tune.ntt3_20) return run_ntt3<F, INV, 20, false>(ctx, f, pl, data, src, mul, batch, src_len, dst_len, mul_mask);
      if (log_n == 16 && !bounded && batch <= (u32)ctx->tune.ntt16_cluster_max_batch) {
        bool done = false;
        RONK_TRY((run_ntt16_cluster<F, INV>(ctx, f, pl, data, src, mul, batch, &done, mul_mask)));
        if (done) return RONK_OK;
      }
      if (log_n == 16 && !bounded && batch >= (u32)ctx->tune.ntt3_min_batch16)
        return run_ntt3<F, INV, 16, false>(ctx, f, pl, data, src, mul, batch, src_len, dst_len, mul_mask);
    }
  }
  Frame fr(ctx);
  u64* ws = nullptr;
  RONK_TRY(fr.take(&ws, (size_t)batch << log_n));
  // preferred tile sizes (log2): 14 / 13 (strided pass-1 reads want 32-byte segments)
  const int pref1 = ctx->tune.tile1, pref2 = ctx->tune.tile2, adapt = ctx->tune.tile_adapt;
  // The preferred sizes are tuned for grids of ≥ 1000 tiles.  A mid-size job (one 2^20 transform is 64 tiles of
  // 2^14) would leave most SMs idle, so shrink the tiles until the grid fills the GPU, but never below 4 columns
  // in pass 1 (32-byte segments) / 2 in pass 2.
  u32 p1 = (u32)pref1, p2 = (u32)pref2;
  if (adapt) {
    const u64 total = (u64)batch << log_n;
    const u64 want = 2ull * (u64)ctx->sm_count;
    while (p1 > pl.log_n1 + 2 && p1 > 11 && (total >> p1) < want) p1--;
    while (p2 > pl.log_n2 + 1 && p2 > 11 && (total >> p2) < 2 * want) p2--;
  }
  u32 tile1, tile2;
  ntt_pass_tiles(log_n, p1, p2, &tile1, &tile2);
  // pass 1: N1-point transforms down the columns, inter-pass twiddle, blocked write to the workspace
  NttTileArgs A1 = ntt_args_pass1(src, ws, pl.tw1_2d[INV ? 1 : 0].get(), pl.tw_lo.get(), (INV ? pl.tw_hi_inv : pl.tw2).get(),
                                  pl.tw2.get(), log_n, batch, tile1, tile2, &tiles);
  A1.src_len = src_len;
  if (tiles > 0x7FFFFFFFULL) return set_err(ctx, RONK_EUNSUPPORTED, "batch too large");
  if (coset) {   // the hooked pass is the first (forward) or the last (inverse); launch_tile_n picks it
    A1.coset_lo = coset;
    A1.coset_hi = coset + ((size_t)1 << coset_h);
    A1.coset_h = coset_h;
  }
  if (ctx->tune.tw_table) {
    const u64* tab = nullptr;
    RONK_TRY(interpass_table(ctx, f, pl, INV, A1.log_c2, A1.tw_lo, A1.tw_hi, &tab));
    A1.tw_full = tab;
  }
  const char* name1 = coset ? (INV ? "intt_pass1_coset" : "ntt_pass1_coset") : (INV ? "intt_pass1" : "ntt_pass1");
  RONK_TRY((launch_tile<F, MODE_PASS1, INV>(ctx, f, A1, (u32)tiles, name1)));
  // pass 2: N2-point transforms along the contiguous workspace tiles, natural-order output
  NttTileArgs A2 = ntt_args_pass2(ws, data, mul, pl.tw2_2d[INV ? 1 : 0].get(), log_n, batch, tile2, &tiles);
  A2.dst_len = dst_len;
  A2.mul_mask = mul_mask;
  if (tiles > 0x7FFFFFFFULL) return set_err(ctx, RONK_EUNSUPPORTED, "batch too large");
  if (coset) {
    A2.coset_lo = coset;
    A2.coset_hi = coset + ((size_t)1 << coset_h);
    A2.coset_h = coset_h;
  }
  const char* name2 = coset ? (INV ? "intt_pass2_coset" : "ntt_pass2_coset") : (INV ? "intt_pass2" : "ntt_pass2");
  return launch_tile<F, MODE_PASS2, INV>(ctx, f, A2, (u32)tiles, name2);
}

template <class F>
static int ntt_with_field(ronk_ctx* ctx, const F& f, u64 p, u64 g, u64* data, const u64* mul, u32 log_n, u32 batch,
                          int inverse, const u64* src = nullptr, u64 src_len = NTT_UNBOUNDED,
                          u64 dst_len = NTT_UNBOUNDED, u64 mul_mask = ~0ULL) {
  NttPlan* pl = nullptr;
  RONK_TRY(plan_for(ctx, f, p, g, log_n, &pl));
  return inverse ? run_ntt<F, true>(ctx, f, *pl, data, mul, batch, src, src_len, dst_len, mul_mask)
                 : run_ntt<F, false>(ctx, f, *pl, data, mul, batch, src, src_len, dst_len, mul_mask);
}

// One transform, out of place: dst[0, dst_len) = NTT(src[0, src_len) zero-extended to 2^log_n) [⊙ mul].
// log_n >= 1; dst needs only dst_len words.  Used by product_bounded and the Newton inversion (poly_div.cu).
int ntt_device_bounded(ronk_ctx* ctx, u64 p, u64 g, const u64* src, u64 src_len, u64* dst, u64 dst_len, const u64* mul,
                       u32 log_n, int inverse) {
  if (!ctx || !src || !dst) return set_err(ctx, RONK_EINVAL, "null argument");
  if (log_n == 0 || !pow2_fits(p, log_n)) return set_err(ctx, RONK_EINVAL, "unsupported transform size");
  return with_field(ctx, p, g, inverse != 0, [&](const auto& f) {
    return ntt_with_field(ctx, f, p, g, dst, mul, log_n, 1, inverse, src, src_len, dst_len);
  });
}

int product_bounded(ronk_ctx* ctx, u64 p, u64 g, const u64* a, u64 la, const u64* b, u64 lb, u32 log_n, u64* X, u64* Y,
                    u64* out, u64 out_len) {
  const u64 n = (u64)1 << log_n;
  RONK_TRY(ntt_device_bounded(ctx, p, g, a, la, X, n, nullptr, log_n, 0));  // Â
  RONK_TRY(ntt_device_bounded(ctx, p, g, b, lb, Y, n, X, log_n, 0));        // B̂ ⊙ Â fused into the last pass
  return ntt_device_bounded(ctx, p, g, Y, n, out, out_len, nullptr, log_n, 1);
}

// dst = NTT(src) ⊙ mul (forward), batch transforms, mul an n-word table shared by all of them (index & (n-1)).
// src may equal dst.  Used by the distributed transform (dist.cu): the twiddle column ω_n'^(r·k) rides on the
// store phase of the local transform instead of two extra passes over the data.
int ntt_device_shared_mul(ronk_ctx* ctx, u64 p, u64 g, const u64* src, u64* dst, const u64* mul, u32 log_n, u32 batch) {
  if (!ctx || !src || !dst) return set_err(ctx, RONK_EINVAL, "null argument");
  if (log_n == 0 || !pow2_fits(p, log_n)) return set_err(ctx, RONK_EINVAL, "unsupported transform size");
  if (batch == 0) return RONK_OK;
  const u64 mask = mul ? (((u64)1 << log_n) - 1) : ~0ULL;
  return with_field(ctx, p, g, false, [&](const auto& f) {
    return ntt_with_field(ctx, f, p, g, dst, mul, log_n, batch, 0, src, NTT_UNBOUNDED, NTT_UNBOUNDED, mask);
  });
}

// The single-tile plan of (p, g, 2^log_n), built on first use: its per-round forward and inverse twiddle tables and n^-1
// in twiddle form.  Used by the fused batched product (poly_batch.cu).
int ntt_single_tables(ronk_ctx* ctx, u64 p, u64 g, u32 log_n, const u64** fwd, const u64** inv, u64* scale_inv) {
  if (log_n == 0 || ntt_shape(log_n).two_pass || (p - 1) % ((u64)1 << log_n) != 0)
    return set_err(ctx, RONK_EINVAL, "internal: not a single-tile transform size");
  return with_field(ctx, p, g, false, [&](const auto& f) {
    NttPlan* pl = nullptr;
    RONK_TRY(plan_for(ctx, f, p, g, log_n, &pl));
    *fwd = pl->tw1_2d[0].get();
    *inv = pl->tw1_2d[1].get();
    *scale_inv = pl->scale_inv;
    return RONK_OK;
  });
}

// A coset transform with s != 1 (ntt_coset.cu checks the arguments; log_n >= 1): the two coset tables in this call's
// scratch, built by one launch, then run_ntt with the factor fused into its first or last pass.
int ntt_device_coset(ronk_ctx* ctx, u64 p, u64 g, u64* data, u32 log_n, u32 batch, u64 shift, int inverse) {
  return with_field(ctx, p, g, inverse != 0, [&](const auto& f) {
    using F = std::decay_t<decltype(f)>;
    NttPlan* pl = nullptr;
    RONK_TRY(plan_for(ctx, f, p, g, log_n, &pl));
    const u32 h = (log_n + 1) / 2;
    const u32 words = (1u << h) + (1u << (log_n - h));
    Frame fr(ctx);
    u64* tab = nullptr;
    RONK_TRY(fr.take(&tab, words));
    const u64 c = inverse ? h_powmod(shift, p - 2, p) : shift;
    RONK_TRY(launch(ctx, "ntt_coset_table", coset_table_kernel<F>, (words + 255) / 256, 256, 0, false, f, c, h, log_n, tab));
    return inverse ? run_ntt<F, true>(ctx, f, *pl, data, nullptr, batch, nullptr, NTT_UNBOUNDED, NTT_UNBOUNDED, ~0ULL, tab)
                   : run_ntt<F, false>(ctx, f, *pl, data, nullptr, batch, nullptr, NTT_UNBOUNDED, NTT_UNBOUNDED, ~0ULL, tab);
  });
}

size_t ntt_workspace_words(u32 log_n, u32 batch) { return ntt_shape(log_n).two_pass ? (size_t)batch << log_n : 0; }

int ntt_device(ronk_ctx* ctx, u64 p, u64 g, u64* data, const u64* mul, u32 log_n, u32 batch, int inverse) {
  if (!ctx || !data) return set_err(ctx, RONK_EINVAL, "null argument");
  RONK_TRY(validate_modulus(ctx, p));
  if (g == 0 || g >= p) return set_err(ctx, RONK_EINVAL, "generator out of range");
  if (log_n >= 64 || (p - 1) % ((u64)1 << log_n) != 0)
    return set_err(ctx, RONK_EINVAL, "n must divide p - 1 (no primitive n-th root of unity)");
  if (log_n > 26) return set_err(ctx, RONK_EUNSUPPORTED, "log_n > 26 not supported");
  if (batch == 0) return RONK_OK;
  if (log_n == 0) {
    if (mul) return ronk_field_mul_u64(ctx, p, (const uint64_t*)data, (const uint64_t*)mul, (uint64_t*)data, batch);
    return RONK_OK;
  }
  return with_field(ctx, p, g, inverse != 0,
                    [&](const auto& f) { return ntt_with_field(ctx, f, p, g, data, mul, log_n, batch, inverse); });
}

}  // namespace ronk

using namespace ronk;

extern "C" int ronk_ntt_u64(ronk_ctx* ctx, uint64_t p, uint64_t g, uint64_t* data, uint32_t log_n, uint32_t batch,
                            int inverse) {
  ronk::DeviceGuard _dg(ctx);
  return ntt_device(ctx, p, g, (u64*)data, nullptr, log_n, batch, inverse);
}

extern "C" int ronk_ntt_mul_u64(ronk_ctx* ctx, uint64_t p, uint64_t g, uint64_t* data, const uint64_t* mul,
                                uint32_t log_n, uint32_t batch) {
  ronk::DeviceGuard _dg(ctx);
  if (!mul) return set_err(ctx, RONK_EINVAL, "null multiplier");
  return ntt_device(ctx, p, g, (u64*)data, (const u64*)mul, log_n, batch, 0);
}

static int pipeline_init(ronk_ctx* ctx) {
  if (ctx->copy_in) return RONK_OK;
  RONK_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->copy_in, cudaStreamNonBlocking));
  RONK_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->copy_out, cudaStreamNonBlocking));
  for (int i = 0; i < ronk_ctx::kSlots; i++) {
    RONK_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_h2d[i], cudaEventDisableTiming));
    RONK_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_compute[i], cudaEventDisableTiming));
    RONK_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_d2h[i], cudaEventDisableTiming));
  }
  return RONK_OK;
}

extern "C" int ronk_ntt_u64_host_wait(ronk_ctx* ctx, int slot) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx || slot < 0 || slot >= ronk_ctx::kSlots) return set_err(ctx, RONK_EINVAL, "bad slot");
  if (!ctx->slot_pending[slot]) return RONK_OK;
  RONK_CUDA(ctx, cudaEventSynchronize(ctx->ev_d2h[slot]));
  ctx->slot_pending[slot] = false;
  return RONK_OK;
}

extern "C" int ronk_ntt_u64_host_submit(ronk_ctx* ctx, uint64_t p, uint64_t g, uint64_t* host_data, uint32_t log_n,
                                        uint32_t batch, int inverse, int slot) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx || !host_data) return set_err(ctx, RONK_EINVAL, "null argument");
  if (slot < 0 || slot >= ronk_ctx::kSlots) return set_err(ctx, RONK_EINVAL, "bad slot");
  if (log_n > 26) return set_err(ctx, RONK_EUNSUPPORTED, "log_n > 26 not supported");
  const size_t bytes = ((size_t)batch << log_n) * sizeof(u64);
  if (bytes == 0) return RONK_OK;
  RONK_TRY(pipeline_init(ctx));
  RONK_TRY(ronk_ntt_u64_host_wait(ctx, slot));  // the slot's previous occupant must be home first
  if (ctx->slot_bytes[slot] < bytes) {
    if (ctx->slot_buf[slot]) RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // alloc frees the old buffer first
    ctx->slot_bytes[slot] = 0;
    RONK_TRY(ctx->slot_buf[slot].alloc(ctx, bytes / sizeof(u64)));
    ctx->slot_bytes[slot] = bytes;
  }
  u64* dbuf = ctx->slot_buf[slot].get();
  RONK_CUDA(ctx, cudaMemcpyAsync(dbuf, host_data, bytes, cudaMemcpyHostToDevice, ctx->copy_in));
  RONK_CUDA(ctx, cudaEventRecord(ctx->ev_h2d[slot], ctx->copy_in));
  RONK_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_h2d[slot], 0));
  RONK_TRY(ntt_device(ctx, p, g, dbuf, nullptr, log_n, batch, inverse));
  RONK_CUDA(ctx, cudaEventRecord(ctx->ev_compute[slot], ctx->stream));
  RONK_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_out, ctx->ev_compute[slot], 0));
  RONK_CUDA(ctx, cudaMemcpyAsync(host_data, dbuf, bytes, cudaMemcpyDeviceToHost, ctx->copy_out));
  RONK_CUDA(ctx, cudaEventRecord(ctx->ev_d2h[slot], ctx->copy_out));
  ctx->slot_pending[slot] = true;
  return RONK_OK;
}

extern "C" int ronk_ntt_u64_host(ronk_ctx* ctx, uint64_t p, uint64_t g, uint64_t* host_data, uint32_t log_n,
                                 uint32_t batch, int inverse) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx || !host_data) return set_err(ctx, RONK_EINVAL, "null argument");
  if (((size_t)batch << log_n) == 0) return RONK_OK;
  RONK_TRY(ronk_ntt_u64_host_submit(ctx, p, g, host_data, log_n, batch, inverse, 0));
  return ronk_ntt_u64_host_wait(ctx, 0);
}
