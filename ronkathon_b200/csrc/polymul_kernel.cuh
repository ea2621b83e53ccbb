// polymul_kernel.cuh — many short polynomial products in one launch (sm_90a).
//
// Polynomial::mul (src/polynomial/arithmetic.rs:97-119) of `batch` row pairs c[r] = a[r]·b[r] (or a[r]·b for one shared
// b) with L = da + db - 1 ≤ N = 2^log_n ≤ 2^PM_MAX_LOG.  One CTA owns two operand tiles of T = 2^PM_TILE_LOG words; each
// holds P = T/N products side by side, laid out as MODE_SINGLE lays out several transforms in one tile (tile index
// e = [row j | coefficient k], log_c = 0), so the radix-16 rounds of ntt_kernel.cuh run on them unchanged.  Per tile:
//   1. load: the P rows of a (of b) are one contiguous run of P·da (P·db) words in HBM, read coalesced and scattered into
//      the swizzled tile; the slack (k ≥ da, rows past the batch) is zeroed;
//   2. the forward rounds on both tiles (N-point plan, per-round twiddle tables staged by TMA);
//   3. the point-wise product into tile A: both spectra are in the same bit-reversed order;
//   4. one bit-reversal permutation A → B, so that the inverse rounds see natural order again;
//   5. the inverse rounds on B;
//   6. store: un-bit-reverse, scale by N^-1 and clip to L words per row, again as one contiguous run of P·L words.
// HBM traffic is the compulsory da + db words in and L words out per product.  The phases are RONK_DEV functions, so
// tests/emu/polymul_emu.cpp runs the same data flow on the CPU.
#pragma once
#include "ntt_kernel.cuh"

namespace ronk {

constexpr u32 PM_TILE_LOG = 11;  // 2 tiles of 16 KiB + both twiddle tables of a 2^11-point plan (2 × 18.1 KiB): 3 CTAs per SM
constexpr u32 PM_MAX_LOG = 11;   // the largest transform that fits one tile
constexpr int PM_THREADS = 128;  // one radix-16 group per thread, round and tile

struct PolyMulArgs {
  const u64* a;
  const u64* b;
  u64* c;
  u32 da, db, L;        // words per row of a, b and c
  u32 b_stride;         // words between rows of b: db, or 0 for one b shared by every row
  u64 batch;            // rows
  u32 rows_log;         // log2 P, rows per tile
  const u64* tw_fwd;    // the N-point plan's per-round tables (forward, inverse), twiddle form
  const u64* tw_inv;
  u64 scale;            // N^-1, twiddle form
  NttTileArgs R;        // round geometry: tile_log, log_m = log_n, log_c = 0, tw_off, tw_words
};

// Host: the arguments of one fused launch; *tiles = number of CTAs.
inline PolyMulArgs polymul_args(const u64* a, u32 da, const u64* b, u32 db, bool b_shared, u64 batch, u64* c, u32 log_n,
                                const u64* tw_fwd, const u64* tw_inv, u64 scale, u64* tiles) {
  PolyMulArgs A = {};
  A.a = a;
  A.b = b;
  A.c = c;
  A.da = da;
  A.db = db;
  A.L = da + db - 1;
  A.b_stride = b_shared ? 0 : db;
  A.batch = batch;
  A.rows_log = PM_TILE_LOG - log_n;
  A.tw_fwd = tw_fwd;
  A.tw_inv = tw_inv;
  A.scale = scale;
  A.R.tile_log = PM_TILE_LOG;
  A.R.log_m = log_n;
  A.R.log_c = 0;
  A.R.log_n = log_n;
  A.R.tw_words = ntt_tw2d_layout(log_n, A.R.tw_off);
  *tiles = (batch + ((u64)1 << A.rows_log) - 1) >> A.rows_log;
  return A;
}

RONK_DEV u32 pm_rows(const PolyMulArgs& A, u64 tile) {  // rows held by this tile (the last one may be partial)
  const u64 r0 = tile << A.rows_log, left = A.batch - r0, full = (u64)1 << A.rows_log;
  return (u32)(left < full ? left : full);
}

// Phase 1 for one operand: rows of d words, `stride` words apart in src (0: the same row for all), into tile s.
RONK_DEV void pm_load(u64* s, const u64* src, u32 d, u32 stride, const PolyMulArgs& A, u64 tile, u32 tid, u32 nthr) {
  const u32 T = 1u << A.R.tile_log, log_n = A.R.log_m, M = (1u << log_n) - 1u;
  const u32 rows = pm_rows(A, tile);
  for (u32 e = tid; e < T; e += nthr)
    if ((e & M) >= d || (e >> log_n) >= rows) s[swz(e)] = 0;
  const u64* base = src + (tile << A.rows_log) * (u64)stride;
  const u32 run = rows * d;
  for (u32 w = tid; w < run; w += nthr) {
    const u32 j = w / d, k = w - j * d;
    s[swz((j << log_n) | k)] = base[stride ? w : k];
  }
}

// Phase 3: sa ← sa ⊙ sb over the whole tile (same positions, same order).
template <class F>
RONK_DEV void pm_pointwise(const F& f, u64* sa, const u64* sb, const PolyMulArgs& A, u32 tid, u32 nthr) {
  const u32 T = 1u << A.R.tile_log;
  for (u32 e = tid; e < T; e += nthr) {
    const u32 x = swz(e);
    sa[x] = f.mul(sa[x], sb[x]);
  }
}

// Phase 4: to[j | bitrev(k)] = from[j | k].  Reads are consecutive; bit reversal puts the lanes' low bits on the top bits
// of k, which the swizzle folds back onto distinct banks.
RONK_DEV void pm_bitrev(const u64* from, u64* to, const PolyMulArgs& A, u32 tid, u32 nthr) {
  const u32 T = 1u << A.R.tile_log, log_n = A.R.log_m, M = (1u << log_n) - 1u;
  for (u32 e = tid; e < T; e += nthr) to[swz((e & ~M) | bitrev(e & M, log_n))] = from[swz(e)];
}

// Phase 6: c rows of this tile, one contiguous run of rows·L words; position bitrev(k) holds coefficient k.
template <class F>
RONK_DEV void pm_store(const F& f, const u64* s, const PolyMulArgs& A, u64 tile, u32 tid, u32 nthr) {
  const u32 log_n = A.R.log_m, L = A.L;
  const u32 run = pm_rows(A, tile) * L;
  u64* base = A.c + (tile << A.rows_log) * (u64)L;
  for (u32 w = tid; w < run; w += nthr) {
    const u32 j = w / L, k = w - j * L;
    base[w] = f.mul_tw(s[swz((j << log_n) | bitrev(k, log_n))], A.scale);
  }
}

// Phases 2 and 5: every round of the N-point plan on one tile (the caller synchronises between rounds).
template <class F, bool INV>
RONK_DEV void pm_round(const F& f, u64* s, const u64* tw, const PolyMulArgs& A, u32 r, u32 tid, u32 nthr) {
  u32 nst, wb, lcur;
  if (ntt_round_plan(A.R, r, &nst, &wb, &lcur)) ntt_round_dispatch<F, INV>(f, s, tw, A.R, nst, wb, lcur, tid, nthr);
}
RONK_DEV u32 pm_round_count(const PolyMulArgs& A) {
  u32 nst, wb, lcur, r = 0;
  while (ntt_round_plan(A.R, r, &nst, &wb, &lcur)) r++;
  return r;
}

#if defined(__CUDACC__)
// Shared memory: [ tile A: T·8 B | tile B: T·8 B | forward twiddles | inverse twiddles | mbarrier ].  ff / fi: the field
// policy of the forward / inverse direction (a Montgomery policy carries its 16th roots of unity per direction).
template <class F>
__global__ void __launch_bounds__(PM_THREADS, 3) polymul_fused_kernel(const F ff, const F fi, const PolyMulArgs A) {
  extern __shared__ __align__(128) u64 smem[];
  const u32 tid = threadIdx.x, T = 1u << A.R.tile_log;
  const u64 tile = blockIdx.x;
  u64* sa = smem;
  u64* sb = sa + T;
  u64* twf = sb + T;
  u64* twi = twf + A.R.tw_words;
  u64* bar = twi + A.R.tw_words;
  const bool use_tw = A.R.log_m > 4;  // a single radix-16 round has no general twiddles
  if (use_tw && tid == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    mbar_expect_tx(bar, 2u * A.R.tw_words * 8u);
    tma_bulk_g2s(twf, A.tw_fwd, A.R.tw_words * 8u, bar);  // both tables land while the operands are being loaded
    tma_bulk_g2s(twi, A.tw_inv, A.R.tw_words * 8u, bar);
  }
  pm_load(sa, A.a, A.da, A.da, A, tile, tid, PM_THREADS);
  pm_load(sb, A.b, A.db, A.b_stride, A, tile, tid, PM_THREADS);
  __syncthreads();
  if (use_tw) mbar_wait(bar, 0);
  const u32 rounds = pm_round_count(A);
  for (u32 r = 0; r < rounds; r++) {
    pm_round<F, false>(ff, sa, twf, A, r, tid, PM_THREADS);
    pm_round<F, false>(ff, sb, twf, A, r, tid, PM_THREADS);
    __syncthreads();
  }
  pm_pointwise(ff, sa, sb, A, tid, PM_THREADS);
  __syncthreads();
  pm_bitrev(sa, sb, A, tid, PM_THREADS);
  __syncthreads();
  for (u32 r = 0; r < rounds; r++) {
    pm_round<F, true>(fi, sb, twi, A, r, tid, PM_THREADS);
    __syncthreads();
  }
  pm_store(fi, sb, A, tile, tid, PM_THREADS);
}
#endif  // __CUDACC__

}  // namespace ronk
