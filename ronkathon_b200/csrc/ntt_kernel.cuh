// ntt_kernel.cuh — the tiled number-theoretic transform kernel (sm_90a).
//
// Replaces Polynomial::fft / ifft (src/polynomial/mod.rs:273-323, :430-484): same map
// X[k] = Σ_j a_j ω^(jk), natural order in and out, canonical residues — computed as a
// decimation-in-frequency transform on a shared-memory tile instead of the reference's recursion.
//
// One CTA owns a tile of T = 2^tile_log field elements (≤ 2^14 = 128 KiB of shared memory) and
// T/16 threads.  Tile index e = [batch-in-tile | NTT index i (log_m bits) | column c (log_c bits)].
// The transform runs over the i bits in "rounds": every thread pulls 16 elements that differ in a
// 4-bit window of i into registers, does a radix-16 DIF butterfly network there (inner twiddles are
// 16th roots of unity — shifts for Goldilocks), multiplies by one general twiddle ω_L^(i2·k1) from a
// table, and writes back in place.  After the last round position i holds X[bitrev(i)]; the store
// phase undoes that permutation for free while it streams the tile out.
//
// Three modes share the code:
//   MODE_SINGLE  n ≤ T: whole transforms inside one tile (several per tile when n < T).
//   MODE_PASS1   n = N1·N2 > T, first pass: tile = all N1 rows × C adjacent columns of the N1×N2
//                matrix view (x[j1·N2 + j2]); N1-point transforms down the columns, then the
//                inter-pass twiddle ω_n^(j2·k1), written to the workspace in the blocked layout
//                W[k1 / C2][j2][k1 % C2] so that pass 2 reads whole contiguous tiles.
//   MODE_PASS2   tile = C2 adjacent k1 × all N2 values of j2 (contiguous in W); N2-point
//                transforms, results to X[k1 + N1·k2] (natural order), optional fused point-wise
//                multiply.
// Only the compulsory input read (pass 1) and output write (pass 2) touch HBM in C·8-byte
// segments; both workspace transfers are fully contiguous.
#pragma once
#include <utility>

#include "field.cuh"

namespace ronk {

enum { MODE_SINGLE = 0, MODE_PASS1 = 1, MODE_PASS2 = 2 };
enum { NTT_FLAG_SCALE = 1, NTT_FLAG_MUL = 2 };

constexpr u64 NTT_UNBOUNDED = ~0ULL;  // NttTileArgs::src_len / dst_len: no bound

struct NttTileArgs {
  const u64* src;
  u64* dst;
  const u64* tw_tile;  // per-round 2-D twiddle tables (see ntt_tw2d_layout), twiddle form
  u32 tw_off[4];       // start of round r's table inside tw_tile (in words)
  u32 tw_words;        // total words of tw_tile (even)
  u32 prefetch_dist;   // pass 1: L2-prefetch the tile of CTA blockIdx.x + prefetch_dist (0 = off)
  // Bounded transforms (batch == 1 only; poly_mul): words of src at index >= src_len read as zero (the
  // zero padding of a shorter operand), words of dst at index >= dst_len are not written (a product with
  // fewer than n coefficients).  NTT_UNBOUNDED = no bound; the unbounded loops are separate code.
  u64 src_len, dst_len;
  const u64* tw_lo;    // PASS1: ω_n^x, x ∈ [0, 2^log_lo)
  const u64* tw_hi;    // PASS1: ω_n^(y·2^log_lo) (· n^-1 for the inverse), y ∈ [0, n >> log_lo)
  const u64* tw_hi_plain;  // PASS1: the same table without the n^-1 factor (twiddle stepping ratio)
  const u64* tw_full;  // PASS1, optional: the whole inter-pass twiddle ω_n^(±j2·k1) [· n^-1], laid out like dst
  const u64* mul_src;  // optional point-wise multiplier, indexed like dst (index & mul_mask)
  u64 mul_mask;        // ~0: one multiplier word per output word; n-1: one n-word multiplier shared by the batch
  u64 scale;           // SINGLE + inverse: n^-1 in twiddle form
  u64 total;           // SINGLE: number of valid elements (batch·n)
  u32 tile_log, log_m, log_c;
  u32 log_n, log_n1, log_n2, log_c2, log_lo;
  u32 tiles_per_batch;
  u32 flags;
  // Coset transforms (COSET instantiations): the word at natural index j of each transform (global index mod n) is
  // multiplied by c^j = coset_lo[j mod 2^coset_h] · coset_hi[j >> coset_h] (twiddle form), in the load of the first pass
  // (forward, c = s) or the store of the last pass (inverse, c = s^-1, after the n^-1 of the inverse).
  const u64* coset_lo;
  const u64* coset_hi;
  u32 coset_h;
};

// v · c^j from the two coset tables (see NttTileArgs::coset_lo): two general multiplies, no n-word table.
template <class F>
RONK_DEV u64 coset_mul(const F& f, u64 v, const u64* lo, const u64* hi, u32 h, u32 j) {
  return f.mul_tw(v, f.mul_tw(lo[j & ((1u << h) - 1u)], hi[j >> h]));
}

// Shared-memory swizzle: 64-bit accesses are served per half-warp against 16 eight-byte banks
// (low 4 bits of the element index).  XOR-folding bits [4,8), [8,12) and [12,14) into the bank
// bits makes every access pattern of this kernel (window at any bit position, digit-reversed
// store) hit 16 distinct banks per half-warp.
RONK_DEV u32 swz(u32 e) { return e ^ (((e >> 4) ^ (e >> 8)) & 15u) ^ (((e >> 12) & 3u) << 2); }

RONK_DEV u32 bitrev(u32 v, u32 bits) {
#if defined(__CUDA_ARCH__)
  return bits ? (__brev(v) >> (32 - bits)) : 0;
#else
  u32 r = 0;
  for (u32 i = 0; i < bits; i++) r |= ((v >> i) & 1u) << (bits - 1 - i);
  return r;
#endif
}
RONK_DEV u64 ld_tw(const u64* p) {
#if defined(__CUDA_ARCH__)
  return __ldg(p);
#else
  return *p;
#endif
}

// One radix-2 DIF butterfly level on register bit BETA of a 16-element register tile.
template <int BETA, int Q, bool INV, class F>
RONK_DEV void bf_one(const F& f, u64 (&x)[16]) {
  constexpr int h = 1 << BETA;
  if constexpr ((Q & h) == 0) {
    u64 a = x[Q], b = x[Q + h];
    x[Q] = f.add(a, b);
    x[Q + h] = f.template w16_sub<(Q & (h - 1)) * (8 / h), INV>(a, b);
  }
}
template <int BETA, bool INV, class F, int... Q>
RONK_DEV void bf_level(const F& f, u64 (&x)[16], std::integer_sequence<int, Q...>) {
  (bf_one<BETA, Q, INV>(f, x), ...);
}
// NST active levels on the low NST bits of the register index (NST = 4: full radix-16).
template <int NST, bool INV, class F>
RONK_DEV void radix_network(const F& f, u64 (&x)[16]) {
  using seq = std::make_integer_sequence<int, 16>;
  if constexpr (NST >= 4) bf_level<3, INV>(f, x, seq{});
  if constexpr (NST >= 3) bf_level<2, INV>(f, x, seq{});
  if constexpr (NST >= 2) bf_level<1, INV>(f, x, seq{});
  if constexpr (NST >= 1) bf_level<0, INV>(f, x, seq{});
}

// Per-round 2-D twiddle tables.  Round r works on sub-transforms of length L = 2^lcur
// (lcur = log_m - 4r, only while lcur > 4) and needs ω_L^(i2·k1) for i2 < L/16, k1 < 16.
// Layout: row i2 holds the 16 values k1 = 0..15 plus one pad word (row stride 17 words), so a thread
// reads its 15 twiddles at fixed offsets from one base (LDS [R + imm], no index arithmetic) and the
// lanes of a warp (consecutive i2) hit distinct banks.
constexpr u32 TW_ROW = 17;
RONK_HD u32 ntt_tw2d_layout(u32 log_m, u32 off[4]) {
  u32 total = 0, r = 0;
  for (u32 lcur = log_m; lcur > 4 && r < 4; lcur -= 4, r++) {
    off[r] = total;
    total += TW_ROW << (lcur - 4);
  }
  for (; r < 4; r++) off[r] = total;
  return (total + 1u) & ~1u;  // even number of words: the TMA bulk copy moves multiples of 16 bytes
}
// word w of the 2-D table → index into the 1-D table ω_M^e (or its negation for the inverse)
RONK_HD u32 ntt_tw2d_source(u32 log_m, u32 w, bool inverse, bool* valid) {
  u32 off[4];
  const u32 total = ntt_tw2d_layout(log_m, off);
  *valid = false;
  if (w >= total) return 0;
  u32 r = 0, lcur = log_m;
  while (r < 3 && lcur - 4 > 4 && w >= off[r + 1]) { r++; lcur -= 4; }
  const u32 rel = w - off[r];
  const u32 i2 = rel / TW_ROW, k1 = rel % TW_ROW;
  if (lcur <= 4 || i2 >= (1u << (lcur - 4)) || k1 >= 16) return 0;  // pad words
  *valid = true;
  const u32 M1 = (1u << log_m) - 1u;
  u32 idx = ((i2 * k1) << (log_m - lcur)) & M1;
  if (inverse) idx = (0u - idx) & M1;
  return idx;
}

// One round: gather the window [wb, wb+4) of the tile index into registers, butterfly, twiddle,
// scatter back in place.  `lcur` = log2 of the current sub-transform length (only used when NST==4).
template <int NST, bool INV, class F>
RONK_DEV void ntt_round(const F& f, u64* smem, const u64* tw, const NttTileArgs& A, u32 wb, u32 lcur, u32 t) {
  const u32 lowmask = (1u << wb) - 1u;
  const u32 e0 = ((t >> wb) << (wb + 4)) | (t & lowmask);
  // The swizzle is XOR-linear and e0 has no bits inside the window, so the 16 addresses are
  // swz(e0) ^ swz(q << wb): walk q in Gray-code order and pay one XOR per access.
  // byte offsets, so each access is a plain LDS/STS [reg] with no index→address arithmetic
  const u32 base = swz(e0) << 3;
  const u32 g0 = swz(1u << wb) << 3, g1 = swz(2u << wb) << 3, g2 = swz(4u << wb) << 3, g3 = swz(8u << wb) << 3;
  char* const sbytes = reinterpret_cast<char*>(smem);
  u64 x[16];
  {
    u32 addr = base;
#pragma unroll
    for (int i = 0; i < 16; i++) {
      const int q = i ^ (i >> 1);
      x[q] = *reinterpret_cast<const u64*>(sbytes + addr);
      const int flip = (i + 1) & -(i + 1);  // Gray code: bit index = ctz(i + 1)
      addr ^= (flip == 1) ? g0 : (flip == 2) ? g1 : (flip == 4) ? g2 : (flip == 8) ? g3 : 0u;
    }
  }
  radix_network<NST, INV>(f, x);
  if (NST == 4 && lcur > 4) {
    const u32 i2 = (e0 >> A.log_c) & ((1u << (lcur - 4)) - 1u);
    const u64* row = tw + A.tw_off[(A.log_m - lcur) >> 2] + i2 * TW_ROW;  // this round's table, row i2
#pragma unroll
    for (int j = 1; j < 16; j++) {
      const int k1 = ((j & 1) << 3) | ((j & 2) << 1) | ((j & 4) >> 1) | ((j & 8) >> 3);
      x[j] = f.mul_tw(x[j], row[k1]);
    }
  }
  {
    u32 addr = base;
#pragma unroll
    for (int i = 0; i < 16; i++) {
      const int q = i ^ (i >> 1);
      *reinterpret_cast<u64*>(sbytes + addr) = x[q];
      const int flip = (i + 1) & -(i + 1);
      addr ^= (flip == 1) ? g0 : (flip == 2) ? g1 : (flip == 4) ? g2 : (flip == 8) ? g3 : 0u;
    }
  }
}

// ---------------- load phase: HBM → shared ----------------
// Which formulation of the load/store phases each mode uses (bit MODE set → per-element index
// math "v0", clear → XOR-composed addresses).  The XOR-composed phases won for the strided pass 1, the
// per-element form for the contiguous pass 2.  tests/emu follows the same selection.
#ifndef RONK_LOAD_V0_MASK
#define RONK_LOAD_V0_MASK 5
#endif
#ifndef RONK_STORE_V0_MASK
#define RONK_STORE_V0_MASK 5
#endif

// Loads are issued LD_BATCH at a time into registers before any is stored, so the HBM latency of a
// tile is paid once per batch, not once per element.  nthr is a power of two, so the tile index of
// the j-th element of a thread is e = tid | (j·nthr): disjoint bit sets.  The swizzle is XOR-linear,
// hence swz(e) = swz(tid) ^ swz(j·nthr) — one XOR per element with a warp-uniform second term.
#ifndef RONK_LD_BATCH
#define RONK_LD_BATCH 8
#endif
constexpr int LD_BATCH = RONK_LD_BATCH;  // strided pass-1 columns: 8 (deeper was slower when the tile came from HBM)
// contiguous pass-2 / single tiles: a thread's whole share (32 elements) in flight (slightly faster than 16)
#ifndef RONK_LD_BATCH_CONTIG
#define RONK_LD_BATCH_CONTIG 32
#endif
RONK_DEV u32 ilog2(u32 v) {
  u32 l = 0;
  while ((1u << l) < v) l++;
  return l;
}
// Pass 1 runs one CTA per SM, so nothing overlaps a tile's strided load (4096 separate 8·C-byte
// segments) with butterflies.  Each CTA therefore asks L2 to fetch the tile of the CTA that will
// follow it on this SM (block index + number of co-resident CTAs); that load then hits L2.
// A distance of one wave of co-resident CTAs paid; two or three waves were slower than no prefetch.  The contiguous pass-2 tiles (two CTAs per SM already
// overlap each other's phases) gain nothing from the same trick, so it is not done there.
RONK_DEV void ntt_prefetch_pass1(const NttTileArgs& A, u32 tile, u32 tid, u32 nthr) {
#if defined(__CUDA_ARCH__)
  const u32 kk = ilog2(nthr);
  const u32 per_thread = (1u << A.tile_log) >> kk;
  const u32 col = tid & ((1u << A.log_c) - 1u);
  if (col & 3u) return;  // one request per 32-byte sector
  const u32 b = tile / A.tiles_per_batch, sub = tile - b * A.tiles_per_batch;
  const u64* base = A.src + ((u64)b << A.log_n) + ((u64)sub << A.log_c) + ((u64)(tid >> A.log_c) << A.log_n2) + col;
  const u64* end = A.src + A.src_len;  // a zero-padded operand is shorter than the transform: stay inside it
  for (u32 j = 0; j < per_thread; j++) {
    const u64* q = base + ((u64)((j << kk) >> A.log_c) << A.log_n2);
    if (A.src_len == NTT_UNBOUNDED || q < end) asm volatile("prefetch.global.L2 [%0];" ::"l"(q));
  }
#endif
}

// LD_BATCH loads into registers, then LD_BATCH swizzled stores (see above); BOUNDED adds `index < src_len`; COSET
// multiplies each word by c^j on its way to shared memory (f is used only then).
template <int MODE, bool BOUNDED, bool COSET = false, class F = GoldilocksField>
RONK_DEV void ntt_load_batches(u64* smem, const NttTileArgs& A, u64 gaddr_t, u32 sw_t, u32 kk, u32 per_thread,
                               const F* f = nullptr) {
  for (u32 j0 = 0; j0 < per_thread; j0 += LD_BATCH) {
    u64 v[LD_BATCH];
#pragma unroll
    for (int i = 0; i < LD_BATCH; i++) {
      const u32 gj = (j0 + i) << kk;  // warp-uniform
      if (j0 + i < per_thread) {
        u64 g;
        if (MODE == MODE_PASS1) g = gaddr_t + ((u64)(gj >> A.log_c) << A.log_n2);  // kk ≥ log_c: gj has no column bits
        else g = gaddr_t + gj;
        bool ok = true;
        if (MODE == MODE_SINGLE) ok = g < A.total;
        if (BOUNDED) ok = ok && g < A.src_len;
        v[i] = ok ? A.src[g] : 0ULL;
        if constexpr (COSET) v[i] = coset_mul(*f, v[i], A.coset_lo, A.coset_hi, A.coset_h, (u32)g & ((1u << A.log_n) - 1u));
      }
    }
#pragma unroll
    for (int i = 0; i < LD_BATCH; i++) {
      const u32 gj = (j0 + i) << kk;
      if (j0 + i < per_thread) smem[sw_t ^ swz(gj)] = v[i];
    }
  }
}

template <class F, int MODE, bool BOUNDED = false, bool COSET = false>
RONK_DEV void ntt_load_phase(u64* smem, const NttTileArgs& A, u32 tile, u32 tid, u32 nthr, const F* f = nullptr) {
  const u32 T = 1u << A.tile_log;
  const u32 kk = ilog2(nthr);
  u32 b = 0, sub = tile;
  if (MODE != MODE_SINGLE) {
    b = tile / A.tiles_per_batch;
    sub = tile - b * A.tiles_per_batch;
  }
  // thread part of the global address
  u64 gaddr_t;
  if (MODE == MODE_SINGLE) gaddr_t = ((u64)tile << A.tile_log) + tid;
  else if (MODE == MODE_PASS1)
    gaddr_t = ((u64)b << A.log_n) + ((u64)sub << A.log_c) + ((u64)(tid >> A.log_c) << A.log_n2) + (tid & ((1u << A.log_c) - 1u));
  else gaddr_t = ((u64)b << A.log_n) + ((u64)sub << A.tile_log) + tid;
  const u32 sw_t = swz(tid);
  const u32 per_thread = T >> kk;  // elements per thread (T ≥ nthr)
  ntt_load_batches<MODE, BOUNDED, COSET>(smem, A, gaddr_t, sw_t, kk, per_thread, f);
}

// Round schedule: full radix-16 rounds from the top of the NTT index down, then one partial
// round for the remaining 1–3 bits.  Returns false when there is no round `r`.
RONK_DEV bool ntt_round_plan(const NttTileArgs& A, u32 r, u32* nst, u32* wb, u32* lcur) {
  const u32 full = A.log_m / 4, rem = A.log_m % 4;
  if (r < full) {
    *nst = 4;
    *lcur = A.log_m - 4 * r;
    *wb = A.log_c + *lcur - 4;
    return true;
  }
  if (r == full && rem) {
    *nst = rem;
    *lcur = rem;
    *wb = A.log_c;
    return true;
  }
  return false;
}

// One round over the whole tile: thread `tid` of `nthr` handles the 16-element groups tid, tid+nthr, …
template <class F, bool INV>
RONK_DEV void ntt_round_dispatch(const F& f, u64* smem, const u64* tw, const NttTileArgs& A, u32 nst, u32 wb, u32 lcur,
                                 u32 tid, u32 nthr) {
  const u32 groups = (1u << A.tile_log) >> 4;
  for (u32 t = tid; t < groups; t += nthr) {
    if (nst == 4) ntt_round<4, INV>(f, smem, tw, A, wb, lcur, t);
    else if (nst == 3) ntt_round<3, INV>(f, smem, tw, A, wb, 0, t);
    else if (nst == 2) ntt_round<2, INV>(f, smem, tw, A, wb, 0, t);
    else ntt_round<1, INV>(f, smem, tw, A, wb, 0, t);
  }
}

// ---------------- store phase: shared → HBM (un-bit-reverse on the fly) ----------------
// g = tid | (j·nthr) enumerates the tile in HBM-friendly order; the tile index holding element g is a
// fixed PERMUTATION OF THE BITS of g (bit-reversal of the transform field, plus the pass-1 chunk
// shuffle), so e(g) = e(tid) | e(j·nthr) and, the swizzle being XOR-linear,
// swz(e(g)) = swz(e(tid)) ^ swz(e(j·nthr)): per element one XOR with a warp-uniform term.
template <int MODE>
RONK_DEV u32 store_perm(const NttTileArgs& A, u32 g) {
  if (MODE == MODE_SINGLE) {
    const u32 M1 = (1u << A.log_m) - 1u;
    return ((g >> A.log_m) << A.log_m) | bitrev(g & M1, A.log_m);
  } else if (MODE == MODE_PASS1) {
    const u32 lc = A.log_c, lc2 = A.log_c2, cl = lc + lc2;
    const u32 rem = g & ((1u << cl) - 1u);
    const u32 k1 = ((g >> cl) << lc2) | (rem & ((1u << lc2) - 1u));
    return (bitrev(k1, A.log_m) << lc) | (rem >> lc2);
  } else {
    const u32 lc2 = A.log_c;
    return (bitrev(g >> lc2, A.log_m) << lc2) | (g & ((1u << lc2) - 1u));
  }
}

template <class F, int MODE, bool INV, bool BOUNDED = false>
RONK_DEV void ntt_store_phase(const F& f, const u64* smem, const NttTileArgs& A, u32 tile, u32 tid, u32 nthr) {
  const u32 T = 1u << A.tile_log;
  const u32 kk = ilog2(nthr);
  const u32 per_thread = T >> kk;
  u32 b = 0, sub = tile;
  if (MODE != MODE_SINGLE) {
    b = tile / A.tiles_per_batch;
    sub = tile - b * A.tiles_per_batch;
  }
  const u32 sw_t = swz(store_perm<MODE>(A, tid));
  if (MODE == MODE_SINGLE) {
    const u64 base_t = ((u64)tile << A.tile_log) + tid;
#pragma unroll 4
    for (u32 j = 0; j < per_thread; j++) {
      const u32 gj = j << kk;
      const u64 ga = base_t + gj;
      if (ga >= A.total || (BOUNDED && ga >= A.dst_len)) continue;
      u64 v = smem[sw_t ^ swz(store_perm<MODE>(A, gj))];
      if (A.flags & NTT_FLAG_SCALE) v = f.mul_tw(v, A.scale);
      if (A.flags & NTT_FLAG_MUL) v = f.mul(v, A.mul_src[ga & A.mul_mask]);
      A.dst[ga] = v;
    }
  } else if (MODE == MODE_PASS1) {
    const u32 lc = A.log_c, lc2 = A.log_c2, cl = lc + lc2;
    const u32 nmask = (A.log_n >= 32) ? 0xFFFFFFFFu : ((1u << A.log_n) - 1u);
    const u32 lomask = (1u << A.log_lo) - 1u;
    const u64 base = (u64)b << A.log_n;
    if (kk >= cl) {
      // (column, k1 % C2) are fixed per thread and k1 advances by a constant per iteration, so the
      // inter-pass twiddle ω_n^(j2·k1) is STEPPED: w ← w·ρ with ρ = ω_n^(j2·Δk1) — one multiply
      // instead of two table gathers, the index arithmetic and the combine-multiply.
      const u32 rem = tid & ((1u << cl) - 1u);
      const u32 c = rem >> lc2, k1_in = rem & ((1u << lc2) - 1u);
      const u32 j2 = (sub << lc) | c;
      const u32 k1_t = ((tid >> cl) << lc2) | k1_in;
      const u32 dk1 = (1u << (kk - cl)) << lc2;
      const u64 dst_t = base + ((u64)(tid >> cl) << (A.log_n2 + lc2)) + ((u64)j2 << lc2) + k1_in;
      const u64 ddst = (u64)(1u << (kk - cl)) << (A.log_n2 + lc2);
      if (A.tw_full) {
        // Table form: the twiddle of workspace word i is tw_full[i mod n] — one coalesced load at the store's own
        // offset replaces the stepping multiply (a general multiply is 4 IMAD.WIDE + 13 ALU-pipe instructions) at the
        // price of 8 B/element more reads; off by default (RONK_TW_TABLE).
        const u64* tw_t = A.tw_full + (dst_t - base);
        constexpr u32 TB = 8;
        for (u32 j0 = 0; j0 < per_thread; j0 += TB) {
          u64 w[TB];
#pragma unroll
          for (u32 i = 0; i < TB; i++) w[i] = ld_tw(tw_t + (u64)(j0 + i) * ddst);
#pragma unroll
          for (u32 i = 0; i < TB; i++) {
            const u32 gj = (j0 + i) << kk;
            A.dst[dst_t + (u64)(j0 + i) * ddst] = f.mul_tw(smem[sw_t ^ swz(store_perm<MODE>(A, gj))], w[i]);
          }
        }
        return;
      }
      u32 ex0 = j2 * k1_t, exd = j2 * dk1;
      if (INV) { ex0 = (0u - ex0) & nmask; exd = (0u - exd) & nmask; }
      u64 w = f.mul_tw(ld_tw(A.tw_lo + (ex0 & lomask)), ld_tw(A.tw_hi + (ex0 >> A.log_lo)));
      const u64 rho = f.mul_tw(ld_tw(A.tw_lo + (exd & lomask)), ld_tw(A.tw_hi_plain + (exd >> A.log_lo)));
#pragma unroll 4
      for (u32 j = 0; j < per_thread; j++) {
        const u32 gj = j << kk;
        const u64 v = f.mul_tw(smem[sw_t ^ swz(store_perm<MODE>(A, gj))], w);
        A.dst[dst_t + (u64)j * ddst] = v;
        w = f.mul_tw(w, rho);
      }
    } else {
#pragma unroll 4
    for (u32 j = 0; j < per_thread; j++) {
      const u32 gj = j << kk;
      const u32 g = tid | gj;
      const u32 k1_blk = g >> cl;
      const u32 rem = g & ((1u << cl) - 1u);
      const u32 c = rem >> lc2, k1_in = rem & ((1u << lc2) - 1u);
      const u32 k1 = (k1_blk << lc2) | k1_in;
      const u32 j2 = (sub << lc) | c;
      u32 ex = j2 * k1;
      if (INV) ex = (0u - ex) & nmask;
      const u64 w = f.mul_tw(ld_tw(A.tw_lo + (ex & lomask)), ld_tw(A.tw_hi + (ex >> A.log_lo)));
      const u64 v = f.mul_tw(smem[sw_t ^ swz(store_perm<MODE>(A, gj))], w);
      A.dst[base + ((u64)k1_blk << (A.log_n2 + lc2)) + ((u64)j2 << lc2) + k1_in] = v;
    }
    }
  } else {
    const u32 lc2 = A.log_c;  // pass-2 tile: columns are the C2 adjacent k1 values
    // address of g: base + k1_in + (k2 << log_n1), additive over the disjoint bit fields of g
    const u64 addr_t = ((u64)b << A.log_n) + ((u64)sub << lc2) + (tid & ((1u << lc2) - 1u)) + ((u64)(tid >> lc2) << A.log_n1);
#pragma unroll 8
    for (u32 j = 0; j < per_thread; j++) {
      const u32 gj = j << kk;  // kk ≥ lc2: gj carries no k1_in bits
      const u64 addr = addr_t + ((u64)(gj >> lc2) << A.log_n1);
      if (BOUNDED && addr >= A.dst_len) continue;
      u64 v = smem[sw_t ^ swz(store_perm<MODE>(A, gj))];
      if (A.flags & NTT_FLAG_MUL) v = f.mul(v, A.mul_src[addr & A.mul_mask]);
      A.dst[addr] = v;
    }
  }
}

// ---- previous formulation of the phases (index math per element), kept selectable per mode ----
template <class F, int MODE, bool BOUNDED = false, bool COSET = false>
RONK_DEV void ntt_load_phase_v0(u64* smem, const NttTileArgs& A, u32 tile, u32 tid, u32 nthr, const F* f = nullptr) {
  const u32 T = 1u << A.tile_log;
  u32 b = 0, sub = tile;
  if (MODE != MODE_SINGLE) {
    b = tile / A.tiles_per_batch;
    sub = tile - b * A.tiles_per_batch;
  }
  u64 base;
  if (MODE == MODE_SINGLE) base = (u64)tile << A.tile_log;
  else if (MODE == MODE_PASS1) base = ((u64)b << A.log_n) + ((u64)sub << A.log_c);
  else base = ((u64)b << A.log_n) + ((u64)sub << A.tile_log);
  const u32 cmask = (1u << A.log_c) - 1u;
  constexpr int LB = (MODE == MODE_PASS1) ? LD_BATCH : RONK_LD_BATCH_CONTIG;
  for (u32 e0 = tid; e0 < T; e0 += nthr * LB) {
    u64 v[LB];
#pragma unroll
    for (int i = 0; i < LB; i++) {
      const u32 e = e0 + i * nthr;
      if (MODE == MODE_SINGLE) {
        const u64 g = base + e;
        v[i] = (e < T && g < A.total && (!BOUNDED || g < A.src_len)) ? A.src[g] : 0ULL;
      } else if (MODE == MODE_PASS1) {
        const u32 j1 = e >> A.log_c, c = e & cmask;
        const u64 g = base + ((u64)j1 << A.log_n2) + c;
        v[i] = (e < T && (!BOUNDED || g < A.src_len)) ? A.src[g] : 0ULL;
      } else {
        v[i] = (e < T) ? A.src[base + e] : 0ULL;
      }
    }
#pragma unroll
    for (int i = 0; i < LB; i++) {
      const u32 e = e0 + i * nthr;
      if constexpr (COSET) {   // the factor once the whole batch of loads is in flight: a word's registers die at its store
        static_assert(MODE != MODE_PASS2, "coset: the first pass");
        const u64 g = MODE == MODE_SINGLE ? base + e : base + ((u64)(e >> A.log_c) << A.log_n2) + (e & cmask);
        if (e < T) smem[swz(e)] = coset_mul(*f, v[i], A.coset_lo, A.coset_hi, A.coset_h, (u32)g & ((1u << A.log_n) - 1u));
      } else {
        if (e < T) smem[swz(e)] = v[i];
      }
    }
  }
}

// FMUL (pass 2 only): the caller guarantees NTT_FLAG_MUL; the point-wise operand is then fetched in batches
// ahead of the stores — in the plain loop every mul_src load sits behind the previous store (the two arrays
// may alias as far as the compiler knows) and pays a full memory latency per element.
template <class F, int MODE, bool INV, bool BOUNDED = false, bool FMUL = false, bool COSET = false>
RONK_DEV void ntt_store_phase_v0(const F& f, const u64* smem, const NttTileArgs& A, u32 tile, u32 tid, u32 nthr) {
  const u32 T = 1u << A.tile_log;
  const u32 M = 1u << A.log_m;
  u32 b = 0, sub = tile;
  if (MODE != MODE_SINGLE) {
    b = tile / A.tiles_per_batch;
    sub = tile - b * A.tiles_per_batch;
  }
  if (MODE == MODE_SINGLE) {
    const u64 base = (u64)tile << A.tile_log;
    for (u32 g = tid; g < T; g += nthr) {
      if (base + g >= A.total || (BOUNDED && base + g >= A.dst_len)) continue;
      const u32 bt = g >> A.log_m, k = g & (M - 1u);
      const u32 e = (bt << A.log_m) | bitrev(k, A.log_m);
      u64 v = smem[swz(e)];
      if (A.flags & NTT_FLAG_SCALE) v = f.mul_tw(v, A.scale);
      if constexpr (COSET) v = coset_mul(f, v, A.coset_lo, A.coset_hi, A.coset_h, (u32)(base + g) & (M - 1u));
      if (A.flags & NTT_FLAG_MUL) v = f.mul(v, A.mul_src[(base + g) & A.mul_mask]);
      A.dst[base + g] = v;
    }
  } else if (MODE == MODE_PASS1) {
    const u32 lc = A.log_c, lc2 = A.log_c2;
    const u32 chunk_log = lc + lc2;
    const u32 nmask = (A.log_n >= 32) ? 0xFFFFFFFFu : ((1u << A.log_n) - 1u);
    const u32 lomask = (1u << A.log_lo) - 1u;
    const u64 base = (u64)b << A.log_n;
    for (u32 g = tid; g < T; g += nthr) {
      const u32 k1_blk = g >> chunk_log;
      const u32 rem = g & ((1u << chunk_log) - 1u);
      const u32 c = rem >> lc2, k1_in = rem & ((1u << lc2) - 1u);
      const u32 k1 = (k1_blk << lc2) | k1_in;
      const u32 e = (bitrev(k1, A.log_m) << lc) | c;
      const u32 j2 = (sub << lc) | c;
      u32 ex = j2 * k1;
      if (INV) ex = (0u - ex) & nmask;
      const u64 w = f.mul_tw(ld_tw(A.tw_lo + (ex & lomask)), ld_tw(A.tw_hi + (ex >> A.log_lo)));
      const u64 v = f.mul_tw(smem[swz(e)], w);
      A.dst[base + ((u64)k1_blk << (A.log_n2 + lc2)) + ((u64)j2 << lc2) + k1_in] = v;
    }
  } else {
    const u32 lc2 = A.log_c;  // pass-2 tile: columns are the C2 adjacent k1 values
    const u64 base = ((u64)b << A.log_n) + ((u64)sub << lc2);
    if (FMUL) {
      constexpr int SB = 8;
      for (u32 g0 = tid; g0 < T; g0 += nthr * SB) {
        u64 m[SB];
#pragma unroll
        for (int i = 0; i < SB; i++) {
          const u32 g = g0 + i * nthr;
          const u64 addr = base + (g & ((1u << lc2) - 1u)) + ((u64)(g >> lc2) << A.log_n1);
          m[i] = (g < T && !(BOUNDED && addr >= A.dst_len)) ? A.mul_src[addr & A.mul_mask] : 0ULL;
        }
#pragma unroll
        for (int i = 0; i < SB; i++) {
          const u32 g = g0 + i * nthr;
          if (g >= T) continue;
          const u32 k2 = g >> lc2, k1_in = g & ((1u << lc2) - 1u);
          const u64 addr = base + k1_in + ((u64)k2 << A.log_n1);
          if (BOUNDED && addr >= A.dst_len) continue;
          A.dst[addr] = f.mul(smem[swz((bitrev(k2, A.log_m) << lc2) | k1_in)], m[i]);
        }
      }
    } else {
      for (u32 g = tid; g < T; g += nthr) {
        const u32 k2 = g >> lc2, k1_in = g & ((1u << lc2) - 1u);
        const u32 e = (bitrev(k2, A.log_m) << lc2) | k1_in;
        const u64 addr = base + k1_in + ((u64)k2 << A.log_n1);
        if (BOUNDED && addr >= A.dst_len) continue;
        u64 v = smem[swz(e)];
        if constexpr (COSET) v = coset_mul(f, v, A.coset_lo, A.coset_hi, A.coset_h, (u32)addr & ((1u << A.log_n) - 1u));
        if (A.flags & NTT_FLAG_MUL) v = f.mul(v, A.mul_src[addr & A.mul_mask]);
        A.dst[addr] = v;
      }
    }
  }
}

// ---------------- launch geometry (host; shared by ntt.cu and the CPU emulator in tests/emu) -------------
struct NttShape {
  bool two_pass;
  u32 log_n1, log_n2;  // n = N1·N2, N1 ≥ N2 (two-pass only)
};
inline NttShape ntt_shape(u32 log_n) {
  NttShape s;
  s.two_pass = log_n > 13;  // tile (128 KiB) + twiddle table must fit in 227 KiB of shared memory
  s.log_n1 = s.two_pass ? (log_n + 1) / 2 : log_n;
  s.log_n2 = s.two_pass ? log_n / 2 : 0;
  return s;
}
constexpr u32 NTT_TILE_LOG_MAX = 14;

// Whole transforms inside one tile.  tile_cap = preferred tile size (log2) when several small
// transforms share a tile.
inline NttTileArgs ntt_args_single(u64* data, const u64* mul, const u64* tw, u64 scale_inv, u32 log_n, u64 total,
                                   bool inverse, u32 tile_cap, u64* tiles) {
  NttTileArgs A = {};
  u32 want = 0;
  while (((u64)1 << want) < total) want++;
  if (want > tile_cap) want = tile_cap;
  u32 tile_log = log_n;
  if (tile_log < want) tile_log = want;
  if (tile_log < 9) tile_log = 9;
  if (tile_log > NTT_TILE_LOG_MAX) tile_log = NTT_TILE_LOG_MAX;
  A.src = data;
  A.dst = data;
  A.src_len = A.dst_len = NTT_UNBOUNDED;
  A.tw_tile = tw;
  A.tw_words = ntt_tw2d_layout(log_n, A.tw_off);
  A.mul_src = mul;
  A.mul_mask = ~0ULL;
  A.scale = scale_inv;
  A.total = total;
  A.tile_log = tile_log;
  A.log_m = log_n;
  A.log_c = 0;
  A.log_n = log_n;
  A.flags = (inverse ? NTT_FLAG_SCALE : 0) | (mul ? NTT_FLAG_MUL : 0);
  *tiles = (total + ((u64)1 << tile_log) - 1) >> tile_log;
  return A;
}
// Tile sizes of the two passes (log2 elements).  `pref` = preferred size (13 → two CTAs per SM);
// a tile can never be smaller than one transform of that pass.
inline void ntt_pass_tiles(u32 log_n, u32 pref1, u32 pref2, u32* t1, u32* t2) {
  const NttShape sh = ntt_shape(log_n);
  *t1 = pref1 < sh.log_n1 ? sh.log_n1 : (pref1 > NTT_TILE_LOG_MAX ? NTT_TILE_LOG_MAX : pref1);
  *t2 = pref2 < sh.log_n2 ? sh.log_n2 : (pref2 > NTT_TILE_LOG_MAX ? NTT_TILE_LOG_MAX : pref2);
}
inline NttTileArgs ntt_args_pass1(const u64* data, u64* ws, const u64* tw1, const u64* tw_lo, const u64* tw_hi,
                                  const u64* tw_hi_plain, u32 log_n, u32 batch, u32 tile1, u32 tile2, u64* tiles) {
  const NttShape sh = ntt_shape(log_n);
  NttTileArgs A = {};
  A.src = data;
  A.dst = ws;
  A.src_len = A.dst_len = NTT_UNBOUNDED;
  A.tw_tile = tw1;
  A.tw_words = ntt_tw2d_layout(sh.log_n1, A.tw_off);
  A.tw_lo = tw_lo;
  A.tw_hi = tw_hi;
  A.tw_hi_plain = tw_hi_plain;
  A.tile_log = tile1;
  A.log_m = sh.log_n1;
  A.log_c = tile1 - sh.log_n1;
  A.log_n = log_n;
  A.log_n1 = sh.log_n1;
  A.log_n2 = sh.log_n2;
  A.log_c2 = tile2 - sh.log_n2;
  A.log_lo = sh.log_n1;
  A.tiles_per_batch = 1u << (sh.log_n2 - A.log_c);
  *tiles = (u64)batch * A.tiles_per_batch;
  return A;
}
inline NttTileArgs ntt_args_pass2(const u64* ws, u64* data, const u64* mul, const u64* tw2, u32 log_n, u32 batch,
                                  u32 tile2, u64* tiles) {
  const NttShape sh = ntt_shape(log_n);
  NttTileArgs A = {};
  A.src = ws;
  A.dst = data;
  A.src_len = A.dst_len = NTT_UNBOUNDED;
  A.tw_tile = tw2;
  A.tw_words = ntt_tw2d_layout(sh.log_n2, A.tw_off);
  A.mul_src = mul;
  A.mul_mask = ~0ULL;
  A.tile_log = tile2;
  A.log_m = sh.log_n2;
  A.log_c = tile2 - sh.log_n2;
  A.log_n = log_n;
  A.log_n1 = sh.log_n1;
  A.log_n2 = sh.log_n2;
  A.log_c2 = A.log_c;
  A.log_lo = sh.log_n1;
  A.tiles_per_batch = 1u << (sh.log_n1 - A.log_c);
  A.flags = mul ? NTT_FLAG_MUL : 0;
  *tiles = (u64)batch * A.tiles_per_batch;
  return A;
}

#if defined(__CUDACC__)
// --- TMA (bulk async copy) staging of the twiddle table into shared memory ---------------------
__device__ __forceinline__ void mbar_init(u64* bar, u32 count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"((u32)__cvta_generic_to_shared(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(u64* bar, u32 bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"((u32)__cvta_generic_to_shared(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(u64* bar, u32 parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra WAIT_DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t}" ::"r"((u32)__cvta_generic_to_shared(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void* smem_dst, const void* gsrc, u32 bytes, u64* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   (u32)__cvta_generic_to_shared(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"((u32)__cvta_generic_to_shared(bar))
               : "memory");
}

// Shared memory: [ tile: T·8 B | twiddles: M·8 B | mbarrier: 8 B ]
// BOUNDED instantiations (poly_mul only) honour A.src_len / A.dst_len; the unbounded ones carry no such code.
// COSET instantiations (unbounded, no point-wise product) apply the coset factor c^j of NttTileArgs::coset_lo: forward in
// the load of MODE_SINGLE / MODE_PASS1, inverse in the store of MODE_SINGLE / MODE_PASS2.
template <class F, int MODE, bool INV, int NTHR, int MINB, bool BOUNDED = false, bool FMUL = false, bool COSET = false>
__global__ void __launch_bounds__(NTHR, MINB) ntt_tile_kernel(const F f, const NttTileArgs A) {
  static_assert(!COSET || (!BOUNDED && !FMUL && (MODE == MODE_SINGLE || (MODE == MODE_PASS1) != INV)),
                "coset: unbounded, forward first pass or inverse last pass");
  static_assert(!COSET || !INV || ((RONK_STORE_V0_MASK >> MODE) & 1), "the inverse coset factor is in the per-element store");
  extern __shared__ __align__(128) u64 smem[];
  const u32 tid = threadIdx.x, tile = blockIdx.x;
  const u32 T = 1u << A.tile_log;
  u64* tw = smem + T;
  u64* bar = tw + A.tw_words;
  const bool use_tw = A.log_m > 4;  // a single radix-16 round has no general twiddles
  if (use_tw && tid == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    mbar_expect_tx(bar, A.tw_words * 8u);
    tma_bulk_g2s(tw, A.tw_tile, A.tw_words * 8u, bar);  // lands while the tile itself is being loaded
  }
  // Programmatic dependent launch: pass 1 lets pass 2's CTAs be scheduled as soon as its own last wave is running;
  // they set up (mbarrier, twiddle TMA) and then wait here until pass 1 has completed and its workspace writes are
  // visible.  Both instructions are no-ops when the launch carries no PDL attribute.
  if (MODE == MODE_PASS1) asm volatile("griddepcontrol.launch_dependents;");
  if (MODE == MODE_PASS2) asm volatile("griddepcontrol.wait;" ::: "memory");
  if constexpr (COSET && !INV) {
    if ((RONK_LOAD_V0_MASK >> MODE) & 1) ntt_load_phase_v0<F, MODE, false, true>(smem, A, tile, tid, NTHR, &f);
    else ntt_load_phase<F, MODE, false, true>(smem, A, tile, tid, NTHR, &f);
  } else {
    if ((RONK_LOAD_V0_MASK >> MODE) & 1) ntt_load_phase_v0<F, MODE, BOUNDED>(smem, A, tile, tid, NTHR);
    else ntt_load_phase<F, MODE, BOUNDED>(smem, A, tile, tid, NTHR);
  }
  if (MODE == MODE_PASS1 && A.prefetch_dist && tile + A.prefetch_dist < gridDim.x)
    ntt_prefetch_pass1(A, tile + A.prefetch_dist, tid, NTHR);
  __syncthreads();
  if (use_tw) mbar_wait(bar, 0);
  u32 nst, wb, lcur;
  for (u32 r = 0; ntt_round_plan(A, r, &nst, &wb, &lcur); r++) {
    ntt_round_dispatch<F, INV>(f, smem, tw, A, nst, wb, lcur, tid, NTHR);
    __syncthreads();
  }
  if ((RONK_STORE_V0_MASK >> MODE) & 1) ntt_store_phase_v0<F, MODE, INV, BOUNDED, FMUL, COSET && INV>(f, smem, A, tile, tid, NTHR);
  else ntt_store_phase<F, MODE, INV, BOUNDED>(f, smem, A, tile, tid, NTHR);
}

// 2-D per-round twiddle table from the 1-D table ω_M^e (both in twiddle form); pads = 0
static __global__ void tw2d_gather_kernel(const u64* __restrict__ tw1d, u32 log_m, int inverse, u64* __restrict__ out, u32 words) {
  const u32 w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= words) return;
  bool valid;
  const u32 idx = ntt_tw2d_source(log_m, w, inverse != 0, &valid);
  out[w] = valid ? tw1d[idx] : 0ULL;
}

// Full inter-pass twiddle table in the pass-1 workspace layout W[k1 / C2][j2][k1 % C2]:
// out[i] = tw_lo[e & lomask] · tw_hi[e >> log_lo], e = ±j2·k1 mod n (tw_hi carries n^-1 for the inverse).
template <class F>
__global__ void interpass_table_kernel(const F f, const u64* __restrict__ tw_lo, const u64* __restrict__ tw_hi, u32 log_n,
                                       u32 log_n1, u32 log_n2, u32 log_c2, u32 log_lo, int inverse, u64* __restrict__ out) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >> log_n) return;
  const u32 k1_in = (u32)i & ((1u << log_c2) - 1u);
  const u32 j2 = (u32)(i >> log_c2) & ((1u << log_n2) - 1u);
  const u32 k1 = ((u32)(i >> (log_n2 + log_c2)) << log_c2) | k1_in;
  const u32 nmask = (log_n >= 32) ? 0xFFFFFFFFu : ((1u << log_n) - 1u);
  u32 ex = (j2 * k1) & nmask;
  if (inverse) ex = (0u - ex) & nmask;
  // product of two twiddle-form values is in twiddle form again for Goldilocks (plain residues); for the
  // Montgomery policy mul_tw(a_plainR, b_R) = a·b·R — tw_lo is stored in twiddle form, so this stays in it too
  out[i] = f.mul_tw(tw_lo[ex & ((1u << log_lo) - 1u)], tw_hi[ex >> log_lo]);
}

// tab[i] = to_tw(w^i · s) for i < count  (plan building; w, s plain residues)
template <class F>
__global__ void pow_table_kernel(const F f, u64 w, u64 s, u64* tab, u32 count) {
  const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < count) tab[i] = f.to_tw(f.mul(field_pow(f, w, (u64)i), s));
}
// The two coset tables of a coset transform of 2^log_n points, h = ⌈log_n / 2⌉ (c plain):
// out[i] = to_tw(c^i) for i < 2^h, out[2^h + i] = to_tw(c^(i·2^h)) for i < 2^(log_n - h).
template <class F>
__global__ void coset_table_kernel(const F f, u64 c, u32 h, u32 log_n, u64* out) {
  const u32 i = blockIdx.x * blockDim.x + threadIdx.x, lo = 1u << h;
  if (i >= lo + (1u << (log_n - h))) return;
  out[i] = f.to_tw(field_pow(f, c, i < lo ? (u64)i : (u64)(i - lo) << h));
}
#endif  // __CUDACC__

}  // namespace ronk
