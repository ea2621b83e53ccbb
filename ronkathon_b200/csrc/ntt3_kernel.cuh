// ntt3_kernel.cuh — the 2^24-point transform as THREE passes of 256-point transforms (round 2).
//
// Same map as Polynomial::fft / ifft (src/polynomial/mod.rs:273-323, :430-484): X[k] = Σ_j a_j ω^(jk), natural order in
// and out, canonical residues.  With j = j1·2^16 + j2·2^8 + j3 and k = k1 + k2·2^8 + k3·2^16 (all digits < 256):
//
//   pass 1  A1[k1, j2, j3] = ( Σ_j1 ω_256^(j1 k1) a[j1, j2, j3] ) · ω_n^(k1·(256 j2 + j3))        src → workspace
//   pass 2  A2[k1, k2, j3] = ( Σ_j2 ω_256^(j2 k2) A1[k1, j2, j3] ) · ω_65536^(k2 j3)               in place in the workspace
//   pass 3  X[k1 + 256 k2 + 65536 k3] = Σ_j3 ω_256^(j3 k3) A2[k1, k2, j3]                          workspace → data
//
// Why three passes when two suffice (ntt_kernel.cuh): the two-pass kernel needs 64–128 KiB tiles, so an SM holds 16 warps
// (4 per scheduler) and every tile goes through three CTA barriers and four shared-memory round trips; it ran well below
// its own integer-pipe floor and stripping a fifth of its instructions did not make it faster (DESIGN.md §3.3):
// it is bound by latency hiding, not by instruction count.  A 256-point transform per tile needs 4096 elements (16 columns:
// every global access is a full 128-byte line in all three passes) = 35 KB of shared memory and 128 threads: five CTAs per
// SM (20 warps at 96 registers; six at 80 registers were slower), ONE barrier and ONE shared-memory round trip per tile:
//
//   round 0   each thread loads its two radix-16 groups (digit d1 of the transform index) straight from HBM into
//             registers, runs the shift-twiddle network, multiplies by ω_256^(d0·k_hi) and writes the tile;
//   barrier
//   round 1   radix-16 over digit d0 from shared memory, then the inter-pass twiddle and the stores — straight from the
//             registers to the rows bitrev8 assigns them (no un-bit-reversing pass through shared memory).
//
// HBM traffic is 3 reads + 3 writes of the data instead of 2 + 2; on the H100 each pass runs close to HBM bandwidth
// (DESIGN.md §3.4).  General multiplications per element: 3·15/16 (inner) + 2 (pass 1: ω_n^(k1·m) stepped; 1 when it
// comes from the plan's n-word table, RONK_NTT3_T1) + 1 (pass 2: 64 Ki-entry table, L2-resident) = 5.8 (4.8 with the table).
//
// n = 2^20 (BASELINE config 2) reuses the two tile passes on SIXTEEN INTERLEAVED 2^16-point transforms and adds one
// register-only radix-16 pass.  With j = j1 + 16·(256 j2h + j2l) and k = 65536 k1 + k2l + 256 k2h:
//
//   pass A1 (PASS 2 code)  T[j1, k2l, j2l] = ( Σ_j2h ω_256^(j2h k2l) a[j1 + 16·(256 j2h + j2l)] ) · ω_65536^(j2l k2l)   src → data
//   pass A2 (PASS 1 code)  Y[j1, k2]       = ( Σ_j2l ω_256^(j2l k2h) T[j1, k2l, j2l] ) · ω_n^(j1·k2)                     data → workspace
//   pass C  (ntt3c_kernel) X[65536 k1 + k2] = Σ_j1 ω_16^(j1 k1) Y[j1, k2]                                               workspace → data
//
// The sixteen columns of a tile are the sixteen interleaved transforms (j1), so every global access is again a full
// 128-byte line; the twiddle of A1 is constant along a row, that of A2 is stepped like pass 1 of the 2^24 transform.
//
// ONE LAUNCH for small batches of 2^16-point transforms (ntt16c_kernel): the sixteen tiles of a transform are the sixteen
// CTAs of a thread-block cluster.  CTA s runs pass 2 on tile s and writes output (k1 = 16 q' + b, j2) straight into the
// shared memory of CTA q' — the one that runs pass 3 on columns k1 ∈ [16 q', 16 q' + 16) — through distributed shared
// memory; after a cluster barrier every CTA runs pass 3 out of its own receive buffer.  The 512 KB intermediate never
// leaves the SMs, the second launch disappears, and the transform is in place without a workspace (every input is in
// shared memory before the first output is stored).  A cluster holds 68 KB × 16 of shared memory, so full grids keep
// the two-launch form (six CTAs per SM); this is the latency path.
//
// Tile index e = (d1 << 8) | (d0 << 4) | c  (transform index i = 16·d1 + d0, column c); shared-memory word
// word(e) = 272·d1 + 17·d0 + c: additive (every access is [R + imm]) and conflict-free for lanes that differ in c
// (passes 1, 2 and every round-1 read) as well as for lanes that differ in d0 (round-0 writes of pass 3, whose
// transform axis is the contiguous one): bank = (c + d0) mod 16.
#pragma once
#include "ntt_kernel.cuh"

namespace ronk {

// 1: the two groups of a thread run as a loop — half the code (the kernel's top stall was no_instruction: six CTAs
// at different places of a 100 KB instruction stream); 2: both groups unrolled
#ifndef RONK_NTT3_UNROLL_GROUPS
#define RONK_NTT3_UNROLL_GROUPS 1
#endif
#ifndef RONK_NTT3_EARLY_TW
// bit 0: prefetch (L1) the pass-1 table twiddles of a group before its shared-memory reads and network; bit 1: the second
// group's data rows (L2) during the first group's round 0; bit 2: the pass-2 table rows; bit 3: the multiplier rows of
// the fused point-wise product in pass 3.  Off on the H100 (profiles/r04_ab_ntt3_t1_early_tw.txt): with the stepped 2^24
// twiddle, bit 0's prefetches of the group's own output lines cost pass 1 0.125 → 0.149 ms; with the 2^20 table it is neutral.
#define RONK_NTT3_EARLY_TW 0
#endif
#ifndef RONK_NTT3_STEP2
// 1: the stepped twiddle (pass 1 of 2^24, pass A2 of 2^20) as two interleaved chains: neutral at 2^24, faster on ONE
// 2^20-point transform (few warps, the dependent chain is exposed) — on.
#define RONK_NTT3_STEP2 1
#endif
#ifndef RONK_NTT3_MINB
// CTAs per SM the register budget is set for.  6 (80 registers; 6 × 35 KB is also the shared-memory limit) was the first
// choice; 5 (102 registers, no spills in pass 3) was faster than 6 and 4 (128 registers) on a 2^24 transform —
// the ALU pipe is the limiter and 20 warps with more registers feed it better than 24 with fewer.
#define RONK_NTT3_MINB 5
#endif
constexpr u32 N3_THREADS = 128;   // NG = 2 groups per thread (full grids); NG = 1: 256 threads, one group each — twice
                                  // the warps per tile for grids that do not fill the GPU (single 2^16 / 2^20 transforms)
constexpr u32 N3_TILE_WORDS = 16 * 272;  // 4352 words = 34 816 B
constexpr u32 N3C_THREADS = 128;         // the register-only passes (ntt3c_kernel, ntt3p_kernel)
RONK_HD constexpr u32 n3_word(u32 d1, u32 d0, u32 c) { return 272u * d1 + 17u * d0 + c; }
RONK_HD constexpr u32 n3_br4(int j) { return (u32)(((j & 1) << 3) | ((j & 2) << 1) | ((j & 4) >> 1) | ((j & 8) >> 3)); }

// n = 2^LOGN, 21 <= LOGN <= 24: first pass = R-point transforms with R = 2^(LOGN - 16) = 16·R0 (R0 = 2, 4, 8, 16); the
// 256-row tile then holds 16 / R0 of them side by side (column blocks of 16), so the thread mapping, the tile layout and
// passes 2 and 3 are those of the 2^24-point transform with 256 replaced by R in the strides.
RONK_HD constexpr int n3_log_r0(int logn) { return logn >= 21 ? logn - 20 : 4; }
RONK_HD constexpr u32 n3_brn(u32 v, int bits) {   // bit reversal of the low `bits` bits
  u32 r = 0;
  for (int i = 0; i < bits; i++) r |= ((v >> i) & 1u) << (bits - 1 - i);
  return r;
}

struct Ntt3Args {
  const u64* src;
  u64* dst;
  const u64* tw256;    // ω_256^x (direction applied), x < 256, twiddle form
  const u64* tw_lo;    // pass 1: ω_n^x, x < 4096 (twiddle form)
  const u64* tw_hi;    // pass 1: ω_n^(4096 y), y < 4096
  const u64* t2;       // pass 2: ω_65536^(±k2·j3) [· n^-1 for the inverse], [k2][j3], twiddle form
  const u64* t1;       // pass 1, optional: ω_n^(±k1·m) as an n-word table [k1][m] (else stepped from tw_lo / tw_hi)
  const u64* mul_src;  // pass 3, optional: point-wise multiplier indexed like the output …
  u64 mul_mask;        // … modulo this mask + 1: ~0 = one multiplier per output word, n - 1 = ONE n-word multiplier shared by
                       // every transform of the batch (the twiddle column of the distributed transform)
  u64 src_len;         // BOUNDED kernels (batch = 1): the first pass reads src[0, src_len) zero-extended,
  u64 dst_len;         //                               the last pass stores dst[0, dst_len) only
  union {
    u64 scale_tw;        // ntt3p_kernel, inverse only: R^-1 in twiddle form (the sub-transforms' tables carry n'^-1, not n^-1)
    const u64* coset;    // COSET passes (first pass forward, last pass inverse, 2^21 … 2^24): c^j = coset[j mod 2^h] ·
                         // coset[2^h + (j >> h)], twiddle form, h = ⌈log2 n / 2⌉, j = index within the transform
  };
  u32 batch;
  u32 flags;           // NTT_FLAG_MUL
};

// ---- round 0: 16 elements per group straight from global memory ----
// PASS 1, 2: group g ↔ (d0 = g >> 4, c = g & 15): element q is row i = 16 q + d0 of the tile, column c.
// PASS 3:    group g ↔ (col = g >> 4, d0 = g & 15): element q is i = 16 q + d0 of column col (i is the contiguous axis).
// First pass of 2^21 … 2^23 (LR0 = log2 R0 < 4, PASS 1 only): register q = u·R0 + d1 is row 16·d1 + d0 of sub-transform u,
// whose sixteen columns start 16·u after this thread's; radix_network<LR0> runs the 16 / R0 networks side by side.
// COSET (first pass of 2^21 … 2^24 only): each word is multiplied by c^j, j its index within its transform (n = 2^(20 + LR0)).
// Last pass of a SPLIT transform (n = 2^LI · n', LI > 0, PASS 3 only): the sixteen columns of the tile are 16 / 2^LI
// consecutive k1' of EACH of the 2^LI sub-transforms (column c ↔ sub-transform c mod 2^LI, sub_stride = n' words apart),
// so that the stores of round 1 — X[sub + 2^LI·k'] — are again sixteen contiguous words.
template <class F, int PASS, bool INV, bool BOUNDED = false, int NG = 2, int LR0 = 4, int LI = 0, bool COSET = false>
RONK_DEV void n3_round0(const F& f, u64* smem, const Ntt3Args& A, u64 tile_base, u64 row_stride, u64 col_stride, u32 tid,
                        u64 sub_stride = 0) {
  static_assert(!COSET || (PASS == 1 && !BOUNDED && LI == 0), "coset: the unbounded first pass of 2^21 … 2^24");
  constexpr u32 R0 = 1u << LR0;
#if RONK_NTT3_UNROLL_GROUPS == 1
#pragma unroll 1
#else
#pragma unroll
#endif
  for (int h = 0; h < NG; h++) {
    const u32 g = tid + (u32)h * N3_THREADS;
    const u32 d0 = (PASS == 3) ? (g & 15u) : (g >> 4), c = (PASS == 3) ? (g >> 4) : (g & 15u);
    const u64* p = A.src + tile_base + (u64)d0 * row_stride +
                   ((PASS == 3 && LI > 0) ? (u64)(c & ((1u << LI) - 1u)) * sub_stride + (u64)(c >> LI) * col_stride : (u64)c * col_stride);
#if (RONK_NTT3_EARLY_TW & 2) && defined(__CUDA_ARCH__)
    if (NG == 2 && h == 0 && !BOUNDED) {   // the second group's sixteen rows on their way (L2) while the first is computed
      const u32 g1 = g + N3_THREADS;
      const u32 e0 = (PASS == 3) ? (g1 & 15u) : (g1 >> 4), e1 = (PASS == 3) ? (g1 >> 4) : (g1 & 15u);
      const u64* pn = A.src + tile_base + (u64)e0 * row_stride + (u64)e1 * col_stride;
#pragma unroll
      for (int q = 0; q < 16; q++) asm volatile("prefetch.global.L2 [%0];" ::"l"(pn + (u64)q * 16u * row_stride) : "memory");
    }
#endif
    u64 x[16];
#pragma unroll
    for (int q = 0; q < 16; q++) {
      const u64 off = (u64)((u32)q & (R0 - 1u)) * 16u * row_stride + (u64)((u32)q >> LR0) * 16u * col_stride;  // LR0 = 4: q·16·row_stride
      if (BOUNDED) {
        const u64 idx = tile_base + (u64)d0 * row_stride + (u64)c * col_stride + off;
        x[q] = idx < A.src_len ? p[off] : 0;
      } else {
        x[q] = p[off];
      }
      if constexpr (COSET) {
        constexpr u32 LOGN = 20 + LR0, H = (LOGN + 1) / 2;
        const u32 j = (u32)(tile_base + (u64)d0 * row_stride + (u64)c * col_stride + off) & ((1u << LOGN) - 1u);
        x[q] = coset_mul(f, x[q], A.coset, A.coset + (1u << H), H, j);
      }
    }
    radix_network<LR0, INV>(f, x);
    // ω_R^(d0·k_lo) = ω_256^(d0·k_lo·16/R0), k_lo = bitrev_LR0(register index mod R0); nothing to do where k_lo = 0
    const u64* tw = A.tw256;
    u64* s = smem + n3_word(0, d0, c);
#pragma unroll
    for (int j = 0; j < 16; j++) {
      constexpr u32 sc = 16u >> LR0;
      const u32 kl = n3_brn((u32)j & (R0 - 1u), LR0);
      if (kl == 0) s[n3_word((u32)j, 0, 0)] = x[j];
      else s[n3_word((u32)j, 0, 0)] = f.mul_tw(x[j], ld_tw(tw + kl * sc * d0));
    }
  }
}

// ---- round 1 + inter-pass twiddle + stores ----
// group g ↔ (d1 = g >> 4, c = g & 15).  Register q is tile position d0 = q, i.e. output k = bitrev8(16 d1 + q) =
// 16·bitrev4(q) + bitrev4(d1); it goes to row k of the output view, column c.
// COSET (last pass of 2^21 … 2^24 only): each output word is multiplied by c^j, j its index within its transform.
template <class F, int PASS, bool INV, bool BOUNDED = false, int LOGN = 24, int NG = 2, bool COSET = false>
RONK_DEV void n3_round1(const F& f, const u64* smem, const Ntt3Args& A, u64 tile_base, u64 row_stride, u32 m_base, u32 tid) {
  static_assert(!COSET || (PASS == 3 && !BOUNDED && LOGN >= 21), "coset: the unbounded last pass of 2^21 … 2^24");
  constexpr u32 LO = (u32)(LOGN + 1) / 2u;                // two-level twiddle tables (the plan's split): ω_n^x, x < 2^LO, and ω_n^(2^LO·y)
  constexpr u32 EMASK = (1u << LOGN) - 1u;                // exponents mod n
  constexpr bool P1 = PASS == 1 && LOGN >= 21;            // first pass of 2^21 … 2^24: R = 16·R0 points, 16 / R0 column blocks per tile
  constexpr int LR0 = P1 ? n3_log_r0(LOGN) : 4;
  constexpr u32 R0 = 1u << LR0;
#if RONK_NTT3_UNROLL_GROUPS == 1
#pragma unroll 1
#else
#pragma unroll
#endif
  for (int h = 0; h < NG; h++) {
    const u32 g = tid + (u32)h * N3_THREADS;
    const u32 d1 = g >> 4, c0 = g & 15u;
    // tile slot d1 = u·R0 + position of the round-0 register: column block u, low output digit b = bitrev(position)
    const u32 b = bitrev(d1 & (R0 - 1u), LR0);
    const u32 c = c0 + 16u * (d1 >> LR0);                 // column within the tile's 256 / R0 columns (LR0 = 4: c0)
    const u64* s = smem + n3_word(d1, 0, c0);
#if (RONK_NTT3_EARLY_TW & 1) && defined(__CUDA_ARCH__)
    // The table twiddles of this group are PREFETCHED (L1) before the shared-memory reads and the network: loaded where
    // they are used (the compiler keeps them behind the run-time `if (A.t1)`, and sinks even explicit early loads to save
    // registers), their DRAM latency was the top stall of pass 1 (long_scoreboard).
    if (PASS == 1 && (LOGN >= 21 || LOGN == 20)) {
      // no branch on A.t1 here (the compiler would merge it with the one below and sink the prefetches into it): without
      // a table the prefetches go to the sixteen lines this group is about to store to — valid, spread over the tile like
      // the table rows (one shared address for all threads was much slower: every warp of the GPU on one L1 line)
      const u64* t = A.t1 ? (LOGN >= 21 ? A.t1 + ((u64)b << 16) + m_base + c : A.t1 + 16u * m_base + ((u64)b << 12) + c)
                          : A.dst + tile_base + (u64)b * row_stride + c;
      const u64 st = A.t1 ? (LOGN >= 21 ? ((u64)R0 << 16) : ((u64)1 << 16)) : (u64)R0 * row_stride;
#pragma unroll
      for (int qp = 0; qp < 16; qp++) asm volatile("prefetch.global.L1 [%0];" ::"l"(t + (u64)qp * st) : "memory");
    }
#endif
#if (RONK_NTT3_EARLY_TW & 8) && defined(__CUDA_ARCH__)
    if (PASS == 3) {   // the point-wise multiplier rows of the fused product (poly_mul), same idea and same select trick
      const bool fm = (A.flags & NTT_FLAG_MUL) != 0;
      const u64* t = fm ? A.mul_src + ((tile_base + (u64)b * row_stride + c) & A.mul_mask) : (const u64*)A.dst + tile_base + (u64)b * row_stride + c;
#pragma unroll
      for (int qp = 0; qp < 16; qp++) asm volatile("prefetch.global.L1 [%0];" ::"l"(t + (u64)qp * 16u * row_stride) : "memory");
    }
#endif
#if (RONK_NTT3_EARLY_TW & 4) && defined(__CUDA_ARCH__)
    if (PASS == 2) {   // the L2-resident 64 Ki-entry table of pass 2 (pass A1 of 2^20), same idea
      const u64* t = A.t2 + ((u64)b << 8) + m_base + (LOGN == 20 ? 0u : c);
#pragma unroll
      for (int qp = 0; qp < 16; qp++) asm volatile("prefetch.global.L1 [%0];" ::"l"(t + ((u64)qp << 12)) : "memory");
    }
#endif
    u64 x[16];
#pragma unroll
    for (int q = 0; q < 16; q++) x[q] = s[n3_word(0, (u32)q, 0)];
    radix_network<4, INV>(f, x);
    u64* o = A.dst + tile_base + (u64)b * row_stride + c;   // row k = R0 q' + b, q' = bitrev4(register index) (R0 = 16 unless first pass of 2^21 … 2^23)
    if (PASS == 1 && LOGN >= 21 && A.t1) {
      // ω_n^(±k1·m) from the n-word table [k1][m]: the same offsets as the stores, one coalesced load each
      const u64* t = A.t1 + ((u64)b << 16) + m_base + c;
      u64 w[16];
#pragma unroll
      for (int qp = 0; qp < 16; qp++) w[qp] = ld_tw(t + (u64)qp * ((u64)R0 << 16));
#pragma unroll
      for (int qp = 0; qp < 16; qp++) o[(u64)qp * R0 * row_stride] = f.mul_tw(x[n3_br4(qp)], w[qp]);
    } else if (PASS == 1 && LOGN == 20 && A.t1) {
      // pass A2 of 2^20: ω_n^(±j1·k2) from the n-word table indexed like this pass's output (16·k2 + j1)
      const u64* t = A.t1 + 16u * m_base + ((u64)b << 12) + c;
      u64 w[16];
#pragma unroll
      for (int qp = 0; qp < 16; qp++) w[qp] = ld_tw(t + ((u64)qp << 16));
#pragma unroll
      for (int qp = 0; qp < 16; qp++) o[(u64)qp * 16u * row_stride] = f.mul_tw(x[n3_br4(qp)], w[qp]);
    } else if (PASS == 1) {
      // ω_n^(±k1·m), m = 256 j2 + j3 (this thread's column), k1 = 16 q' + b: stepped over q' with ρ = ω_n^(±16 m)
      // 2^20 (pass A2): ω_n^(j1·k2), j1 = c (this thread's column), k2 = m_base + 256·(16 q' + b): ρ = ω_n^(4096 c)
      // first pass of 2^21 … 2^23: k1 = R0 q' + b, ρ = ω_n^(±R0 m)
      const u32 m = m_base + c;
      u32 ex0 = (LOGN == 20) ? c * (m_base + 256u * b) : m * b, exd = (LOGN == 20) ? (c << 12) : (m * R0);
      if (INV) { ex0 = (0u - ex0) & EMASK; exd = (0u - exd) & EMASK; }
      u64 w = f.mul_tw(ld_tw(A.tw_lo + (ex0 & ((1u << LO) - 1u))), ld_tw(A.tw_hi + (ex0 >> LO)));
      const u64 rho = f.mul_tw(ld_tw(A.tw_lo + (exd & ((1u << LO) - 1u))), ld_tw(A.tw_hi + (exd >> LO)));
#if RONK_NTT3_STEP2
      // two interleaved stepping chains (even / odd rows, ratio ρ²): one more multiply per group, half the dependent chain
      const u64 rho2 = f.mul_tw(rho, rho);
      u64 w1 = f.mul_tw(w, rho);
#pragma unroll
      for (int qp = 0; qp < 16; qp += 2) {
        o[(u64)qp * R0 * row_stride] = f.mul_tw(x[n3_br4(qp)], w);
        o[(u64)(qp + 1) * R0 * row_stride] = f.mul_tw(x[n3_br4(qp + 1)], w1);
        if (qp < 14) { w = f.mul_tw(w, rho2); w1 = f.mul_tw(w1, rho2); }
      }
#else
#pragma unroll
      for (int qp = 0; qp < 16; qp++) {
        o[(u64)qp * R0 * row_stride] = f.mul_tw(x[n3_br4(qp)], w);
        if (qp < 15) w = f.mul_tw(w, rho);
      }
#endif
    } else if (PASS == 2) {
      // ω_65536^(±k2·j3) from the 64 Ki-entry table [k2][j3]; m_base = first j3 of the tile
      // 2^20 (pass A1): ω_65536^(k2l·j2l) with j2l = m_base the same for all sixteen columns
      const u64* t = A.t2 + ((u64)b << 8) + m_base + (LOGN == 20 ? 0u : c);
      u64 w[16];
#pragma unroll
      for (int qp = 0; qp < 16; qp++) w[qp] = ld_tw(t + ((u64)qp << 12));
#pragma unroll
      for (int qp = 0; qp < 16; qp++) o[(u64)qp * 16u * row_stride] = f.mul_tw(x[n3_br4(qp)], w[qp]);
    } else {
      const u64 idx0 = tile_base + (u64)b * row_stride + c;   // index of row q' = 0 within the transform (BOUNDED: batch = 1)
      if (A.flags & NTT_FLAG_MUL) {
        const u64* mp = A.mul_src + (idx0 & A.mul_mask);   // a tile never straddles two transforms: the row offsets stay inside
        u64 w[16];
#pragma unroll
        for (int qp = 0; qp < 16; qp++) w[qp] = mp[(u64)qp * 16u * row_stride];
#pragma unroll
        for (int qp = 0; qp < 16; qp++)
          if (!BOUNDED || idx0 + (u64)qp * 16u * row_stride < A.dst_len) o[(u64)qp * 16u * row_stride] = f.mul(x[n3_br4(qp)], w[qp]);
      } else if constexpr (COSET) {
#pragma unroll
        for (int qp = 0; qp < 16; qp++)
          o[(u64)qp * 16u * row_stride] =
              coset_mul(f, x[n3_br4(qp)], A.coset, A.coset + (1u << LO), LO, (u32)(idx0 + (u64)qp * 16u * row_stride) & EMASK);
      } else {
#pragma unroll
        for (int qp = 0; qp < 16; qp++)
          if (!BOUNDED || idx0 + (u64)qp * 16u * row_stride < A.dst_len) o[(u64)qp * 16u * row_stride] = x[n3_br4(qp)];
      }
    }
  }
}

// ---- round 1 of pass 2 inside a cluster: twiddle as PASS 2 (LOGN = 16), stores into the pass-3 CTAs' receive buffers ----
// receive buffer of CTA t: R[col][i] = A2[k1 = 16 t + col][j2 = i] at word col·N3_RECV_STRIDE + i — exactly the view
// n3_round0<PASS 3> reads with row stride 1 and column stride N3_RECV_STRIDE.  Both the stores (16 lanes = 16 consecutive
// j2 of one column) and those reads (16 lanes = 16 consecutive i) are 128-byte runs: conflict-free.
constexpr u32 N3_RECV_STRIDE = 256;
constexpr u32 N3_RECV_WORDS = 16 * N3_RECV_STRIDE;
template <class F, bool INV, int NG, class Remote>
RONK_DEV void n3_round1_cluster(const F& f, const u64* smem, const Ntt3Args& A, u32 s_tile, u32 tid, const Remote& remote) {
#pragma unroll 1
  for (int h = 0; h < NG; h++) {
    const u32 g = tid + (u32)h * N3_THREADS;
    const u32 d1 = g >> 4, c = g & 15u;
    const u64* s = smem + n3_word(d1, 0, c);
    u64 x[16];
#pragma unroll
    for (int q = 0; q < 16; q++) x[q] = s[n3_word(0, (u32)q, 0)];
    radix_network<4, INV>(f, x);
    const u32 b = bitrev(d1, 4);
    const u32 j2 = 16u * s_tile + c;
    const u64* t = A.t2 + ((u64)b << 8) + j2;   // ω_65536^(±k1·j2) [· n^-1], k1 = 16 q' + b
    u64 w[16];
#pragma unroll
    for (int qp = 0; qp < 16; qp++) w[qp] = ld_tw(t + ((u64)qp << 12));
#pragma unroll
    for (int qp = 0; qp < 16; qp++) remote((u32)qp)[b * N3_RECV_STRIDE + j2] = f.mul_tw(x[n3_br4(qp)], w[qp]);
  }
}

// tile → addresses.  LOGN = 24: 4096 tiles per transform in every pass:
//   pass 1: tile = (j2, s): rows j1 (stride 65536), columns j3 = 16 s + c           — in and out views identical
//   pass 2: tile = (k1, s): rows j2 (stride 256),   columns j3 = 16 s + c           — in and out views identical
//   pass 3: tile = (k2, t): input column col ↔ k1 = 16 t + col (stride 65536), index i = j3 contiguous;
//                           output rows k3 (stride 65536), columns k1 = 16 t + col
// LOGN = 16 (n = 256·256, BASELINE config 5): the same two kernels without pass 1 — 16 tiles per transform:
//   pass 2: tile = s: rows j1 (stride 256), columns j2 = 16 s + c, twiddle ω_n^(k1·j2) = the [k1][j2] table
//   pass 3: tile = t: input column col ↔ k1 = 16 t + col (stride 256), i = j2 contiguous; output X[k1 + 256 k2]
template <int PASS, int LOGN, int LI = 0>
RONK_DEV void n3_tile_geometry(u32 tile, u64* in_base, u64* in_row, u64* in_col, u64* out_base, u64* out_row, u32* m_base) {
  if (PASS == 3 && LI > 0) {
    // last pass of a split transform n = 2^LI·n', n' = 2^LOGN (16 or >= 21): a tile serves 16 >> LI values of k1' of all
    // 2^LI sub-transforms of one n-point transform gb; out view: X[sub + 2^LI·(k1' + R' k2 [+ 256 R' k3])]
    constexpr int L = LOGN >= 21 ? LOGN : 24;
    if (LOGN == 16) {
      const u64 gb = tile >> (4 + LI);
      const u32 tt = tile & ((16u << LI) - 1u);
      *in_base = (gb << (16 + LI)) + ((u64)((16u >> LI) * tt) << 8);
      *in_row = 1;
      *in_col = 256;
      *out_base = (gb << (16 + LI)) + 16u * tt;
      *out_row = (u64)256 << LI;
    } else {
      const u64 gb = tile >> (L - 12 + LI);
      const u32 t = tile & ((1u << (L - 12 + LI)) - 1u);
      const u32 hi = t >> (L - 20 + LI), lo = t & ((1u << (L - 20 + LI)) - 1u);   // hi = k2, lo = tt
      *in_base = (gb << (L + LI)) + ((u64)((16u >> LI) * lo) << 16) + ((u64)hi << 8);
      *in_row = 1;
      *in_col = 65536;
      *out_base = (gb << (L + LI)) + ((u64)hi << (L - 16 + LI)) + 16u * lo;
      *out_row = (u64)1 << (L - 8 + LI);
    }
    *m_base = 0;
    return;
  }
  if (LOGN == 16) {
    const u64 b = tile >> 4;
    const u32 lo = tile & 15u;
    if (PASS == 2) {
      *in_base = *out_base = (b << 16) + 16u * lo;
      *in_row = *out_row = 256;
      *in_col = 1;
      *m_base = 16u * lo;
    } else {
      *in_base = (b << 16) + ((u64)(16u * lo) << 8);
      *in_row = 1;
      *in_col = 256;
      *out_base = (b << 16) + 16u * lo;
      *out_row = 256;
      *m_base = 0;
    }
    return;
  }
  if (LOGN == 20) {   // 256 tiles per transform in both passes; the 16 columns are the interleaved transforms j1
    const u64 b = tile >> 8;
    const u32 t = tile & 255u;
    *in_col = 1;
    *m_base = t;
    *out_base = (b << 20) + 16u * t;
    *out_row = 4096;
    if (PASS == 2) {      // A1: t = j2l, rows j2h → k2l, in and out views identical
      *in_base = *out_base;
      *in_row = 4096;
    } else {              // A2: t = k2l, rows j2l (one contiguous 4096-word block) → rows k2h of the natural-order view
      *in_base = (b << 20) + 4096u * t;
      *in_row = 16;
    }
    return;
  }
  // LOGN = 21 … 24: R = 2^(LOGN-16) rows in pass 1 (R = 256 at 2^24), n / 4096 tiles per transform in every pass:
  //   pass 1: tile t: rows j1 (stride 65536), columns m = (4096 / R)·t + …  (16 / R0 column blocks of 16)   — in = out view
  //   pass 2: tile (k1 = t >> 4, s = t & 15): rows j2 (stride 256), columns j3 = 16 s + c                    — in = out view
  //   pass 3: tile (k2 = t / (R/16), tt): input column col ↔ k1 = 16 tt + col (stride 65536), i = j3 contiguous;
  //           output X[k1 + R k2 + 256 R k3]: rows k3 (stride 256 R), columns k1
  constexpr int L = LOGN >= 21 ? LOGN : 24;   // (the two small sizes returned above; keeps their dead code well-formed)
  const u64 b = tile >> (L - 12);
  const u32 t = tile & ((1u << (L - 12)) - 1u);
  if (PASS == 1) {
    const u32 mb = t << (24 - L + 4);   // (4096 / R) columns per tile
    *in_base = *out_base = (b << L) + mb;
    *in_row = *out_row = 65536;
    *in_col = 1;
    *m_base = mb;
  } else if (PASS == 2) {
    const u32 hi = t >> 4, lo = t & 15u;   // hi = k1, lo = s
    *in_base = *out_base = (b << L) + ((u64)hi << 16) + 16u * lo;
    *in_row = *out_row = 256;
    *in_col = 1;
    *m_base = 16u * lo;
  } else {
    const u32 hi = t >> (L - 20), lo = t & ((1u << (L - 20)) - 1u);   // hi = k2, lo = tt
    *in_base = (b << L) + ((u64)(16u * lo) << 16) + ((u64)hi << 8);
    *in_row = 1;
    *in_col = 65536;
    *out_base = (b << L) + ((u64)hi << (L - 16)) + 16u * lo;
    *out_row = (u64)1 << (L - 8);
    *m_base = 0;
  }
}

// First pass of a split transform n = R·n', R = 2^LI <= 8 (2^17 … 2^19 = R·2^16, 2^25 / 2^26 = R·2^24): for every column
// m < n' a radix-R network over the R elements n' apart, times ω_n^(±k1·m) (w = ω_n^(±m) from the two-level tables, its
// powers by repeated multiplication), in place.  A thread takes 16 / R columns, n' / (16 / R) apart: sixteen registers,
// every access coalesced.  Sub-transform k1 = bitrev(register index) is the contiguous block [k1·n', (k1+1)·n').
template <class F, bool INV, int LI>
RONK_DEV void n3p_columns(const F& f, const Ntt3Args& A, u64 base, u64 mm, u32 log_np, u32 log_lo) {
  constexpr u32 R = 1u << LI, CT = 16u >> LI;
  const u64 np = (u64)1 << log_np, cstep = np / CT;
  const u64* p = A.src + base + mm;
  u64 x[16];
#pragma unroll
  for (int q = 0; q < 16; q++) x[q] = p[(u64)((u32)q & (R - 1u)) * np + (u64)((u32)q >> LI) * cstep];
  radix_network<LI, INV>(f, x);
  u64* o = A.dst + base + mm;
  const u32 nmask = (u32)((np << LI) - 1u);
#pragma unroll
  for (u32 u = 0; u < CT; u++) {
    u32 ex = (u32)(mm + (u64)u * cstep);          // m < n' <= 2^24
    if (INV) ex = (0u - ex) & nmask;
    const u64 w1 = f.mul_tw(ld_tw(A.tw_lo + (ex & ((1u << log_lo) - 1u))), ld_tw(A.tw_hi + (ex >> log_lo)));
    u64 wk[R];                                     // wk[k] = ω_n^(±k·m) [· R^-1 for the inverse] in twiddle form, k >= 1
    wk[1] = INV ? f.mul_tw(w1, A.scale_tw) : w1;
#pragma unroll
    for (u32 k = 2; k < R; k++) wk[k] = f.mul_tw(wk[k - 1], w1);
#pragma unroll
    for (u32 j = 0; j < R; j++) {
      const u32 k1 = n3_brn(j, LI);
      const u64 v = x[u * R + j];
      o[(u64)k1 * np + (u64)u * cstep] = k1 ? f.mul_tw(v, wk[k1]) : (INV ? f.mul_tw(v, A.scale_tw) : v);
    }
  }
}

// pass C body for one (transform b, k2): register q of the DIF network holds output k1 = bitrev4(q)
template <class F, bool INV>
RONK_DEV void n3c_point(const F& f, const Ntt3Args& A, u64 b, u64 k2) {
  const u64* p = A.src + (b << 20) + 16u * k2;
  u64 x[16];
#pragma unroll
  for (int q = 0; q < 16; q++) x[q] = p[q];
  radix_network<4, INV>(f, x);
  u64* o = A.dst + (b << 20) + k2;
  if (A.flags & NTT_FLAG_MUL) {
    const u64* mp = A.mul_src + (((b << 20) + k2) & A.mul_mask);
#pragma unroll
    for (int q = 0; q < 16; q++) o[(u64)n3_br4(q) << 16] = f.mul(x[q], mp[(u64)n3_br4(q) << 16]);
  } else {
#pragma unroll
    for (int q = 0; q < 16; q++) o[(u64)n3_br4(q) << 16] = x[q];
  }
}

#if defined(__CUDACC__)
// COSET: the coset factor of Ntt3Args::coset_lo on the loads of PASS 1 (forward) or the stores of PASS 3 (inverse), 2^21 … 2^24.
template <class F, int PASS, bool INV, int LOGN, bool BOUNDED, int NG = 2, int LI = 0, bool COSET = false>
__global__ void __launch_bounds__(N3_THREADS * (2 / NG), RONK_NTT3_MINB / (2 / NG)) ntt3_kernel(const F f, const Ntt3Args A) {
  __shared__ u64 smem[N3_TILE_WORDS];
  const u32 tid = threadIdx.x;
  u64 in_base, in_row, in_col, out_base, out_row;
  u32 m_base;
  n3_tile_geometry<PASS, LOGN, LI>(blockIdx.x, &in_base, &in_row, &in_col, &out_base, &out_row, &m_base);
  // programmatic dependent launch: a pass may be scheduled while its predecessor's last wave is still running; it must
  // not touch the predecessor's output before griddepcontrol.wait (no-ops without the launch attribute)
  asm volatile("griddepcontrol.launch_dependents;");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  n3_round0<F, PASS, INV, BOUNDED && PASS == (LOGN >= 21 ? 1 : 2), NG, (PASS == 1 && LOGN >= 21) ? n3_log_r0(LOGN) : 4, LI,
            COSET && !INV>(f, smem, A, in_base, in_row, in_col, tid, (u64)1 << LOGN);  // src_len: first pass only
  __syncthreads();
  n3_round1<F, PASS, INV, BOUNDED, LOGN, NG, COSET && INV>(f, smem, A, out_base, out_row, m_base, tid);
}

// One 2^16-point transform per 16-CTA cluster, in place (see the header comment).  256 threads, one group each.
struct N3ClusterRemote {
  u64* recv;
  __device__ __forceinline__ u64* operator()(u32 rank) const {
    u64* r;   // mapa: the same shared-memory offset in CTA `rank` of this cluster (generic address)
    asm("mapa.u64 %0, %1, %2;" : "=l"(r) : "l"(recv), "r"(rank));
    return r;
  }
};
template <class F, bool INV>
__global__ void __launch_bounds__(2 * N3_THREADS, 3) ntt16c_kernel(const F f, const Ntt3Args A) {
  extern __shared__ __align__(16) u64 n3_dyn[];
  u64* tile = n3_dyn;
  u64* recv = n3_dyn + N3_TILE_WORDS;
  const u32 tid = threadIdx.x;
  u32 rank;
  asm("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
  u64 in_base, in_row, in_col, out_base, out_row;
  u32 m_base;
  n3_tile_geometry<2, 16>(blockIdx.x, &in_base, &in_row, &in_col, &out_base, &out_row, &m_base);
  n3_round0<F, 2, INV, false, 1>(f, tile, A, in_base, in_row, in_col, tid);
  __syncthreads();
  // every CTA of the cluster is running (its receive buffer exists) and has its inputs in shared memory
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
  n3_round1_cluster<F, INV, 1>(f, tile, A, rank, tid, N3ClusterRemote{recv});
  // all sixteen CTAs' stores into this CTA's receive buffer have landed
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
  Ntt3Args B = A;
  B.src = recv;
  n3_round0<F, 3, INV, false, 1>(f, tile, B, 0, 1, N3_RECV_STRIDE, tid);
  __syncthreads();
  n3_tile_geometry<3, 16>(blockIdx.x, &in_base, &in_row, &in_col, &out_base, &out_row, &m_base);
  n3_round1<F, 3, INV, false, 16, 1>(f, tile, A, out_base, out_row, m_base, tid);
}

template <class F, bool INV, int LI>
__global__ void __launch_bounds__(N3C_THREADS) ntt3p_kernel(const F f, const Ntt3Args A, u32 log_np, u32 log_lo) {
  const u64 i = (u64)blockIdx.x * N3C_THREADS + threadIdx.x;   // < batch · n' / (16 / R)
  const u32 log_ct = 4 - LI, log_per = log_np - log_ct;
  asm volatile("griddepcontrol.launch_dependents;");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (i >= ((u64)A.batch << log_per)) return;
  const u64 b = i >> log_per, mm = i & (((u64)1 << log_per) - 1);
  n3p_columns<F, INV, LI>(f, A, b << (log_np + LI), mm, log_np, log_lo);
}

// pass C of the 2^20-point transform: one thread per (transform, k2) — sixteen contiguous words in, a radix-16 network in
// registers (no twiddles: ω_16 is a power of two), sixteen stores at stride 65536, coalesced across the warp.
template <class F, bool INV>
__global__ void __launch_bounds__(N3C_THREADS) ntt3c_kernel(const F f, const Ntt3Args A) {
  const u64 i = (u64)blockIdx.x * N3C_THREADS + threadIdx.x;   // < batch · 65536
  asm volatile("griddepcontrol.launch_dependents;");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (i >= ((u64)A.batch << 16)) return;
  const u64 b = i >> 16, k2 = i & 0xFFFFu;
  n3c_point<F, INV>(f, A, b, k2);
}

// T1[k1][m] = ω_n^(±k1·m), k1 < 256, m < 65536 (twiddle form), from the two-level tables
template <class F>
__global__ void ntt3_t1_kernel(const F f, const u64* __restrict__ tw_lo, const u64* __restrict__ tw_hi, int inverse, u64* __restrict__ out,
                               u32 log_n) {
  const u32 i = blockIdx.x * blockDim.x + threadIdx.x;  // < n = 2^log_n, 21 <= log_n <= 24; two-level tables split at ceil(log_n / 2)
  const u32 k1 = i >> 16, m = i & 0xFFFFu, mask = (1u << log_n) - 1u, lo = (log_n + 1u) / 2u;
  u32 ex = (k1 * m) & mask;
  if (inverse) ex = (0u - ex) & mask;
  out[i] = f.mul_tw(tw_lo[ex & ((1u << lo) - 1u)], tw_hi[ex >> lo]);
}

// 2^20: T1[16·k2 + j1] = ω_n^(±j1·k2), k2 < 65536, j1 < 16 — indexed like the output of pass A2 (10 / 10 two-level tables)
template <class F>
__global__ void ntt3_t1_20_kernel(const F f, const u64* __restrict__ tw_lo, const u64* __restrict__ tw_hi, int inverse, u64* __restrict__ out) {
  const u32 i = blockIdx.x * blockDim.x + threadIdx.x;  // < 2^20
  u32 ex = ((i >> 4) * (i & 15u)) & 0xFFFFFu;
  if (inverse) ex = (0u - ex) & 0xFFFFFu;
  out[i] = f.mul_tw(tw_lo[ex & 1023u], tw_hi[ex >> 10]);
}

// T2[k2][j3] = to_tw(ω_65536^(±k2·j3) · s): 64 Ki entries
template <class F>
__global__ void ntt3_t2_kernel(const F f, u64 w65536, u64 s, u64* out) {
  const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 65536u) return;
  const u32 k2 = i >> 8, j3 = i & 255u;
  out[i] = f.to_tw(f.mul(field_pow(f, w65536, (u64)(k2 * j3)), s));
}
#endif

}  // namespace ronk
