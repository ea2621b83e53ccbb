// field.cuh — device-side PrimeField arithmetic (sm_90a, integer pipes only).
//
// Mirrors src/algebra/field/prime/arithmetic.rs (Add :6, Sub :22-27, Mul :37, Neg :64) on
// canonical residues.  Two field policies share every kernel in this library:
//   GoldilocksField  p = 2^64 - 2^32 + 1 baked in: reduction by 2^64 ≡ 2^32-1, 2^96 ≡ -1 and
//                    multiplication by the 16th roots of unity as shifts (they are powers of two);
//   MontField        any odd modulus < 2^64 given at run time (Montgomery REDC) — the path the
//                    reference's own moduli p = 101 / 17 / 127 run through as the bit-exact cross-check.
// "Twiddle form" is what mul_tw's second operand must be in: plain residues for Goldilocks,
// Montgomery form (w·2^64 mod p) for MontField, so data never leaves normal form.
#pragma once
#include <cstdint>

namespace ronk {

typedef uint64_t u64;
typedef unsigned int u32;

// Every arithmetic routine is __host__ __device__ so that tests/emu can compile the very same
// source for the CPU and check the kernel logic without a GPU (test infrastructure only — the
// product library never runs these on the host).
#if defined(__CUDACC__)
#define RONK_DEV __host__ __device__ __forceinline__
#define RONK_HD __host__ __device__ __forceinline__
#else
#define RONK_DEV inline
#define RONK_HD inline
#endif

RONK_HD uint64_t mulhi64(uint64_t a, uint64_t b) {
#if defined(__CUDA_ARCH__)
  return __umul64hi(a, b);
#else
  return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}

constexpr u64 GL_P = 0xFFFFFFFF00000001ULL;
constexpr u64 GL_EPS = 0xFFFFFFFFULL;  // 2^64 mod p

// ------------------------------------------------------------------------------------------
// Goldilocks
// ------------------------------------------------------------------------------------------
// Correction tail "(hi:lo) -= EPS·borrow" with m = 0 / 0xFFFFFFFF the borrow mask.  Two forms:
//   sub-family: lo -= m (borrow out), hi -= borrow       → IADD3 + IADD3.X (both on the ALU pipe)
//   add-family: (hi:lo) += (m : m·m), m·m = 0 / 1        → IMAD + IADD3 + IMAD.X (one ALU op)
// The butterfly network is throttled by the ALU pipe while the FMA pipe idles, so the longer
// add-family form is the faster one where ptxas keeps it on the FMA pipe.  RONK_FMA_TAIL selects it
// per operation: bit 0 sub, bit 1 add, bit 2 both reduce tails, bit 3 / bit 4 first / second reduce
// tail only.  3 is the default: 0 (every tail on the ALU pipe) was clearly slower, 11 / 19 no faster on a 2^24
// transform, and the longer add-family chains of 19 slow a latency-bound single 2^20-point transform.
#ifndef RONK_FMA_TAIL
#define RONK_FMA_TAIL 3
#endif
#define RONK_TAIL_SUBFAM(lo, hi) "sub.cc.u32 " lo ", " lo ", m;\n\t" "subc.u32 " hi ", " hi ", 0;\n\t"
#define RONK_TAIL_ADDFAM(lo, hi) \
  "mul.lo.u32 bw, m, m;\n\t" "add.cc.u32 " lo ", " lo ", bw;\n\t" "madc.lo.u32 " hi ", m, 1, " hi ";\n\t"
#if RONK_FMA_TAIL & 1
#define RONK_TAIL_SUB(lo, hi) RONK_TAIL_ADDFAM(lo, hi)
#else
#define RONK_TAIL_SUB(lo, hi) RONK_TAIL_SUBFAM(lo, hi)
#endif
#if RONK_FMA_TAIL & 2
#define RONK_TAIL_ADD(lo, hi) RONK_TAIL_ADDFAM(lo, hi)
#else
#define RONK_TAIL_ADD(lo, hi) RONK_TAIL_SUBFAM(lo, hi)
#endif
#if RONK_FMA_TAIL & (4 | 8)
#define RONK_TAIL_RED1(lo, hi) RONK_TAIL_ADDFAM(lo, hi)
#else
#define RONK_TAIL_RED1(lo, hi) RONK_TAIL_SUBFAM(lo, hi)
#endif
#if RONK_FMA_TAIL & (4 | 16)
#define RONK_TAIL_RED2(lo, hi) RONK_TAIL_ADDFAM(lo, hi)
#else
#define RONK_TAIL_RED2(lo, hi) RONK_TAIL_SUBFAM(lo, hi)
#endif
struct GoldilocksField {
  RONK_HD u64 modulus() const { return GL_P; }

#if defined(__CUDA_ARCH__)
  // ---- device path: explicit carry chains (inline PTX).  All values canonical in and out. ----
  // Canonical by construction — no compare/select anywhere:
  //   sub: a - b, borrow → +p (≡ -EPS mod 2^64); a, b < p ⇒ result in [0, p).
  //   add: a + b = a - (p - b); p - b ∈ [1, p] and sub(a, p) = a still holds (borrow path).
  static __device__ __forceinline__ u64 sub_words(u32 a0, u32 a1, u32 b0, u32 b1) {
    u32 d0, d1;
    asm("{\n\t.reg .u32 m, bw;\n\t"
        "sub.cc.u32 %0, %2, %4;\n\t"
        "subc.cc.u32 %1, %3, %5;\n\t"
        "subc.u32 m, 0, 0;\n\t"        // m = -borrow = EPS·borrow
        RONK_TAIL_SUB("%0", "%1") "}"
        : "=&r"(d0), "=&r"(d1)
        : "r"(a0), "r"(a1), "r"(b0), "r"(b1));
    return ((u64)d1 << 32) | d0;
  }
  __device__ __forceinline__ u64 sub(u64 a, u64 b) const {
    return sub_words((u32)a, (u32)(a >> 32), (u32)b, (u32)(b >> 32));
  }
  // a + b = a - (p - b) ≡ a + (b + EPS) (mod 2^64); that subtraction borrows exactly when this addition
  // does NOT carry (then +p, i.e. -EPS).  b + EPS < 2^64 because b < p.  Add-family carries only.
  __device__ __forceinline__ u64 add(u64 a, u64 b) const {
    u32 s0, s1;
    asm("{\n\t.reg .u32 t0, t1, m, bw;\n\t"
        "add.cc.u32 t0, %4, 0xFFFFFFFF;\n\t"
        "addc.u32 t1, %5, 0;\n\t"
        "add.cc.u32 %0, %2, t0;\n\t"
        "addc.cc.u32 %1, %3, t1;\n\t"
        "addc.u32 m, 0xFFFFFFFF, 0;\n\t"      // carry - 1: 0 or 0xFFFFFFFF (= EPS·borrow)
        RONK_TAIL_ADD("%0", "%1") "}"
        : "=&r"(s0), "=&r"(s1)
        : "r"((u32)a), "r"((u32)(a >> 32)), "r"((u32)b), "r"((u32)(b >> 32)));
    return ((u64)s1 << 32) | s0;
  }
  __device__ __forceinline__ u64 neg(u64 a) const { return a ? GL_P - a : 0; }

  // words r0 + r1·B + r2·B² + r3·B³ (B = 2^32; B² ≡ B-1, B³ ≡ -1) → canonical residue:
  //   Y = r2·EPS + r0 (one IMAD.WIDE, ≤ p-1), W = r1·B ≤ p-1, so
  //   x = (Y - r3) + W = sub(sub(Y, r3), p - W) with p - W = (~r1 : 1) — two canonical subs.
  // RONK_REDUCE_V2 (round 2): Y = r2·EPS + r0 is (r2 : r0) - r2 — one borrow chain (IADD3 + IMAD.X) instead
  // of the wide multiply, which ptxas had lowered to IMAD.MOV + IMAD.HI + IADD3 + IMAD.X and which, like
  // every IMAD.WIDE / IMAD.HI, holds the issue port for several cycles (tools/pipe_microbench2.cu measures it).
#ifndef RONK_REDUCE_V2
#define RONK_REDUCE_V2 1
#endif
  static __device__ __forceinline__ u64 reduce_words(u32 r0, u32 r1, u32 r2, u32 r3) {
    u32 z0, z1;
#if RONK_REDUCE_V2
    asm("{\n\t.reg .u32 m, bw;\n\t"
        "sub.cc.u32 %0, %2, %4;\n\t"        // (r2 : r0) - r2  =  r2·EPS + r0  (≥ 0: no borrow out of the pair)
        "subc.u32 %1, %4, 0;\n\t"
        "sub.cc.u32 %0, %0, %5;\n\t"        // t = Y - r3
        "subc.cc.u32 %1, %1, 0;\n\t"
        "subc.u32 m, 0, 0;\n\t"
        RONK_TAIL_RED1("%0", "%1")
        "add.cc.u32 %0, %0, 0xFFFFFFFF;\n\t" // t + (r1 : 0xFFFFFFFF)
        "addc.cc.u32 %1, %1, %3;\n\t"
        "addc.u32 m, 0xFFFFFFFF, 0;\n\t"     // carry - 1
        RONK_TAIL_RED2("%0", "%1") "}"
        : "=&r"(z0), "=&r"(z1)
        : "r"(r0), "r"(r1), "r"(r2), "r"(r3));
    return ((u64)z1 << 32) | z0;
#else
    // second step: t - (p - W) ≡ t + (r1 : 0xFFFFFFFF) (mod 2^64), and it borrows exactly when this
    // addition does NOT carry; m = carry - 1 is then the EPS mask of the "+p" correction.
    asm("{\n\t.reg .u64 y;\n\t.reg .u32 y0, y1, m, bw;\n\t"
        "mad.wide.u32 y, %4, 0xFFFFFFFF, %6;\n\t"
        "mov.b64 {y0, y1}, y;\n\t"
        "sub.cc.u32 %0, y0, %5;\n\t"        // t = Y - r3
        "subc.cc.u32 %1, y1, 0;\n\t"
        "subc.u32 m, 0, 0;\n\t"
        RONK_TAIL_RED1("%0", "%1")
        "add.cc.u32 %0, %0, 0xFFFFFFFF;\n\t" // t + (r1 : 0xFFFFFFFF)
        "addc.cc.u32 %1, %1, %3;\n\t"
        "addc.u32 m, 0xFFFFFFFF, 0;\n\t"     // carry - 1
        RONK_TAIL_RED2("%0", "%1") "}"
        : "=&r"(z0), "=&r"(z1)
        : "r"(r0), "r"(r1), "r"(r2), "r"(r3), "l"((u64)r0));
    return ((u64)z1 << 32) | z0;
#endif
  }
  // three-word form (r3 = 0): x = Y + W only
  static __device__ __forceinline__ u64 reduce_words3(u32 r0, u32 r1, u32 r2) {
    u32 z0, z1;
    asm("{\n\t.reg .u64 y;\n\t.reg .u32 y0, y1, m, bw;\n\t"
        "mad.wide.u32 y, %4, 0xFFFFFFFF, %5;\n\t"
        "mov.b64 {y0, y1}, y;\n\t"
        "add.cc.u32 %0, y0, 0xFFFFFFFF;\n\t"
        "addc.cc.u32 %1, y1, %3;\n\t"
        "addc.u32 m, 0xFFFFFFFF, 0;\n\t"
        RONK_TAIL_RED2("%0", "%1") "}"
        : "=&r"(z0), "=&r"(z1)
        : "r"(r0), "r"(r1), "r"(r2), "l"((u64)r0));
    return ((u64)z1 << 32) | z0;
  }
  __device__ __forceinline__ u64 reduce128(u64 lo, u64 hi) const {
    return reduce_words((u32)lo, (u32)(lo >> 32), (u32)hi, (u32)(hi >> 32));
  }
  __device__ __forceinline__ u64 mul(u64 a, u64 b) const {
    const u32 a0 = (u32)a, a1 = (u32)(a >> 32), b0 = (u32)b, b1 = (u32)(b >> 32);
    u32 r0, r1, r2, r3;
    asm("{\n\t.reg .u64 t, u, v, z;\n\t.reg .u32 t1, u0, u1, v1;\n\t"
        "mul.wide.u32 t, %4, %6;\n\t"            // a0·b0
        "mov.b64 {%0, t1}, t;\n\t"
        "cvt.u64.u32 u, t1;\n\t"
        "mad.wide.u32 u, %4, %7, u;\n\t"         // a0·b1 + t1        (no overflow)
        "mov.b64 {u0, u1}, u;\n\t"
        "cvt.u64.u32 v, u0;\n\t"
        "mad.wide.u32 v, %5, %6, v;\n\t"         // a1·b0 + u0        (no overflow)
        "mov.b64 {%1, v1}, v;\n\t"
        "cvt.u64.u32 z, u1;\n\t"
        "mad.wide.u32 z, %5, %7, z;\n\t"         // a1·b1 + u1
        "cvt.u64.u32 t, v1;\n\t"
        "add.u64 z, z, t;\n\t"                   // + v1               (< 2^64: product < 2^128)
        "mov.b64 {%2, %3}, z;\n\t}"
        : "=&r"(r0), "=&r"(r1), "=&r"(r2), "=&r"(r3)
        : "r"(a0), "r"(a1), "r"(b0), "r"(b1));
    return reduce_words(r0, r1, r2, r3);
  }
  // ---- a · 2^S for a compile-time S: three single-correction forms (round 2) ---------------------
  // Every form ends in ONE canonical add/sub (one EPS correction) and needs no wide multiply; the
  // round-1 form (shift to 96 bits, then the generic two-correction word reduction) is kept behind
  // RONK_SHIFT_V2=0 for A/B runs.  Derivations, with B = 2^32, B² ≡ B - 1, B³ ≡ -1 and
  // 2^-32 ≡ -EPS (mod p); each was checked exhaustively over S against big-integer arithmetic
  // (tools/shift_formulas.py) before it was written as PTX:
  //  A  0 < S < 32   x·2^S = y0 + y1·B + y2·B²,  y2 < 2^S:   ≡ (y1:y0) + y2·EPS.
  //                  (y2·EPS) + EPS = (y2 : ~y2), so the "a + (b + EPS), no carry → -EPS" add needs
  //                  just one NOT; the result is canonical even when (y1:y0) ≥ p because y2·EPS ≤ EPS².
  //  B  32 ≤ S < 64  x·2^S = (y0 + y1·B + y2·B²)·B ≡ (y0 + y1)·B - (y1 + y2); with y0 + y1 = S0 + c·B
  //                  this is ((S0 + c) : 0) - (y1 + y2 + c): both operands canonical → one sub.
  //  C  64 ≤ S < 96  k = 96 - S ∈ (0, 32]:  x·2^S = -x·2^-k,  x·2^-k = (x >> k) + v - v·B with
  //                  v = (x0 << (32-k)) mod B  →  x·2^S = sub((v : 0), (x >> k) + v).
  template <int S>
  static __device__ __forceinline__ u64 shl_a(u32 a0, u32 a1) {  // 0 < S < 32
    const u32 y0 = a0 << S, y1 = __funnelshift_l(a0, a1, S), y2 = a1 >> (32 - S);
    u32 r0, r1;
    asm("{\n\t.reg .u32 m, bw, n2;\n\t"
        "not.b32 n2, %4;\n\t"
        "add.cc.u32 %0, %2, n2;\n\t"
        "addc.cc.u32 %1, %3, %4;\n\t"
        "addc.u32 m, 0xFFFFFFFF, 0;\n\t"      // carry - 1: 0 or 0xFFFFFFFF (= EPS·[no carry])
        RONK_TAIL_ADD("%0", "%1") "}"
        : "=&r"(r0), "=&r"(r1)
        : "r"(y0), "r"(y1), "r"(y2));
    return ((u64)r1 << 32) | r0;
  }
  template <int SP>
  static __device__ __forceinline__ u64 shl_b(u32 a0, u32 a1) {  // S = 32 + SP, 0 ≤ SP < 32
    u32 y0, y1, y2;
    if constexpr (SP == 0) { y0 = a0; y1 = a1; y2 = 0u; }
    else { y0 = a0 << SP; y1 = __funnelshift_l(a0, a1, SP); y2 = a1 >> (32 - SP); }
    u32 r0, r1;
    asm("{\n\t.reg .u32 s0, hi, b0, b1, m, bw;\n\t"
        "add.cc.u32 s0, %2, %3;\n\t"          // y0 + y1 = s0 + c·B
        "addc.u32 hi, s0, 0;\n\t"             // s0 + c  (≤ 2^32 - 1)
        "addc.cc.u32 b0, %3, %4;\n\t"         // y1 + y2 + c
        "addc.u32 b1, 0, 0;\n\t"
        "sub.cc.u32 %0, 0, b0;\n\t"           // (hi : 0) - (b1 : b0)
        "subc.cc.u32 %1, hi, b1;\n\t"
        "subc.u32 m, 0, 0;\n\t"
        RONK_TAIL_SUB("%0", "%1") "}"
        : "=&r"(r0), "=&r"(r1)
        : "r"(y0), "r"(y1), "r"(y2));
    return ((u64)r1 << 32) | r0;
  }
  template <int K>
  static __device__ __forceinline__ u64 shl_c(u64 a) {  // S = 96 - K, 0 < K ≤ 32
    const u32 a0 = (u32)a;
    const u64 xh = a >> K;
    const u32 v = (K == 32) ? a0 : (a0 << (32 - K));
    u32 r0, r1;
    asm("{\n\t.reg .u32 t0, t1, m, bw;\n\t"
        "add.cc.u32 t0, %2, %4;\n\t"          // (x >> k) + v  < p, no carry out
        "addc.u32 t1, %3, 0;\n\t"
        "sub.cc.u32 %0, 0, t0;\n\t"           // (v : 0) - that
        "subc.cc.u32 %1, %4, t1;\n\t"
        "subc.u32 m, 0, 0;\n\t"
        RONK_TAIL_SUB("%0", "%1") "}"
        : "=&r"(r0), "=&r"(r1)
        : "r"((u32)xh), "r"((u32)(xh >> 32)), "r"(v));
    return ((u64)r1 << 32) | r0;
  }
#ifndef RONK_SHIFT_V2
#define RONK_SHIFT_V2 1
#endif
  // a · 2^S for a compile-time S in [0, 192), on 32-bit words (2^96 ≡ -1).
  template <int S>
  __device__ __forceinline__ u64 mul_pow2(u64 a) const {
    static_assert(S >= 0 && S < 192, "shift out of range");
    if constexpr (S == 0) {
      return a;
    } else if constexpr (S >= 96) {
      return neg(mul_pow2<S - 96>(a));
    } else if constexpr (RONK_SHIFT_V2 != 0) {
      if constexpr (S < 32) return shl_a<S>((u32)a, (u32)(a >> 32));
      else if constexpr (S < 64) return shl_b<S - 32>((u32)a, (u32)(a >> 32));
      else return shl_c<96 - S>(a);
    } else {
      const u32 a0 = (u32)a, a1 = (u32)(a >> 32);
      constexpr int s = S % 32;
      // (y2:y1:y0) = a << s (96 bits).  Written as a·2^s; ptxas turns the literal multiplier back into
      // SHF/IMAD.SHL.  Keeping it opaque (constant memory) forces two half-rate IMAD.WIDE instead, which
      // was slower.
      u32 y0, y1, y2;
      if constexpr (s == 0) {
        y0 = a0; y1 = a1; y2 = 0u;
      } else {
        const u64 lo = (u64)a0 * (u64)(1u << s);
        const u64 hi = (u64)a1 * (u64)(1u << s) + (lo >> 32);   // no overflow: < 2^(32+s)
        y0 = (u32)lo; y1 = (u32)hi; y2 = (u32)(hi >> 32);
      }
      if constexpr (S < 32) return reduce_words3(y0, y1, y2);
      else if constexpr (S < 64) return reduce_words(0u, y0, y1, y2);
      else {
        // y·B² = y0·B² + y1·B³ + y2·B⁴ ≡ y0·EPS - (y2:y1);  y0·EPS < p and (y2:y1) < 2^63 < p
        const u64 yy = (u64)y0 * 0xFFFFFFFFull;
        return sub(yy, ((u64)y2 << 32) | y1);
      }
    }
  }
#else
  // ---- host path (tests/emu only): portable C with identical results ----
  RONK_DEV u64 add(u64 a, u64 b) const {
    u64 s = a + b;
    u64 t = s + GL_EPS;
    return (s < a || t < s) ? t : s;
  }
  RONK_DEV u64 sub(u64 a, u64 b) const {
    u64 d = a - b;
    return (a < b) ? d - GL_EPS : d;
  }
  RONK_DEV u64 neg(u64 a) const { return a ? GL_P - a : 0; }
  RONK_DEV u64 reduce128(u64 lo, u64 hi) const {
    u64 hh = hi >> 32, hl = hi & 0xFFFFFFFFULL;
    u64 t0 = lo - hh;
    if (lo < hh) t0 -= GL_EPS;
    u64 t1 = (hl << 32) - hl;
    u64 r = t0 + t1;
    if (r < t1) r += GL_EPS;
    return (r >= GL_P) ? r - GL_P : r;
  }
  RONK_DEV u64 mul(u64 a, u64 b) const { return reduce128(a * b, mulhi64(a, b)); }
  template <int S>
  RONK_DEV u64 mul_pow2(u64 a) const {
    static_assert(S >= 0 && S < 192, "shift out of range");
    if constexpr (S == 0) {
      return a;
    } else if constexpr (S >= 96) {
      return neg(mul_pow2<S - 96>(a));
    } else if constexpr (S < 64) {
      return reduce128(a << S, a >> (64 - S));
    } else {
      return mul_pow2<S - 32>(mul_pow2<32>(a));
    }
  }
#endif
  RONK_DEV u64 mul_tw(u64 a, u64 w) const { return mul(a, w); }
  RONK_DEV u64 to_tw(u64 w) const { return w; }

  // a · ω16^E (forward) or a · ω16^-E (INV), E in [0,8).  ω16 = g^((p-1)/16) = 2^156 for g = 7.
  template <int E, bool INV>
  RONK_DEV u64 w16(u64 a) const {
    constexpr int fwd = (156 * E) % 192;
    constexpr int sh = INV ? (192 - fwd) % 192 : fwd;
    return mul_pow2<sh>(a);
  }
  // (a - b) · ω16^±E: a shift of 96+s is -2^s, so the sign is folded into the subtraction for free.
  template <int E, bool INV>
  RONK_DEV u64 w16_sub(u64 a, u64 b) const {
    constexpr int fwd = (156 * E) % 192;
    constexpr int sh = INV ? (192 - fwd) % 192 : fwd;
    if constexpr (sh >= 96) return mul_pow2<sh - 96>(sub(b, a));
    else return mul_pow2<sh>(sub(a, b));
  }
};

// ------------------------------------------------------------------------------------------
// Generic odd modulus < 2^64, Montgomery multiplication with R = 2^64.
// ------------------------------------------------------------------------------------------
struct MontField {
  u64 p;        // modulus (odd)
  u64 pinv;     // p^-1 mod 2^64
  u64 r2;       // 2^128 mod p
  u64 w16t[8];  // ω16^e (direction already applied) in Montgomery form; unused entries = R mod p

  RONK_HD u64 modulus() const { return p; }

  RONK_DEV u64 add(u64 a, u64 b) const {
    u64 s = a + b;
    return (s < a || s >= p) ? s - p : s;
  }
  RONK_DEV u64 sub(u64 a, u64 b) const {
    u64 d = a - b;
    return (a < b) ? d + p : d;
  }
  RONK_DEV u64 neg(u64 a) const { return a ? p - a : 0; }
  // REDC(a·b) = a·b·2^-64 mod p, subtractive form (no 129-bit intermediate for p > 2^63).
  RONK_DEV u64 redc_mul(u64 a, u64 b) const {
    u64 lo = a * b, hi = mulhi64(a, b);
    u64 m = lo * pinv;
    u64 mp = mulhi64(m, p);
    u64 t = hi - mp;
    return (hi < mp) ? t + p : t;
  }
  RONK_DEV u64 mul_tw(u64 a, u64 w_mont) const { return redc_mul(a, w_mont); }
  RONK_DEV u64 mul(u64 a, u64 b) const { return redc_mul(redc_mul(a, b), r2); }
  RONK_DEV u64 to_tw(u64 w) const { return redc_mul(w, r2); }
  template <int E, bool INV>
  RONK_DEV u64 w16(u64 a) const {
    if constexpr (E == 0) return a;
    return redc_mul(a, w16t[E]);
  }
  template <int E, bool INV>
  RONK_DEV u64 w16_sub(u64 a, u64 b) const {
    return w16<E, INV>(sub(a, b));
  }
};

// a^e by square-and-multiply (value of Field::pow, prime/mod.rs:74-84).
template <class F>
RONK_DEV u64 field_pow(const F& f, u64 a, u64 e) {
  u64 r = 1 % f.modulus();
  u64 base = a;
  while (e) {
    if (e & 1) r = f.mul(r, base);
    base = f.mul(base, base);
    e >>= 1;
  }
  return r;
}

// ------------------------------------------------------------------------------------------
// Host-side scalar helpers (plan building only: roots of unity, Montgomery constants).
// ------------------------------------------------------------------------------------------
inline u64 h_mulmod(u64 a, u64 b, u64 p) { return (u64)(((unsigned __int128)a * b) % p); }
inline u64 h_powmod(u64 a, u64 e, u64 p) {
  u64 r = 1 % p;
  a %= p;
  while (e) {
    if (e & 1) r = h_mulmod(r, a, p);
    a = h_mulmod(a, a, p);
    e >>= 1;
  }
  return r;
}
inline u64 h_inv64(u64 p) {  // p^-1 mod 2^64 (p odd), Newton
  u64 x = p;
  for (int i = 0; i < 6; i++) x *= 2 - p * x;
  return x;
}
// The Montgomery policy of an odd modulus p without roots of unity: every w16t entry is R mod p (the identity).
inline MontField h_mont_field(u64 p) {
  MontField f;
  f.p = p;
  f.pinv = h_inv64(p);
  const u64 r1 = (u64)((((unsigned __int128)1) << 64) % p);
  f.r2 = h_mulmod(r1, r1, p);
  for (int e = 0; e < 8; e++) f.w16t[e] = r1;
  return f;
}

}  // namespace ronk
