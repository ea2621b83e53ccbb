// msm_curve.cuh — GF(101²) and AffinePoint<PlutoExtendedCurve> arithmetic shared by the MSM kernels and the
// element-wise point kernels of msm.cu.  Host-compilable (RONK_DEV), so tests/emu can run it on the CPU tier.
// Mirrors src/algebra/field/extension/gf_101_2.rs (inverse :35-47, Mul :86-100) and src/curve/mod.rs
// (Add :178-213, Neg :225-235, is_on_curve :130-139); curve y² = x³ + 3 (src/curve/pluto_curve.rs:40-51).
#pragma once
#include "field.cuh"

namespace ronk {

constexpr u32 Q101 = 101;
constexpr u32 PT_INF = 0xFFFFFFFFu;

struct Gf { u32 c0, c1; };
struct Pt { Gf x, y; bool inf; };

RONK_DEV u32 fq_mul(u32 a, u32 b) { return (a * b) % Q101; }
RONK_DEV u32 fq_add(u32 a, u32 b) { u32 s = a + b; return s >= Q101 ? s - Q101 : s; }
RONK_DEV u32 fq_sub(u32 a, u32 b) { return a >= b ? a - b : a + Q101 - b; }
RONK_DEV u32 fq_neg(u32 a) { return a ? Q101 - a : 0; }
// a^99 = a^-1 (Fermat; prime/mod.rs:62-72).  99 = 0b1100011.
RONK_DEV u32 fq_inv(u32 a) {
  const u32 a2 = fq_mul(a, a), a3 = fq_mul(a2, a);
  const u32 a6 = fq_mul(a3, a3), a12 = fq_mul(a6, a6), a24 = fq_mul(a12, a12);
  const u32 a48 = fq_mul(a24, a24), a96 = fq_mul(a48, a48);
  return fq_mul(a96, a3);
}

RONK_DEV Gf gf_add(Gf a, Gf b) { return {fq_add(a.c0, b.c0), fq_add(a.c1, b.c1)}; }
RONK_DEV Gf gf_sub(Gf a, Gf b) { return {fq_sub(a.c0, b.c0), fq_sub(a.c1, b.c1)}; }
RONK_DEV Gf gf_neg(Gf a) { return {fq_neg(a.c0), fq_neg(a.c1)}; }
RONK_DEV bool gf_eq(Gf a, Gf b) { return a.c0 == b.c0 && a.c1 == b.c1; }
// (a0 + a1 t)(b0 + b1 t) mod (t² + 2) = (a0b0 - 2a1b1) + (a0b1 + a1b0) t
RONK_DEV Gf gf_mul(Gf a, Gf b) {
  return {(a.c0 * b.c0 + 99u * (a.c1 * b.c1 % Q101)) % Q101, (a.c0 * b.c1 + a.c1 * b.c0) % Q101};
}
// conj / norm, norm = a0² + 2a1²  (gf_101_2.rs:35-47); caller guarantees a != 0
RONK_DEV Gf gf_inv(Gf a) {
  const u32 s = fq_inv((a.c0 * a.c0 + 2u * a.c1 * a.c1) % Q101);
  return {fq_mul(a.c0, s), fq_mul(fq_neg(a.c1), s)};
}

// norm inverse from a table tab[a] = a^-1 mod 101 (a in 1..100)
RONK_DEV Gf gf_inv_tab(Gf a, const uint8_t* tab) {
  const u32 s = tab[(a.c0 * a.c0 + 2u * a.c1 * a.c1) % Q101];
  return {fq_mul(a.c0, s), fq_mul(fq_neg(a.c1), s)};
}

RONK_DEV Pt pt_unpack(u32 w) {
  Pt p;
  p.inf = (w == PT_INF);
  p.x = {w & 0xFF, (w >> 8) & 0xFF};
  p.y = {(w >> 16) & 0xFF, w >> 24};
  return p;
}
RONK_DEV u32 pt_pack(const Pt& p) {
  return p.inf ? PT_INF : (p.x.c0 | (p.x.c1 << 8) | (p.y.c0 << 16) | (p.y.c1 << 24));
}
// Well-formed (canonical coordinates) and on y² = x³ + 3  (curve/mod.rs:130-139).
RONK_DEV bool pt_valid(u32 w) {
  if (w == PT_INF) return true;
  const Pt p = pt_unpack(w);
  if (p.x.c0 >= Q101 || p.x.c1 >= Q101 || p.y.c0 >= Q101 || p.y.c1 >= Q101) return false;
  const Gf lhs = gf_mul(p.y, p.y);
  const Gf rhs = gf_add(gf_mul(gf_mul(p.x, p.x), p.x), Gf{3, 0});
  return gf_eq(lhs, rhs);
}
// AffinePoint + AffinePoint  (curve/mod.rs:178-213), same case order as the reference.
RONK_DEV Pt pt_add(const Pt& a, const Pt& b) {
  if (a.inf) return b;
  if (b.inf) return a;
  const bool same_x = gf_eq(a.x, b.x);
  if (same_x && gf_eq(a.y, gf_neg(b.y))) { Pt r; r.inf = true; r.x = {0, 0}; r.y = {0, 0}; return r; }
  Gf num, den;
  if (same_x && gf_eq(a.y, b.y)) {  // tangent: 3x² / 2y   (a = 0)
    num = gf_mul(Gf{3, 0}, gf_mul(a.x, a.x));
    den = gf_add(a.y, a.y);
  } else {                          // chord: (y2 - y1) / (x2 - x1)
    num = gf_sub(b.y, a.y);
    den = gf_sub(b.x, a.x);
  }
  const Gf lam = gf_mul(num, gf_inv(den));
  Pt r;
  r.inf = false;
  r.x = gf_sub(gf_sub(gf_mul(lam, lam), a.x), b.x);
  r.y = gf_sub(gf_mul(lam, gf_sub(a.x, r.x)), a.y);
  return r;
}
RONK_DEV u32 pt_add_w(u32 a, u32 b) { return pt_pack(pt_add(pt_unpack(a), pt_unpack(b))); }

// Same addition law with the table inverse (MSM kernels).
RONK_DEV u32 pt_add_t(u32 wa, u32 wb, const uint8_t* tab) {
  if (wa == PT_INF) return wb;
  if (wb == PT_INF) return wa;
  const Pt a = pt_unpack(wa), b = pt_unpack(wb);
  const bool same_x = gf_eq(a.x, b.x);
  if (same_x && gf_eq(a.y, gf_neg(b.y))) return PT_INF;
  Gf num, den;
  if (same_x && gf_eq(a.y, b.y)) {
    num = gf_mul(Gf{3, 0}, gf_mul(a.x, a.x));
    den = gf_add(a.y, a.y);
  } else {
    num = gf_sub(b.y, a.y);
    den = gf_sub(b.x, a.x);
  }
  const Gf lam = gf_mul(num, gf_inv_tab(den, tab));
  Pt r;
  r.inf = false;
  r.x = gf_sub(gf_sub(gf_mul(lam, lam), a.x), b.x);
  r.y = gf_sub(gf_mul(lam, gf_sub(a.x, r.x)), a.y);
  return pt_pack(r);
}
RONK_DEV void build_inv_table(uint8_t* tab, u32 tid, u32 nthr) {
  for (u32 a = tid; a < Q101; a += nthr) tab[a] = (uint8_t)(a ? fq_inv(a) : 0);
}

// ---- point bins (shared by the histogram and the group-coordinate commit kernels) ----
//   bin(P) = 2·(x0 + 101·x1) + ybit(y),  ybit(y) = y0 ? (y0 > 50) : (y1 > 50)   (y and -y get different bits)
constexpr u32 MSM_XS = Q101 * Q101;   // 10201 x values
constexpr u32 MSM_BINS = 2 * MSM_XS;  // 20402
constexpr u32 MSM_EXP = 102;          // group exponent of E(F_101²) ≅ (Z/102)²
RONK_DEV u32 y_bit(u32 y0, u32 y1) { return y0 ? (y0 > 50u) : (y1 > 50u); }
RONK_DEV u32 pt_bin(u32 w) { return 2u * ((w & 0xFF) + Q101 * ((w >> 8) & 0xFF)) + y_bit((w >> 16) & 0xFF, w >> 24); }

// The term test of the group-coordinate commit: whether the packed point w is canonical and on y² = x³ + 3
// (curve/mod.rs:130-139), with e = its bintab entry (y0 | y1 << 8 | a << 16 | b << 24; 0xFFFFFFFF when w is not
// canonical).  Every coordinate < 101  ⟺  no byte of w or of w + 27·0x01010101 has bit 7 set (bytes < 128 cannot carry
// into their neighbour); Infinity (0xFFFFFFFF) is not canonical and is reported as not on the curve.
RONK_DEV bool coord_term(u32 w, const u32* tab, u32& e) {
  const bool canon = ((w | (w + 0x1B1B1B1Bu)) & 0x80808080u) == 0u;
  e = canon ? tab[pt_bin(w)] : 0xFFFFFFFFu;
  return canon && (e & 0xFFFFu) == (w >> 16);   // empty bins hold 0xFFFF in the y field
}
// Nonzero iff some byte of the four packed scalars s4 is ≥ 17, i.e. not an F17 residue: a byte < 17 stays below 128 after
// adding 111, and a byte ≥ 128 flags itself (its carry can only reach bytes above it, which the word is already flagged by).
RONK_DEV u32 scalar4_over(u32 s4) { return (s4 | (s4 + 0x6F6F6F6Fu)) & 0x80808080u; }

// ---- group coordinates (host only; plan building for msm_coord_kernel, also compiled by tests/emu) ----
// E(F_101²): y² = x³ + 3 has 102² points and exponent 102, i.e. E ≅ (Z/102)².  With a basis (G1, G2) every point is
// a·G1 + b·G2 for exactly one (a, b) ∈ (Z/102)², and Σ s_i·P_i = (Σ s_i a_i)·G1 + (Σ s_i b_i)·G2: the whole commit is two
// integer dot products mod 102 plus ONE table lookup — the same group element the reference's chain of affine
// additions (curve/mod.rs:178-213) arrives at, because the addition law is associative and commutative.
//   bintab[bin(P)] = y0 | y1 << 8 | a << 16 | b << 24   (0xFFFFFFFF: no curve point in the bin — doubles as is_on_curve)
//   pttab[102 a + b] = packed a·G1 + b·G2                (PT_INF at 0)
// On the device the bintab is padded to kTabWords (a multiple of four words), with pttab after it (ctx->msm_coord).
// The basis is found by search, deterministically (first points in x order that work), with the reference's own
// addition law; injectivity of (a, b) → point is CHECKED while the table is filled, so a wrong basis cannot survive.
// Returns false if no basis was found (cannot happen for this curve; the caller reports an internal error).
constexpr u32 kTabWords = (MSM_BINS + 3) / 4 * 4;
inline bool build_group_tables(u32* bintab /*MSM_BINS*/, u32* pttab /*MSM_EXP²*/) {
  // curve points in x order: sq[idx(y²)] = y
  static const u32 kNone = 0xFFFFFFFFu;
  u32* sq = new u32[MSM_XS];
  for (u32 i = 0; i < MSM_XS; i++) sq[i] = kNone;
  for (u32 i = 0; i < MSM_XS; i++) {
    const Gf y = {i % Q101, i / Q101};
    const Gf y2 = gf_mul(y, y);
    u32& slot = sq[y2.c0 + Q101 * y2.c1];
    if (slot == kNone) slot = i;  // the smaller of the two roots (deterministic)
  }
  u32* cand = new u32[2 * MSM_XS];
  u32 ncand = 0;
  for (u32 i = 0; i < MSM_XS; i++) {
    const Gf x = {i % Q101, i / Q101};
    const Gf rhs = gf_add(gf_mul(gf_mul(x, x), x), Gf{3, 0});
    const u32 r = sq[rhs.c0 + Q101 * rhs.c1];
    if (r == kNone) continue;
    Pt p;
    p.inf = false;
    p.x = x;
    p.y = {r % Q101, r / Q101};
    cand[ncand++] = pt_pack(p);
    const Gf ny = gf_neg(p.y);
    if (!gf_eq(ny, p.y)) { p.y = ny; cand[ncand++] = pt_pack(p); }
  }
  delete[] sq;
  auto order_is_102 = [](u32 w) {
    u32 acc = w;
    for (u32 k = 1; k < MSM_EXP; k++) {  // acc = k·w
      if (acc == PT_INF) return false;
      acc = pt_add_w(acc, w);
    }
    return acc == PT_INF;  // 102·w = O and no smaller multiple was
  };
  bool ok = false;
  if (ncand == MSM_EXP * MSM_EXP - 1) {
    u32 g1 = PT_INF;
    u32 i1 = 0;
    for (; i1 < ncand; i1++)
      if (order_is_102(cand[i1])) { g1 = cand[i1]; break; }
    for (u32 i2 = i1 + 1; g1 != PT_INF && i2 < ncand && !ok; i2++) {
      const u32 g2 = cand[i2];
      if (!order_is_102(g2)) continue;
      for (u32 i = 0; i < MSM_BINS; i++) bintab[i] = kNone;
      bool inj = true, seen_inf = false;
      u32 row = PT_INF;  // a·G1
      for (u32 a = 0; a < MSM_EXP && inj; a++) {
        u32 cur = row;   // a·G1 + b·G2
        for (u32 b = 0; b < MSM_EXP; b++) {
          if (cur == PT_INF) {
            if (seen_inf) { inj = false; break; }
            seen_inf = true;
          } else {
            u32& e = bintab[pt_bin(cur)];
            if (e != kNone) { inj = false; break; }
            e = (cur >> 16) | (a << 16) | (b << 24);
          }
          pttab[MSM_EXP * a + b] = cur;
          cur = pt_add_w(cur, g2);
        }
        row = pt_add_w(row, g1);
      }
      ok = inj;
    }
  }
  delete[] cand;
  return ok;
}

}  // namespace ronk
