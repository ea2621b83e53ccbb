// pairing.cuh — the reference's Tate pairing on E(F_101²)[17] (src/curve/pairing.rs:33-198), literally: the Miller loop
// with its zero-skipping and `zeros` counter, the `z + p == Infinity` branch and the final exponentiation, on
// msm_curve.cuh's GF(101²) and affine-point arithmetic.  Host-compilable (RONK_DEV), so tests/emu can run it on the CPU.
//
// The literal values are not bilinear (e(P, A + B) ≠ e(P, A)·e(P, B) for some triples), so pairing.cu tabulates the
// loop itself on every pair of E[17] rather than deriving the table from a basis.
#pragma once
#include "msm_curve.cuh"

namespace ronk {

constexpr u32 PAIR_R = 17;                             // pairing::<PlutoExtendedCurve, 17>
constexpr u32 PAIR_FINAL_EXP = (Q101 * Q101 - 1) / PAIR_R;  // 600: the result lies in μ17
constexpr u32 E17_STEP = MSM_EXP / PAIR_R;             // 6: a·G1 + b·G2 is 17-torsion iff 6 | a and 6 | b
constexpr u32 E17_PTS = PAIR_R * PAIR_R;               // 289 points of E[17], Infinity included
constexpr u32 PAIR_TAB = E17_PTS * E17_PTS;            // 83 521 pairs
constexpr uint8_t PAIR_PANIC = 0xFF;                   // table sentinel: the reference panics on this pair

RONK_DEV bool gf_is_zero(Gf a) { return a.c0 == 0 && a.c1 == 0; }
RONK_DEV Gf gf_pow(Gf a, u32 e) {
  Gf r = {1, 0};
  for (; e; e >>= 1) {
    if (e & 1u) r = gf_mul(r, a);
    a = gf_mul(a, a);
  }
  return r;
}
RONK_DEV Pt pt_neg(Pt a) {  // curve/mod.rs:225-235
  if (!a.inf) a.y = gf_neg(a.y);
  return a;
}

// line_function (pairing.rs:130-164): false where the reference panics (an argument is Infinity, or the tangent's 2y is 0).
RONK_DEV bool line_function(const Pt& a, const Pt& b, const Pt& in, Gf& out) {
  if (a.inf || b.inf || in.inf) return false;
  Gf m;
  if (!gf_eq(a.x, b.x)) {
    m = gf_mul(gf_sub(b.y, a.y), gf_inv(gf_sub(b.x, a.x)));
  } else if (gf_eq(a.y, b.y)) {
    const Gf den = gf_add(a.y, a.y);
    if (gf_is_zero(den)) return false;  // "invalid inverse"
    m = gf_mul(gf_mul(Gf{3, 0}, gf_mul(a.x, a.x)), gf_inv(den));  // EQUATION_A = 0
  } else {
    out = gf_sub(in.x, a.x);
    return true;
  }
  out = gf_sub(gf_add(gf_mul(m, gf_sub(in.x, a.x)), a.y), in.y);
  return true;
}
// vertical_line (:179-181) and tangent_line (:196-198)
RONK_DEV bool vertical_line(const Pt& a, const Pt& in, Gf& out) { return line_function(a, pt_neg(a), in, out); }
RONK_DEV bool tangent_line(const Pt& a, const Pt& in, Gf& out) { return line_function(a, a, in, out); }

// miller_loop::<_, 17> (pairing.rs:58-115): false where the reference panics, including `assert_eq!(zeros, 0)`.
RONK_DEV bool miller_loop(const Pt& p, const Pt& q, Gf& x) {
  x = Gf{1, 0};
  Pt z = p;
  int zeros = 0;
  for (int bit = 3; bit >= 0; bit--) {  // the bits of 17 = 0b10001 after the leading one
    const Pt z2 = pt_add(z, z);         // 2 * z
    Gf tangent, vertical;
    if (!tangent_line(z, q, tangent) || !vertical_line(z2, q, vertical)) return false;
    x = gf_mul(x, x);
    if (gf_is_zero(tangent)) zeros++;
    else x = gf_mul(x, tangent);
    if (gf_is_zero(vertical)) zeros--;
    else x = gf_mul(x, gf_inv(vertical));
    z = z2;
    if ((PAIR_R >> bit) & 1u) {
      Gf line;
      if (!line_function(z, p, q, line)) return false;
      const Pt zp = pt_add(z, p);
      if (zp.inf) {
        if (gf_is_zero(line)) zeros++;
        else x = gf_mul(x, line);
      } else {
        Gf v;
        if (!vertical_line(zp, q, v)) return false;
        if (gf_is_zero(line)) zeros++;
        else x = gf_mul(x, line);
        if (gf_is_zero(v)) zeros--;
        else x = gf_mul(x, gf_inv(v));
      }
      z = zp;
    }
  }
  return zeros == 0;
}

// pairing::<_, 17> (pairing.rs:33-54) for p, q in E[17]; the torsion asserts are the callers' (in group coordinates).
RONK_DEV bool tate_pairing(const Pt& p, const Pt& q, Gf& out) {
  Gf x;
  if (!miller_loop(p, q, x)) return false;
  out = gf_pow(x, PAIR_FINAL_EXP);
  return true;
}

// Index of a point of E[17] in the pairing table: 17·(a/6) + b/6 for P = a·G1 + b·G2 (Infinity is 0).
RONK_DEV u32 e17_index(u32 a, u32 b) { return PAIR_R * (a / E17_STEP) + b / E17_STEP; }

// One table entry: the index in mu (the 17 elements of μ17 in (c0, c1) order, c0 | c1 << 8) of the pairing of the
// E[17] points with indices ip and iq, or PAIR_PANIC where the reference panics.  pttab is build_group_tables' point table.
RONK_DEV uint8_t pairing_entry(u32 ip, u32 iq, const u32* pttab, const uint16_t* mu) {
  const u32 wp = pttab[MSM_EXP * (E17_STEP * (ip / PAIR_R)) + E17_STEP * (ip % PAIR_R)];
  const u32 wq = pttab[MSM_EXP * (E17_STEP * (iq / PAIR_R)) + E17_STEP * (iq % PAIR_R)];
  Gf v;
  if (!tate_pairing(pt_unpack(wp), pt_unpack(wq), v)) return PAIR_PANIC;
  const u32 key = v.c0 | (v.c1 << 8);
  for (u32 k = 0; k < PAIR_R; k++)
    if (mu[k] == key) return (uint8_t)k;
  return PAIR_PANIC;  // not in μ17: cannot happen (x^600 has order dividing 17); the tests check where the sentinels sit
}

// Group coordinates (a, b) of a packed point from bintab (build_group_tables): false for an off-curve or non-canonical
// word.  Infinity is (0, 0).
RONK_DEV bool point_coords(u32 w, const u32* bintab, u32& a, u32& b) {
  u32 e;
  const bool on = coord_term(w, bintab, e);
  a = on ? (e >> 16) & 0xFFu : 0u;
  b = on ? e >> 24 : 0u;
  return on || w == PT_INF;
}
// P − s·Q in group coordinates, one coordinate: (p − s·q) mod 102 for p, q < 102 and s < 17 (s·q ≤ 1616 < 17·102).
// Mul<ScalarField> is repeated addition with 0 giving Infinity (curve/mod.rs:157-172): the same group element.
RONK_DEV u32 coord_sub_smul(u32 p, u32 s, u32 q) { return (p + PAIR_R * MSM_EXP - s * q) % MSM_EXP; }
// Whether (a, b) is a finite point of E[17], the points the reference's pairing accepts (pairing.rs:37-47, and
// line_function panics on Infinity).
RONK_DEV bool e17_finite(u32 a, u32 b) { return a % E17_STEP == 0 && b % E17_STEP == 0 && (a | b) != 0; }

// PlutoExtendedCurve::GENERATOR = (36, 31t) (pluto_curve.rs:46-49), packed
constexpr u32 PLUTO_EXT_GEN = 36u | (31u << 24);

// The 17 elements x of GF(101²) with x^17 = 1, in (c0, c1) order, as c0 | c1 << 8.
inline void mu17_list(uint16_t* mu) {
  u32 k = 0;
  for (u32 c0 = 0; c0 < Q101; c0++)
    for (u32 c1 = 0; c1 < Q101; c1++) {
      const Gf x = {c0, c1};
      if (gf_eq(gf_pow(x, PAIR_R), Gf{1, 0}) && k < PAIR_R) mu[k++] = (uint16_t)(c0 | (c1 << 8));
    }
}

// kzg::check of one row (kzg/setup.rs:81-103) in group coordinates: 1 when lhs == rhs.  Raises `bad` where the reference
// panics or the ABI rejects the input; g1 = g1_srs[0], g2 = g2_srs[1], gen_idx = e17_index(GEN); T is the pairing table.
RONK_DEV uint8_t kzg_check_row(u32 wc, u32 wq, u32 z, u32 v, u32 g1a, u32 g1b, u32 g2a, u32 g2b, u32 gena, u32 genb,
                          u32 gen_idx, const u32* bintab, const uint8_t* T, u32& bad) {
  u32 ca, cb, qa, qb;
  bad |= (u32)!point_coords(wc, bintab, ca, cb) | (u32)!point_coords(wq, bintab, qa, qb) | (u32)(z >= PAIR_R) | (u32)(v >= PAIR_R);
  const u32 ba = coord_sub_smul(g2a, z, gena), bb = coord_sub_smul(g2b, z, genb);  // g2 − GEN·point
  const u32 ra = coord_sub_smul(ca, v, g1a), rb = coord_sub_smul(cb, v, g1b);      // p − g1·value
  bad |= (u32)!e17_finite(qa, qb) | (u32)!e17_finite(ba, bb) | (u32)!e17_finite(ra, rb);
  const u32 lhs = T[E17_PTS * e17_index(qa, qb) + e17_index(ba, bb)];
  const u32 rhs = T[E17_PTS * e17_index(ra, rb) + gen_idx];
  bad |= (u32)(lhs == PAIR_PANIC) | (u32)(rhs == PAIR_PANIC);
  return lhs == rhs ? 1 : 0;
}

}  // namespace ronk
