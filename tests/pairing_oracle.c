/* pairing_oracle.c — TEST INFRASTRUCTURE: the reference's Tate pairing (src/curve/pairing.rs:33-198) and kzg::check
 * (src/kzg/setup.rs:81-103), restated in C from the reference's algorithm on their own GF(101²) and affine-point
 * arithmetic (gf_101_2.rs, curve/mod.rs), independent of the library's kernels and tables.  Each function returns 1
 * where the reference panics.  Loaded by tests/pairing_oracle.py; never linked into libronk_b200.so. */
#include <stddef.h>
#include <stdint.h>

typedef struct { int c0, c1; } gf;
typedef struct { int inf; gf x, y; } pt;

static int md(int a) { a %= 101; return a < 0 ? a + 101 : a; }
static gf g_add(gf a, gf b) { gf r = {md(a.c0 + b.c0), md(a.c1 + b.c1)}; return r; }
static gf g_sub(gf a, gf b) { gf r = {md(a.c0 - b.c0), md(a.c1 - b.c1)}; return r; }
static gf g_neg(gf a) { gf r = {md(-a.c0), md(-a.c1)}; return r; }
static gf g_mul(gf a, gf b) { gf r = {md(a.c0 * b.c0 - 2 * a.c1 * b.c1), md(a.c0 * b.c1 + a.c1 * b.c0)}; return r; }  /* t² = −2 */
static int g_eq(gf a, gf b) { return a.c0 == b.c0 && a.c1 == b.c1; }
static int g_zero(gf a) { return a.c0 == 0 && a.c1 == 0; }
static int f_pow(int a, int e) { int r = 1; a = md(a); while (e) { if (e & 1) r = r * a % 101; a = a * a % 101; e >>= 1; } return r; }
/* inverse (gf_101_2.rs:35-47): conjugate over the norm; 0 has none ("invalid inverse") */
static int g_inv(gf a, gf *out) {
  if (g_zero(a)) return 1;
  const int s = f_pow(md(a.c0 * a.c0 + 2 * a.c1 * a.c1), 99);
  out->c0 = md(a.c0 * s);
  out->c1 = md(-a.c1 * s);
  return 0;
}
static int g_div(gf a, gf b, gf *out) { gf i; if (g_inv(b, &i)) return 1; *out = g_mul(a, i); return 0; }
static gf g_pow(gf a, unsigned e) { gf r = {1, 0}; for (unsigned k = 0; k < e; k++) r = g_mul(r, a); return r; }  /* literal */

static pt p_inf(void) { pt r = {1, {0, 0}, {0, 0}}; return r; }
static pt p_unpack(const uint8_t *w) {
  pt r;
  r.inf = w[0] == 0xFF && w[1] == 0xFF && w[2] == 0xFF && w[3] == 0xFF;
  r.x.c0 = w[0]; r.x.c1 = w[1]; r.y.c0 = w[2]; r.y.c1 = w[3];
  return r;
}
static int p_eq(pt a, pt b) { return a.inf || b.inf ? a.inf == b.inf : g_eq(a.x, b.x) && g_eq(a.y, b.y); }
/* canonical and on y² = x³ + 3 (curve/mod.rs:130-139; AffinePoint::new asserts it) */
static int p_valid(const uint8_t *w) {
  pt p = p_unpack(w);
  if (p.inf) return 1;
  if (w[0] > 100 || w[1] > 100 || w[2] > 100 || w[3] > 100) return 0;
  gf three = {3, 0};
  return g_eq(g_mul(p.y, p.y), g_add(g_mul(g_mul(p.x, p.x), p.x), three));
}
static pt p_neg(pt a) { if (!a.inf) a.y = g_neg(a.y); return a; }
/* Add (curve/mod.rs:178-213) */
static int p_add(pt a, pt b, pt *out) {
  if (a.inf) { *out = b; return 0; }
  if (b.inf) { *out = a; return 0; }
  if (g_eq(a.x, b.x) && g_eq(a.y, g_neg(b.y))) { *out = p_inf(); return 0; }
  gf lam;
  if (g_eq(a.x, b.x) && g_eq(a.y, b.y)) {
    gf three = {3, 0};
    if (g_div(g_mul(three, g_mul(a.x, a.x)), g_add(a.y, a.y), &lam)) return 1;
  } else if (g_div(g_sub(b.y, a.y), g_sub(b.x, a.x), &lam)) {
    return 1;
  }
  pt r;
  r.inf = 0;
  r.x = g_sub(g_sub(g_mul(lam, lam), a.x), b.x);
  r.y = g_sub(g_mul(lam, g_sub(a.x, r.x)), a.y);
  *out = r;
  return 0;
}
/* Mul<ScalarField> (curve/mod.rs:157-172): repeated addition, 0 gives Infinity */
static int p_smul(pt a, unsigned s, pt *out) {
  if (s == 0) { *out = p_inf(); return 0; }
  pt r = a;
  for (unsigned k = 1; k < s; k++) if (p_add(r, a, &r)) return 1;
  *out = r;
  return 0;
}

/* line_function (pairing.rs:130-164) */
static int line(pt a, pt b, pt in, gf *out) {
  if (a.inf || b.inf || in.inf) return 1;  /* "Cannot use point at infinity" */
  gf m;
  if (!g_eq(a.x, b.x)) {
    if (g_div(g_sub(b.y, a.y), g_sub(b.x, a.x), &m)) return 1;
  } else if (g_eq(a.y, b.y)) {
    gf three = {3, 0}, two = {2, 0};
    if (g_div(g_mul(three, g_mul(a.x, a.x)), g_mul(two, a.y), &m)) return 1;  /* + EQUATION_A = 0 */
  } else {
    *out = g_sub(in.x, a.x);
    return 0;
  }
  *out = g_sub(g_add(g_mul(m, g_sub(in.x, a.x)), a.y), in.y);
  return 0;
}

/* miller_loop::<_, 17> (pairing.rs:58-115) */
static int miller(pt p, pt q, gf *out) {
  gf x = {1, 0};
  pt z = p;
  int zeros = 0;
  const char *bits = "0001";  /* format!("{:b}", 17) = "10001", skip(1) */
  for (const char *c = bits; *c; c++) {
    gf tangent, vertical, inv;
    pt z2;
    if (line(z, z, q, &tangent)) return 1;
    if (p_add(z, z, &z2) || line(z2, p_neg(z2), q, &vertical)) return 1;  /* vertical_line(2 * z, q) */
    x = g_mul(x, x);
    if (g_zero(tangent)) zeros++; else x = g_mul(x, tangent);
    if (g_zero(vertical)) zeros--; else { if (g_inv(vertical, &inv)) return 1; x = g_mul(x, inv); }
    z = z2;
    if (*c == '1') {
      gf l, v;
      pt zp;
      if (line(z, p, q, &l) || p_add(z, p, &zp)) return 1;
      if (zp.inf) {
        if (g_zero(l)) zeros++; else x = g_mul(x, l);
      } else {
        if (line(zp, p_neg(zp), q, &v)) return 1;
        if (g_zero(l)) zeros++; else x = g_mul(x, l);
        if (g_zero(v)) zeros--; else { if (g_inv(v, &inv)) return 1; x = g_mul(x, inv); }
      }
      z = zp;
    }
  }
  if (zeros != 0) return 1;  /* assert_eq!(zeros, 0) */
  *out = x;
  return 0;
}

static int torsion17(pt p) {  /* pairing.rs:37-47: p added to itself 17 times returns p */
  pt r = p;
  for (int k = 0; k < 17; k++) if (p_add(r, p, &r)) return 0;
  return p_eq(r, p);
}

static int pairing(pt p, pt q, gf *out) {
  if (!torsion17(p) || !torsion17(q)) return 1;
  gf x;
  if (miller(p, q, &x)) return 1;
  *out = g_pow(x, (101 * 101 - 1) / 17);
  return 0;
}

/* out = (c0, c1) of pairing(p, q); 1 where the reference panics (and for off-curve bytes, which it cannot hold) */
int orc_pairing(const uint8_t *p, const uint8_t *q, uint8_t *out) {
  if (!p_valid(p) || !p_valid(q)) return 1;
  gf v;
  if (pairing(p_unpack(p), p_unpack(q), &v)) return 1;
  out[0] = (uint8_t)v.c0;
  out[1] = (uint8_t)v.c1;
  return 0;
}

/* *ok = kzg::check(c, q, z, v, g1_srs, g2_srs); 1 where the reference panics (or a point is off the curve) */
int orc_kzg_check(const uint8_t *c, const uint8_t *q, unsigned z, unsigned v, const uint8_t *g1_srs, size_t n_g1,
                  const uint8_t *g2_srs, size_t n_g2, uint8_t *ok) {
  if (n_g1 == 0 || n_g2 < 2) return 1;  /* expect("has g1 srs"), g2_srs[1] */
  if (!p_valid(c) || !p_valid(q) || !p_valid(g1_srs) || !p_valid(g2_srs + 4) || z >= 17 || v >= 17) return 1;
  const uint8_t gen_w[4] = {36, 0, 0, 31};  /* PlutoExtendedCurve::GENERATOR (pluto_curve.rs:46-49) */
  const pt gen = p_unpack(gen_w);
  pt zg, b, vg, r;
  if (p_smul(gen, z, &zg) || p_add(p_unpack(g2_srs + 4), p_neg(zg), &b)) return 1;   /* g2 - GEN * point */
  if (p_smul(p_unpack(g1_srs), v, &vg) || p_add(p_unpack(c), p_neg(vg), &r)) return 1;  /* p - g1 * value */
  gf lhs, rhs;
  if (pairing(p_unpack(q), b, &lhs) || pairing(r, gen, &rhs)) return 1;
  *ok = g_eq(lhs, rhs) ? 1 : 0;
  return 0;
}

/* Order of a packed curve point in E(F_101²) (1 for Infinity), 0 for an off-curve point */
unsigned orc_point_order(const uint8_t *w) {
  if (!p_valid(w)) return 0;
  const pt p = p_unpack(w);
  pt r = p;
  unsigned k = 1;
  while (!r.inf) {
    if (p_add(r, p, &r)) return 0;
    k++;
  }
  return p.inf ? 1 : k;
}

/* Many rows: panic[i] = 1 where orc_pairing / orc_kzg_check returns 1 */
void orc_pairing_many(const uint8_t *p, const uint8_t *q, size_t n, uint8_t *out, uint8_t *panic) {
  for (size_t i = 0; i < n; i++) panic[i] = (uint8_t)orc_pairing(p + 4 * i, q + 4 * i, out + 2 * i);
}
void orc_kzg_check_many(const uint8_t *c, const uint8_t *q, const uint8_t *z, const uint8_t *v, size_t n, const uint8_t *g1_srs,
                        size_t n_g1, const uint8_t *g2_srs, size_t n_g2, uint8_t *ok, uint8_t *panic) {
  for (size_t i = 0; i < n; i++)
    panic[i] = (uint8_t)orc_kzg_check(c + 4 * i, q + 4 * i, z[i], v[i], g1_srs, n_g1, g2_srs, n_g2, ok + i);
}
