/*
 * ronk_oracle.c — CPU restatement of pluto/ronkathon's field / polynomial / kzg::commit path.
 *
 * THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline / --impl reference legs may load it.  The product library
 * (ronkathon_b200/libronk_b200.so) never links, loads or calls anything in this file.
 *
 * Parity status: the reference is Rust (nightly-2024-06-10) and cannot be compiled in this
 * environment, so this file is a line-by-line restatement, PINNED by every known-answer vector
 * the reference's own tests hold for this path (tests/golden/reference_kats.json, checked by
 * tests/test_oracle_golden.py).  For p = 101 / 17 / 127 the results are therefore pinned
 * bit-for-bit.  The 64-bit (Goldilocks) instantiation cannot be instantiated by the reference at
 * all (SURVEY.md §8a D1-D6); there the oracle is the same code with 128-bit widening and is
 * cross-checked by an independent pure-Python big-int implementation (tests/golden/gen_goldilocks.py).
 *
 * Every function cites the reference file:line (relative to the reference's checkout root) it follows.
 * Values are canonical residues in uint64_t.  No global state; thread safe.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef uint64_t u64;
typedef unsigned __int128 u128;

#define ORC_OK 0
#define ORC_EINVAL 1

#define GOLDILOCKS 0xFFFFFFFF00000001ULL

/* ------------------------------------------------------------------------------------------
 * PrimeField<P>  (src/algebra/field/prime/mod.rs, src/algebra/field/prime/arithmetic.rs)
 * ---------------------------------------------------------------------------------------- */

/* PrimeField::new — prime/mod.rs:48-51: value % P */
u64 orc_new(u64 p, u64 v) { return v % p; }

/* Add — prime/arithmetic.rs:6: (a + b) % P.  Delta D1: widened so a 64-bit P cannot overflow. */
u64 orc_add(u64 p, u64 a, u64 b) { return (u64)(((u128)a + b) % p); }

/* Sub — prime/arithmetic.rs:22-27: overflowing_sub, add ORDER back on borrow. */
u64 orc_sub(u64 p, u64 a, u64 b) {
  u64 diff = a - b;
  if (a < b) diff += p;
  return diff;
}

/* Mul — prime/arithmetic.rs:37: (a * b) % P.  Delta D1: 128-bit product. */
u64 orc_mul(u64 p, u64 a, u64 b) { return (u64)(((u128)a * b) % p); }

/* Neg — prime/arithmetic.rs:64: ZERO - self */
u64 orc_neg(u64 p, u64 a) { return orc_sub(p, 0, a); }

/* Field::pow — prime/mod.rs:74-84.  Same recursion (power==0 → ONE, power==1 → self, even →
 * h*h, odd → h*h*self) with the half power evaluated once instead of twice (delta D2): the
 * value is identical, the cost is O(log e) instead of O(e). */
u64 orc_pow(u64 p, u64 a, u64 e) {
  if (e == 0) return 1 % p;
  if (e == 1) return a;
  u64 h = orc_pow(p, a, e / 2);
  u64 hh = orc_mul(p, h, h);
  return (e % 2 == 0) ? hh : orc_mul(p, hh, a);
}

/* Literal double recursion of prime/mod.rs:74-84, kept to show D2 changes no value (small e only). */
u64 orc_pow_literal(u64 p, u64 a, u64 e) {
  if (e == 0) return 1 % p;
  if (e == 1) return a;
  if (e % 2 == 0) return orc_mul(p, orc_pow_literal(p, a, e / 2), orc_pow_literal(p, a, e / 2));
  return orc_mul(p, orc_mul(p, orc_pow_literal(p, a, e / 2), orc_pow_literal(p, a, e / 2)), a);
}

/* Field::inverse — prime/mod.rs:62-72: None for 0, else a^(P-2).  Returns ORC_EINVAL for None. */
int orc_inverse(u64 p, u64 a, u64 *out) {
  if (a == 0) return ORC_EINVAL;
  *out = orc_pow(p, a, p - 2);
  return ORC_OK;
}

/* Div — prime/arithmetic.rs:54: self * rhs.inverse().unwrap()  (panics on 0 → ORC_EINVAL). */
int orc_div(u64 p, u64 a, u64 b, u64 *out) {
  u64 inv;
  if (orc_inverse(p, b, &inv)) return ORC_EINVAL;
  *out = orc_mul(p, a, inv);
  return ORC_OK;
}

/* Rem — prime/arithmetic.rs:70: self - (self / rhs) * rhs */
int orc_rem(u64 p, u64 a, u64 b, u64 *out) {
  u64 q;
  if (orc_div(p, a, b, &q)) return ORC_EINVAL;
  *out = orc_sub(p, a, orc_mul(p, q, b));
  return ORC_OK;
}

/* is_prime — prime/mod.rs:92-100 (trial division; panics for composite → returns 0).
 * Delta D3: only called for small moduli; Goldilocks primality is a known fact. */
int orc_is_prime(u64 n) {
  if (n == GOLDILOCKS) return 1;
  for (u64 i = 2; i * i <= n; i++)
    if (n % i == 0) return 0;
  return 1;
}

/* find_primitive_element — prime/mod.rs:110-123, literal (including its quirk of testing only one
 * cofactor).  Delta D4: for Goldilocks the literal search returns 3, which is a quadratic residue;
 * g is pinned to 7 (ω_{2^32} = 1753635133440165772).  P == 2 → ONE (prime/mod.rs:88-89). */
u64 orc_find_primitive_element(u64 p) {
  if (p == 2) return 1;
  if (p == GOLDILOCKS) return 7;
  for (u64 i = 2; i * i <= p; i++) {
    if ((p - 1) % i == 0) {
      if (orc_pow(p, i % p, (p - 1) / i) != 1) return i;
      else if (orc_pow(p, (p + 1 - i) % p, i) != 1) return p + 1 - i;
    }
  }
  return 0; /* panic!("generator not found") */
}

/* FiniteField::primitive_root_of_unity — algebra/field/mod.rs:70-75:
 * assert!((ORDER-1) % n == 0); PRIMITIVE_ELEMENT.pow((ORDER-1)/n) */
int orc_primitive_root_of_unity(u64 p, u64 g, u64 n, u64 *out) {
  if (n == 0 || (p - 1) % n != 0) return ORC_EINVAL;
  *out = orc_pow(p, g, (p - 1) / n);
  return ORC_OK;
}

/* ------------------------------------------------------------------------------------------
 * Polynomial<Monomial|Lagrange, F, D>  (src/polynomial/mod.rs, src/polynomial/arithmetic.rs)
 * ---------------------------------------------------------------------------------------- */

/* evaluate (Monomial) — polynomial/mod.rs:133-139: result += c * x.pow(i), not Horner. */
u64 orc_poly_eval(u64 p, const u64 *c, u64 d, u64 x) {
  u64 r = 0;
  for (u64 i = 0; i < d; i++) r = orc_add(p, r, orc_mul(p, c[i], orc_pow(p, x, i)));
  return r;
}

/* degree — polynomial/mod.rs:113-115: rposition of a nonzero coeff, else 0 */
u64 orc_poly_degree(const u64 *c, u64 d) {
  for (u64 i = d; i-- > 0;)
    if (c[i] != 0) return i;
  return 0;
}

/* leading_coefficient — polynomial/mod.rs:120-122 */
u64 orc_poly_leading(const u64 *c, u64 d) {
  for (u64 i = d; i-- > 0;)
    if (c[i] != 0) return c[i];
  return 0;
}

/* pow_mult::<D2>(coeff) — polynomial/mod.rs:153-157: out has D + D2 terms */
void orc_poly_pow_mult(u64 p, const u64 *c, u64 d, u64 d2, u64 coeff, u64 *out) {
  for (u64 i = 0; i < d + d2; i++) out[i] = (i >= d2) ? orc_mul(p, c[i - d2], coeff) : 0;
}

/* Add — polynomial/arithmetic.rs:23-34: zip self with rhs padded by zeros, take D. */
void orc_poly_add(u64 p, const u64 *a, u64 da, const u64 *b, u64 db, u64 *out) {
  for (u64 i = 0; i < da; i++) out[i] = orc_add(p, a[i], i < db ? b[i] : 0);
}

/* Sub — polynomial/arithmetic.rs:56-67 */
void orc_poly_sub(u64 p, const u64 *a, u64 da, const u64 *b, u64 db, u64 *out) {
  for (u64 i = 0; i < da; i++) out[i] = orc_sub(p, a[i], i < db ? b[i] : 0);
}

/* Neg — polynomial/arithmetic.rs:81-94 */
void orc_poly_neg(u64 p, const u64 *a, u64 da, u64 *out) {
  for (u64 i = 0; i < da; i++) out[i] = orc_neg(p, a[i]);
}

/* Mul — polynomial/arithmetic.rs:110-118: schoolbook, out has D + D2 - 1 terms, no trimming. */
void orc_poly_mul(u64 p, const u64 *a, u64 da, const u64 *b, u64 db, u64 *out) {
  for (u64 i = 0; i < da + db - 1; i++) out[i] = 0;
  for (u64 i = 0; i < da; i++)
    for (u64 j = 0; j < db; j++) out[i + j] = orc_add(p, out[i + j], orc_mul(p, a[i], b[j]));
}

/* quotient_and_remainder — polynomial/mod.rs:170-225 (Div/Rem: arithmetic.rs:130-146).
 * q and r both have `da` terms.  Returns ORC_EINVAL where the reference would panic
 * (all-zero divisor → rposition().unwrap() / inverse().unwrap()). */
int orc_poly_divrem(u64 p, const u64 *a, u64 da, const u64 *b, u64 db, u64 *q, u64 *r) {
  u64 *pc = (u64 *)malloc((da ? da : 1) * sizeof(u64));
  u64 plen = da;
  memcpy(pc, a, da * sizeof(u64));
  for (u64 i = 0; i < da; i++) q[i] = 0;
  u64 c = orc_poly_leading(b, db); /* :180 */
  int rc = ORC_OK;
  for (;;) {
    /* :183-184 loop condition */
    u64 nz = 0;
    for (u64 i = 0; i < plen; i++) nz += (pc[i] != 0);
    if (!(nz > 0 && plen >= db)) break;
    u64 p_degree = 0, rhs_degree = 0;
    int found = 0;
    for (u64 i = plen; i-- > 0;) if (pc[i] != 0) { p_degree = i; found = 1; break; }
    (void)found;
    found = 0;
    for (u64 i = db; i-- > 0;) if (b[i] != 0) { rhs_degree = i; found = 1; break; }
    if (!found) { rc = ORC_EINVAL; break; } /* unwrap on None */
    if (p_degree < rhs_degree) break;      /* :190-192 */
    u64 diff = p_degree - rhs_degree;
    u64 cinv;
    if (orc_inverse(p, c, &cinv)) { rc = ORC_EINVAL; break; }
    u64 s = orc_mul(p, pc[p_degree], cinv); /* :195 */
    q[diff] = s;
    for (u64 i = 0; i < db; i++) { /* :198-200; out-of-range index panics in the reference */
      if (diff + i >= plen) { rc = ORC_EINVAL; break; }
      pc[diff + i] = orc_sub(p, pc[diff + i], orc_mul(p, b[i], s));
    }
    if (rc) break;
    while (plen > 0 && pc[plen - 1] == 0) plen--; /* trim_zeros :202 */
  }
  for (u64 i = 0; i < da; i++) r[i] = (i < plen) ? pc[i] : 0; /* :215-221 */
  free(pc);
  return rc;
}

/* dft — polynomial/mod.rs:240-258: X[i] = Σ_j a_j ω^(i*j); any n | p-1. */
int orc_dft(u64 p, u64 g, const u64 *a, u64 n, u64 *out) {
  u64 w;
  if (orc_primitive_root_of_unity(p, g, n, &w)) return ORC_EINVAL;
  for (u64 i = 0; i < n; i++) {
    u64 acc = 0;
    for (u64 j = 0; j < n; j++) acc = orc_add(p, acc, orc_mul(p, a[j], orc_pow(p, w, i * j)));
    out[i] = acc;
  }
  return ORC_OK;
}

/* fft_recursive — polynomial/mod.rs:295-323 (ifft_recursive :455-484 is the same body).
 * Faithful: two fresh vectors per call, omega.pow(2) passed down, running current_root. */
static void fft_recursive(u64 p, u64 *values, u64 n, u64 omega) {
  if (n <= 1) return;
  u64 half = n / 2;
  u64 *even = (u64 *)malloc(half * sizeof(u64));
  u64 *odd = (u64 *)malloc(half * sizeof(u64));
  for (u64 i = 0; i < half; i++) {
    even[i] = values[2 * i];
    odd[i] = values[2 * i + 1];
  }
  u64 w2 = orc_pow(p, omega, 2);
  fft_recursive(p, even, half, w2);
  fft_recursive(p, odd, half, w2);
  u64 current_root = 1;
  for (u64 i = 0; i < half; i++) {
    u64 t = orc_mul(p, current_root, odd[i]);
    values[i] = orc_add(p, even[i], t);
    values[i + half] = orc_sub(p, even[i], t);
    current_root = orc_mul(p, current_root, omega);
  }
  free(even);
  free(odd);
}

static int is_pow2(u64 n) { return n && !(n & (n - 1)); }

/* fft — polynomial/mod.rs:273-290.  In place on `values`.  The Lagrange node table the reference
 * then materialises (:358-365, O(n²)) is implicit here (delta D6). */
int orc_fft(u64 p, u64 g, u64 *values, u64 n) {
  u64 w;
  if (!is_pow2(n)) return ORC_EINVAL; /* compile-time bound :274 */
  if (orc_primitive_root_of_unity(p, g, n, &w)) return ORC_EINVAL;
  fft_recursive(p, values, n, w);
  return ORC_OK;
}

/* ifft — polynomial/mod.rs:430-453: omega = root.inverse(); recurse; scale by F::from(D).inverse() */
int orc_ifft(u64 p, u64 g, u64 *values, u64 n) {
  u64 w, winv, dinv;
  if (!is_pow2(n)) return ORC_EINVAL;
  if (orc_primitive_root_of_unity(p, g, n, &w)) return ORC_EINVAL;
  if (orc_inverse(p, w, &winv)) return ORC_EINVAL;
  fft_recursive(p, values, n, winv);
  if (orc_inverse(p, n % p, &dinv)) return ORC_EINVAL;
  for (u64 i = 0; i < n; i++) values[i] = orc_mul(p, values[i], dinv);
  return ORC_OK;
}

/* Lagrange-basis evaluate — polynomial/mod.rs:382-415 (barycentric, nodes = ω^i from :363). */
int orc_lagrange_eval(u64 p, u64 g, const u64 *c, u64 n, u64 x, u64 *out) {
  u64 w;
  if (orc_primitive_root_of_unity(p, g, n, &w)) return ORC_EINVAL;
  u64 *nodes = (u64 *)malloc(n * sizeof(u64));
  u64 *weights = (u64 *)malloc(n * sizeof(u64));
  for (u64 i = 0; i < n; i++) nodes[i] = orc_pow(p, w, i);
  for (u64 idx = 0; idx < n; idx++) {
    u64 wt = 1;
    for (u64 m = 0; m < n; m++)
      if (idx != m) {
        u64 inv;
        /* :386-393 F::ONE.div(x_j - x_m) panics when ω's order is below n and two nodes coincide */
        if (orc_div(p, 1, orc_sub(p, nodes[idx], nodes[m]), &inv)) {
          free(nodes);
          free(weights);
          return ORC_EINVAL;
        }
        wt = orc_mul(p, wt, inv);
      }
    weights[idx] = wt;
  }
  u64 l = 1;
  for (u64 i = 0; i < n; i++) l = orc_mul(p, l, orc_sub(p, x, nodes[i]));
  /* fold (:405-414): `if n == x { return c }` returns from the closure, i.e. acc := c */
  u64 acc = 0;
  for (u64 j = 0; j < n; j++) {
    if (nodes[j] == x) { acc = c[j]; continue; }
    u64 t;
    orc_div(p, orc_mul(p, c[j], weights[j]), orc_sub(p, x, nodes[j]), &t);
    acc = orc_add(p, acc, t);
  }
  *out = orc_mul(p, l, acc);
  free(nodes);
  free(weights);
  return ORC_OK;
}

/* ------------------------------------------------------------------------------------------
 * Fast iterative NTT — NOT a reference algorithm; same mathematical map X[k] = Σ a_j ω^(jk) as
 * fft_recursive, used only to check large sizes quickly (validated against orc_fft in tests).
 * ---------------------------------------------------------------------------------------- */
int orc_ntt_fast(u64 p, u64 g, u64 *a, u64 n, int inverse) {
  u64 w;
  if (!is_pow2(n)) return ORC_EINVAL;
  if (orc_primitive_root_of_unity(p, g, n, &w)) return ORC_EINVAL;
  if (inverse && orc_inverse(p, w, &w)) return ORC_EINVAL;
  unsigned lg = 0;
  while ((1ULL << lg) < n) lg++;
  for (u64 i = 0; i < n; i++) {
    u64 r = 0;
    for (unsigned b = 0; b < lg; b++) r |= ((i >> b) & 1) << (lg - 1 - b);
    if (r > i) { u64 t = a[i]; a[i] = a[r]; a[r] = t; }
  }
  u64 *tw = (u64 *)malloc((n / 2 ? n / 2 : 1) * sizeof(u64));
  tw[0] = 1;
  for (u64 i = 1; i < n / 2; i++) tw[i] = orc_mul(p, tw[i - 1], w);
  for (u64 len = 2; len <= n; len <<= 1) {
    u64 half = len / 2, step = n / len;
    for (u64 s = 0; s < n; s += len)
      for (u64 i = 0; i < half; i++) {
        u64 t = orc_mul(p, tw[i * step], a[s + i + half]);
        u64 u = a[s + i];
        a[s + i] = orc_add(p, u, t);
        a[s + i + half] = orc_sub(p, u, t);
      }
  }
  free(tw);
  if (inverse) {
    u64 ninv;
    orc_inverse(p, n % p, &ninv);
    for (u64 i = 0; i < n; i++) a[i] = orc_mul(p, a[i], ninv);
  }
  return ORC_OK;
}

/* out[i] = a[i]*b[i] (prime/arithmetic.rs:37 element-wise) — used to build the convolution-theorem check. */
void orc_vec_mul(u64 p, const u64 *a, const u64 *b, u64 *out, u64 n) {
  for (u64 i = 0; i < n; i++) out[i] = orc_mul(p, a[i], b[i]);
}
/* Horner evaluation: same value as orc_poly_eval (which is the reference's O(D²) form); used for
 * spot checks X[k] == a(ω^k) at sizes where the literal form is too slow. */
u64 orc_poly_eval_horner(u64 p, const u64 *c, u64 d, u64 x) {
  u64 r = 0;
  for (u64 i = d; i-- > 0;) r = orc_add(p, orc_mul(p, r, x), c[i]);
  return r;
}

/* splitmix64 stream reduced mod p — SURVEY.md §8c/§8d synthetic-input definition. */
void orc_splitmix_fill(u64 p, u64 seed, u64 *out, u64 n) {
  u64 s = seed;
  for (u64 i = 0; i < n; i++) {
    s += 0x9E3779B97F4A7C15ULL;
    u64 z = s;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    z ^= z >> 31;
    out[i] = z % p;
  }
}

/* ------------------------------------------------------------------------------------------
 * GF(101²) = F101[t]/(t²+2)  (src/algebra/field/extension/gf_101_2.rs, extension/arithmetic.rs)
 * element = {c0, c1} meaning c0 + c1·t
 * ---------------------------------------------------------------------------------------- */
#define Q 101
typedef struct { u64 c[2]; } gf2;

static gf2 gf_new(u64 a, u64 b) { gf2 r = {{a % Q, b % Q}}; return r; }
/* Add/Sub/Neg — extension/arithmetic.rs:7-53: coefficient-wise */
static gf2 gf_add(gf2 a, gf2 b) { return gf_new(orc_add(Q, a.c[0], b.c[0]), orc_add(Q, a.c[1], b.c[1])); }
static gf2 gf_sub(gf2 a, gf2 b) { return gf_new(orc_sub(Q, a.c[0], b.c[0]), orc_sub(Q, a.c[1], b.c[1])); }
static gf2 gf_neg(gf2 a) { return gf_new(orc_neg(Q, a.c[0]), orc_neg(Q, a.c[1])); }
static int gf_eq(gf2 a, gf2 b) { return a.c[0] == b.c[0] && a.c[1] == b.c[1]; }

/* Mul — gf_101_2.rs:86-100: (poly_self * poly_rhs) % (t² + 2), literally through the polynomial
 * routines above (schoolbook mul then long division), as the reference does. */
static gf2 gf_mul(gf2 a, gf2 b) {
  u64 prod[3], irred[3] = {2, 0, 1}, q[3], r[3];
  orc_poly_mul(Q, a.c, 2, b.c, 2, prod);
  orc_poly_divrem(Q, prod, 3, irred, 3, q, r);
  return gf_new(r[0], r[1]);
}

/* inverse — gf_101_2.rs:35-47: scalar = (a0² + 2·a1²)⁻¹; (a0·scalar, -a1·scalar) */
static int gf_inv(gf2 a, gf2 *out) {
  if (a.c[0] == 0 && a.c[1] == 0) return ORC_EINVAL;
  u64 norm = orc_add(Q, orc_pow(Q, a.c[0], 2), orc_mul(Q, 2, orc_pow(Q, a.c[1], 2)));
  u64 s;
  if (orc_inverse(Q, norm, &s)) return ORC_EINVAL;
  *out = gf_new(orc_mul(Q, a.c[0], s), orc_mul(Q, orc_neg(Q, a.c[1]), s));
  return ORC_OK;
}

/* Div — gf_101_2.rs:113-118 */
static int gf_div(gf2 a, gf2 b, gf2 *out) {
  gf2 bi;
  if (gf_inv(b, &bi)) return ORC_EINVAL;
  *out = gf_mul(a, bi);
  return ORC_OK;
}

void orc_gf_add(const uint8_t a[2], const uint8_t b[2], uint8_t out[2]) {
  gf2 r = gf_add(gf_new(a[0], a[1]), gf_new(b[0], b[1])); out[0] = r.c[0]; out[1] = r.c[1];
}
void orc_gf_sub(const uint8_t a[2], const uint8_t b[2], uint8_t out[2]) {
  gf2 r = gf_sub(gf_new(a[0], a[1]), gf_new(b[0], b[1])); out[0] = r.c[0]; out[1] = r.c[1];
}
void orc_gf_neg(const uint8_t a[2], uint8_t out[2]) {
  gf2 r = gf_neg(gf_new(a[0], a[1])); out[0] = r.c[0]; out[1] = r.c[1];
}
void orc_gf_mul(const uint8_t a[2], const uint8_t b[2], uint8_t out[2]) {
  gf2 r = gf_mul(gf_new(a[0], a[1]), gf_new(b[0], b[1])); out[0] = r.c[0]; out[1] = r.c[1];
}
int orc_gf_inv(const uint8_t a[2], uint8_t out[2]) {
  gf2 r;
  if (gf_inv(gf_new(a[0], a[1]), &r)) return ORC_EINVAL;
  out[0] = r.c[0]; out[1] = r.c[1];
  return ORC_OK;
}

/* ------------------------------------------------------------------------------------------
 * AffinePoint<PlutoExtendedCurve>  (src/curve/mod.rs, src/curve/pluto_curve.rs)
 * y² = x³ + 3 over GF(101²) (pluto_curve.rs:40-51; a = 0, b = 3).  PlutoBaseCurve points embed
 * with c1 = 0 (pluto_curve.rs:53-64).  Wire format: 4 bytes x0,x1,y0,y1; 0xFF×4 = Infinity.
 * ---------------------------------------------------------------------------------------- */
typedef struct { gf2 x, y; int inf; } pt;

static pt pt_load(const uint8_t b[4]) {
  pt r;
  if (b[0] == 0xFF && b[1] == 0xFF && b[2] == 0xFF && b[3] == 0xFF) { r.inf = 1; r.x = gf_new(0, 0); r.y = gf_new(0, 0); return r; }
  r.inf = 0; r.x = gf_new(b[0], b[1]); r.y = gf_new(b[2], b[3]);
  return r;
}
static void pt_store(pt a, uint8_t b[4]) {
  if (a.inf) { b[0] = b[1] = b[2] = b[3] = 0xFF; return; }
  b[0] = a.x.c[0]; b[1] = a.x.c[1]; b[2] = a.y.c[0]; b[3] = a.y.c[1];
}

/* is_on_curve — curve/mod.rs:130-139: y² == x³ + a·x + b */
static int pt_on_curve(pt a) {
  if (a.inf) return 1;
  gf2 lhs = gf_mul(a.y, a.y);
  gf2 rhs = gf_add(gf_mul(gf_mul(a.x, a.x), a.x), gf_new(3, 0));
  return gf_eq(lhs, rhs);
}

/* Add — curve/mod.rs:178-213.  Returns ORC_EINVAL where AffinePoint::new (:78-82) would panic. */
static int pt_add(pt a, pt b, pt *out) {
  if (a.inf) { *out = b; return ORC_OK; }
  if (b.inf) { *out = a; return ORC_OK; }
  if (gf_eq(a.x, b.x) && gf_eq(a.y, gf_neg(b.y))) { out->inf = 1; out->x = gf_new(0, 0); out->y = gf_new(0, 0); return ORC_OK; }
  gf2 lambda;
  if (gf_eq(a.x, b.x) && gf_eq(a.y, b.y)) {
    gf2 three = gf_new(3, 0), two = gf_new(2, 0);
    if (gf_div(gf_mul(gf_mul(three, a.x), a.x), gf_mul(two, a.y), &lambda)) return ORC_EINVAL;
  } else {
    if (gf_div(gf_sub(b.y, a.y), gf_sub(b.x, a.x), &lambda)) return ORC_EINVAL;
  }
  pt r;
  r.inf = 0;
  r.x = gf_sub(gf_sub(gf_mul(lambda, lambda), a.x), b.x);
  r.y = gf_sub(gf_mul(lambda, gf_sub(a.x, r.x)), a.y);
  if (!pt_on_curve(r)) return ORC_EINVAL;
  *out = r;
  return ORC_OK;
}

/* Neg — curve/mod.rs:225-235 */
static pt pt_neg(pt a) { if (!a.inf) a.y = gf_neg(a.y); return a; }

/* Mul<ScalarField> — curve/mod.rs:157-172: 0 → Infinity, else (s-1) repeated `+=`. */
static int pt_smul(pt a, u64 s, pt *out) {
  if (s == 0) { out->inf = 1; out->x = gf_new(0, 0); out->y = gf_new(0, 0); return ORC_OK; }
  pt val = a;
  for (u64 i = 1; i < s; i++)
    if (pt_add(val, a, &val)) return ORC_EINVAL;
  *out = val;
  return ORC_OK;
}

int orc_point_on_curve(const uint8_t a[4]) { return pt_on_curve(pt_load(a)); }
int orc_point_add(const uint8_t a[4], const uint8_t b[4], uint8_t out[4]) {
  pt r;
  if (pt_add(pt_load(a), pt_load(b), &r)) return ORC_EINVAL;
  pt_store(r, out);
  return ORC_OK;
}
void orc_point_neg(const uint8_t a[4], uint8_t out[4]) { pt_store(pt_neg(pt_load(a)), out); }
/* double — curve/mod.rs:113-128 (same tangent formula as the P==Q arm of Add; Infinity → Infinity). */
int orc_point_double(const uint8_t a[4], uint8_t out[4]) {
  pt p = pt_load(a), r;
  if (p.inf) { pt_store(p, out); return ORC_OK; }
  gf2 m;
  if (gf_div(gf_mul(gf_mul(gf_new(3, 0), p.x), p.x), gf_mul(gf_new(2, 0), p.y), &m)) return ORC_EINVAL;
  r.inf = 0;
  r.x = gf_sub(gf_mul(m, m), gf_mul(gf_new(2, 0), p.x));
  r.y = gf_sub(gf_mul(m, gf_sub(gf_mul(gf_new(3, 0), p.x), gf_mul(m, m))), p.y);
  if (!pt_on_curve(r)) return ORC_EINVAL;
  pt_store(r, out);
  return ORC_OK;
}
int orc_point_smul(const uint8_t a[4], u64 s, uint8_t out[4]) {
  pt r;
  if (pt_smul(pt_load(a), s % 17, &r)) return ORC_EINVAL;
  pt_store(r, out);
  return ORC_OK;
}

/* kzg::commit — kzg/setup.rs:48-60: assert srs.len() >= coeffs.len(); zip; map g1*coeff; sum
 * (Sum = reduce(+) or Infinity, curve/mod.rs:219-223).  Literal: repeated-addition scalar mul. */
int orc_commit(const uint8_t *points, u64 n_points, const uint8_t *scalars, u64 n_scalars, uint8_t out[4]) {
  if (n_points < n_scalars) return ORC_EINVAL;
  pt acc; acc.inf = 1; acc.x = gf_new(0, 0); acc.y = gf_new(0, 0);
  int first = 1;
  for (u64 i = 0; i < n_scalars; i++) {
    pt term, P = pt_load(points + 4 * i);
    if (!pt_on_curve(P)) return ORC_EINVAL;
    if (pt_smul(P, scalars[i] % 17, &term)) return ORC_EINVAL;
    if (first) { acc = term; first = 0; }
    else if (pt_add(acc, term, &acc)) return ORC_EINVAL;
  }
  pt_store(acc, out);
  return ORC_OK;
}

/* kzg::setup — kzg/setup.rs:10-43: tau = 2; 7 G1 powers of (1,2), 2 G2 powers of (36, 31t). */
int orc_setup(uint8_t g1[7 * 4], uint8_t g2[2 * 4]) {
  const uint8_t G1[4] = {1, 0, 2, 0}, G2[4] = {36, 0, 0, 31};
  for (u64 i = 0; i < 7; i++) {
    u64 s = orc_pow(17, 2, i);
    if (orc_point_smul(G1, s, g1 + 4 * i)) return ORC_EINVAL;
    if (i < 2 && orc_point_smul(G2, s, g2 + 4 * i)) return ORC_EINVAL;
  }
  return ORC_OK;
}

/* kzg::open::<D> — kzg/setup.rs:63-78: poly / (x - z) via Polynomial::div, then commit(quotient). */
int orc_open(const uint8_t *coeffs, u64 d, uint8_t z, const uint8_t *points, u64 n_points, uint8_t out[4]) {
  u64 *c = (u64 *)malloc(d * sizeof(u64)), *q = (u64 *)malloc(d * sizeof(u64)), *r = (u64 *)malloc(d * sizeof(u64));
  u64 divisor[2] = {orc_neg(17, z % 17), 1};
  for (u64 i = 0; i < d; i++) c[i] = coeffs[i] % 17;
  int rc = orc_poly_divrem(17, c, d, divisor, 2, q, r);
  if (!rc) {
    uint8_t *qs = (uint8_t *)malloc(d);
    for (u64 i = 0; i < d; i++) qs[i] = (uint8_t)q[i];
    rc = orc_commit(points, n_points, qs, d, out);
    free(qs);
  }
  free(c); free(q); free(r);
  return rc;
}

/* Fast MSM check (NOT a reference algorithm): double-and-add per term; used to check 2^20-term
 * commits quickly.  Validated against orc_commit in tests. */
int orc_commit_fast(const uint8_t *points, u64 n_points, const uint8_t *scalars, u64 n_scalars, uint8_t out[4]) {
  if (n_points < n_scalars) return ORC_EINVAL;
  pt bucket[17];
  for (int s = 0; s < 17; s++) { bucket[s].inf = 1; bucket[s].x = gf_new(0, 0); bucket[s].y = gf_new(0, 0); }
  for (u64 i = 0; i < n_scalars; i++) {
    pt P = pt_load(points + 4 * i);
    if (!pt_on_curve(P)) return ORC_EINVAL;
    if (pt_add(bucket[scalars[i] % 17], P, &bucket[scalars[i] % 17])) return ORC_EINVAL;
  }
  pt run, acc; run.inf = acc.inf = 1; run.x = run.y = acc.x = acc.y = gf_new(0, 0);
  for (int s = 16; s >= 1; s--) {
    if (pt_add(run, bucket[s], &run)) return ORC_EINVAL;
    if (pt_add(acc, run, &acc)) return ORC_EINVAL;
  }
  pt_store(acc, out);
  return ORC_OK;
}

/* Reed–Solomon encode (next row) — codes/reed_solomon.rs:42-52: y_i = poly.evaluate(ω_N^i),
 * x_i = ω_N^i, for i in 0..N. */
int orc_rs_encode(u64 p, u64 g, const u64 *msg, u64 k, u64 n, u64 *xs, u64 *ys) {
  u64 w;
  if (orc_primitive_root_of_unity(p, g, n, &w)) return ORC_EINVAL;
  for (u64 i = 0; i < n; i++) {
    xs[i] = orc_pow(p, w, i);
    ys[i] = orc_poly_eval(p, msg, k, xs[i]);
  }
  return ORC_OK;
}

/* Reed–Solomon decode (next row) — codes/reed_solomon.rs:55-107, literally: the first K coordinates
 * are interpolated coefficient by coefficient,
 *   data[i] = Σ_j  sign(i) · e_{K-1-i}(x without x_j) · y_j / Π_{k≠j} (x_k - x_j),
 * sign(i) = -1 for odd i (:78-82), e_m = sum over all m-element combinations of the product (:83-89;
 * the empty combination contributes ONE).  Exponential in K like the reference; K <= 20 here.
 * A repeated x makes the denominator zero and `/` panics (prime/arithmetic.rs:54) -> ORC_EINVAL. */
int orc_rs_decode(u64 p, const u64 *xs, const u64 *ys, u64 k, u64 *data) {
  if (k > 20) return ORC_EINVAL;
  for (u64 i = 0; i < k; i++) data[i] = 0;
  for (u64 i = 0; i < k; i++) {
    for (u64 j = 0; j < k; j++) {
      u64 others[20];
      u64 m = 0;
      for (u64 t = 0; t < k; t++) if (t != j) others[m++] = xs[t];
      const u64 want = k - 1 - i;
      u64 esum = 0;
      for (u64 mask = 0; mask < ((u64)1 << m); mask++) {
        if ((u64)__builtin_popcountll(mask) != want) continue;
        u64 prod = 1 % p;
        for (u64 t = 0; t < m; t++) if (mask >> t & 1) prod = orc_mul(p, prod, others[t]);
        esum = orc_add(p, esum, prod);
      }
      const u64 sign = (i % 2 == 1) ? orc_sub(p, 0, 1 % p) : 1 % p; /* :78-82 */
      const u64 num = orc_mul(p, orc_mul(p, sign, esum), ys[j]);     /* :90-91 */
      u64 den = 1 % p;                                               /* :94-100 */
      for (u64 t = 0; t < k; t++) if (t != j) den = orc_mul(p, den, orc_sub(p, xs[t], xs[j]));
      u64 dinv;
      if (orc_inverse(p, den, &dinv)) return ORC_EINVAL;
      data[i] = orc_add(p, data[i], orc_mul(p, num, dinv));          /* :102 */
    }
  }
  return ORC_OK;
}

/* ------------------------------------------------------------------------------------------
 * Timed CPU baseline entry points (bench.py cpu_baseline / --impl reference).
 * orc_bench_fft_threads: `threads` independent faithful fft_recursive transforms, one per thread
 * (the reference itself is single-threaded; independent transforms are the only parallelism it
 * admits).  Inputs: splitmix64(seed 42 + t) mod p.  Returns wall seconds for the slowest thread.
 * ---------------------------------------------------------------------------------------- */
#include <pthread.h>
#include <time.h>

typedef struct { u64 p, g, n; u64 seed; double secs; u64 checksum; int rc; } bench_arg;

static double now_s(void) {
  struct timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return ts.tv_sec + 1e-9 * ts.tv_nsec;
}

static void *bench_worker(void *vp) {
  bench_arg *a = (bench_arg *)vp;
  u64 *buf = (u64 *)malloc(a->n * sizeof(u64));
  orc_splitmix_fill(a->p, a->seed, buf, a->n);
  double t0 = now_s();
  a->rc = orc_fft(a->p, a->g, buf, a->n);
  a->secs = now_s() - t0;
  u64 cs = 0;
  for (u64 i = 0; i < a->n; i++) cs += buf[i];
  a->checksum = cs;
  free(buf);
  return 0;
}

double orc_bench_fft_threads(u64 p, u64 g, u64 n, int threads, u64 *checksum0) {
  if (threads < 1) threads = 1;
  pthread_t *th = (pthread_t *)malloc(threads * sizeof(pthread_t));
  bench_arg *args = (bench_arg *)malloc(threads * sizeof(bench_arg));
  double t0 = now_s();
  for (int t = 0; t < threads; t++) {
    args[t].p = p; args[t].g = g; args[t].n = n; args[t].seed = 42 + t; args[t].rc = 0;
    pthread_create(&th[t], 0, bench_worker, &args[t]);
  }
  for (int t = 0; t < threads; t++) pthread_join(th[t], 0);
  double wall = now_s() - t0;
  (void)wall;
  double worst = 0;
  for (int t = 0; t < threads; t++) if (args[t].secs > worst) worst = args[t].secs;
  if (checksum0) *checksum0 = args[0].checksum;
  for (int t = 0; t < threads; t++) if (args[t].rc) worst = -1.0;
  free(th); free(args);
  return worst;
}
