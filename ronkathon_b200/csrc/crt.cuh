// crt.cuh — the multi-modular product's primes, prime count and Garner step (poly_crt.cu).
//
// A product over a prime p whose p - 1 has no power-of-two root of the product's length is convolved over the integers:
// the coefficients of the lifted operands are convolved modulo k ≤ 3 auxiliary NTT primes q_i, each residue vector on
// the power-of-two transforms of q_i, and every coefficient x < q_1⋯q_k is rebuilt by Garner's algorithm,
//   x = c1 + q1·t2 + q1·q2·t3,   t2 = (c2 - c1)·q1^-1 mod q2,   t3 = (c3 - c1 - q1·t2)·(q1·q2)^-1 mod q3,
// and reduced mod p.  Every routine here is host-and-device code, so that tests/emu compiles this very step for the CPU.
#pragma once
#include "field.cuh"

namespace ronk {

// The auxiliary primes in the order they are used, with a generator of each (a quadratic non-residue): Goldilocks
// (2-adicity 32, the specialised transforms), 0xFFFFFFFF70000001 (2-adicity 28) and 29·2^57 + 1 (2-adicity 57).
constexpr int kCrtPrimes = 3;
constexpr u64 kCrtQ[kCrtPrimes] = {GL_P, 0xFFFFFFFF70000001ULL, 0x3A00000000000001ULL};
constexpr u64 kCrtG[kCrtPrimes] = {7, 3, 3};

// Exact 256-bit helpers for the prime count: x (four little-endian words) *= m, and a < b.
inline void crt_mul_words(u64 x[4], u64 m) {
  unsigned __int128 carry = 0;
  for (int i = 0; i < 4; i++) {
    const unsigned __int128 t = (unsigned __int128)x[i] * m + carry;
    x[i] = (u64)t;
    carry = t >> 64;
  }
}
inline bool crt_less(const u64 a[4], const u64 b[4]) {
  for (int i = 3; i >= 0; i--)
    if (a[i] != b[i]) return a[i] < b[i];
  return false;
}

// The number of auxiliary primes a product over p needs when the shorter operand has m terms: the smallest k with
// q_1⋯q_k > m·(p - 1)², the largest coefficient the integer product can have.  0 when even all three fall short (never
// for m ≤ 2^26: the bound is then below 2^154 and the three primes' product above 2^189).
inline int crt_prime_count(u64 p, u64 m) {
  u64 bound[4] = {m, 0, 0, 0};
  crt_mul_words(bound, p - 1);
  crt_mul_words(bound, p - 1);
  u64 Q[4] = {1, 0, 0, 0};
  for (int k = 1; k <= kCrtPrimes; k++) {
    crt_mul_words(Q, kCrtQ[k - 1]);
    if (crt_less(bound, Q)) return k;
  }
  return 0;
}

// Garner's constants.  A constant c in Montgomery form (c·2^64 mod q) turns redc_mul(x, c) into x·c mod q, canonical
// for ANY 64-bit x, since the product stays below q·2^64: a residue of one modulus needs no reduction before it is
// multiplied modulo another.
struct CrtConsts {
  MontField m2, m3;  // q2, q3 (h_mont_field: only the modulus, p^-1 mod 2^64 and 2^128 mod p are used)
  u64 inv1;          // q1^-1 mod q2, Montgomery form
  u64 inv12;         // (q1·q2)^-1 mod q3, Montgomery form
  u64 q1inv12;       // q1·(q1·q2)^-1 mod q3, Montgomery form
  u64 one_tw;        // 1, q1 mod p and q1·q2 mod p in the twiddle form of p's policy (mul_tw's second operand)
  u64 q1_tw;
  u64 q12_tw;
};

template <class F>
inline CrtConsts crt_consts(const F& f) {
  const u64 q1 = kCrtQ[0], q2 = kCrtQ[1], q3 = kCrtQ[2], p = f.modulus();
  auto mont = [](u64 x, u64 q) { return h_mulmod(x % q, (u64)((((unsigned __int128)1) << 64) % q), q); };
  CrtConsts k;
  k.m2 = h_mont_field(q2);
  k.m3 = h_mont_field(q3);
  k.inv1 = mont(h_powmod(q1 % q2, q2 - 2, q2), q2);
  const u64 inv12 = h_powmod(h_mulmod(q1 % q3, q2 % q3, q3), q3 - 2, q3);
  k.inv12 = mont(inv12, q3);
  k.q1inv12 = mont(h_mulmod(q1 % q3, inv12, q3), q3);
  k.one_tw = f.to_tw(1 % p);
  k.q1_tw = f.to_tw(q1 % p);
  k.q12_tw = f.to_tw(h_mulmod(q1 % p, q2 % p, p));
  return k;
}

// One coefficient: its K residues c_i < q_i in, the exact integer coefficient mod p (canonical) out.  Each product
// below has a canonical constant as its second operand, so none of its first operands needs reducing: c1 < q1 may be
// ≥ q3 or ≥ p, t2 < q2 may be ≥ q3 or ≥ p, t3 < q3 may be ≥ p.  c1 < q1 < q2 is canonical mod q2.
template <int K, class F>
RONK_HD u64 crt_garner(const F& f, const CrtConsts& k, u64 c1, u64 c2, u64 c3) {
  u64 x = f.mul_tw(c1, k.one_tw);  // c1 mod p
  if constexpr (K >= 2) {
    const u64 t2 = k.m2.redc_mul(k.m2.sub(c2, c1), k.inv1);
    x = f.add(x, f.mul_tw(t2, k.q1_tw));
    if constexpr (K >= 3) {
      const MontField& m = k.m3;
      const u64 t3 = m.sub(m.sub(m.redc_mul(c3, k.inv12), m.redc_mul(c1, k.inv12)), m.redc_mul(t2, k.q1inv12));
      x = f.add(x, f.mul_tw(t3, k.q12_tw));
    }
  }
  return x;
}

// x mod q for x < 2^64 and q > 2^61: at most four subtractions (2^64 < 4.5·q3).
RONK_HD u64 crt_below(u64 x, u64 q) {
  while (x >= q) x -= q;
  return x;
}

}  // namespace ronk
