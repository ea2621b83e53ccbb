// poseidon.cuh — the reference's Poseidon permutation (src/hashes/poseidon/mod.rs:137-149) and the batched sponge of
// ronk_poseidon_sponge_u64 (sponge.rs:71-294) on one row, state in registers.  Host-compilable (RONK_DEV), so tests/emu
// can run the very routine the kernel runs.
//
// The whole permutation runs in the policy's twiddle form (field.cuh): plain residues for Goldilocks, Montgomery form
// x·2^64 mod p for MontField.  Addition is the same in both forms and mul_tw(x̃, ỹ) = (x·y)~, so every product of the
// S-box and of the MDS layer is one mul_tw, with the round constants and the MDS matrix already in that form.  Rows are
// converted in on load (to_tw) and out on store (pos_from_tw).
//
// Round i of R = num_f + num_p (mod.rs:141-146): add rc[i·T + k], the S-box x^α on every element when
// i < num_f/2 or i ≥ num_p + num_f/2 (mod.rs:87-93; an odd num_f puts its extra full round at the end), else on element
// 0 only, then the literal MDS product new[i] = Σ_j state[j]·mds[i][j].  No sparse partial-round form: it would need
// other constants than the reference's.
#pragma once
#include "field.cuh"

namespace ronk {

constexpr int POS_MIN_WIDTH = 2, POS_MAX_WIDTH = 16;
// constants the kernel keeps in shared memory: (num_f + num_p)·width round constants + width² MDS words ≤ 6144 words
// (48 KiB, the default dynamic shared-memory limit).  At width 16 that is 368 rounds.
constexpr u64 POS_MAX_CONST_WORDS = 6144;

RONK_DEV u64 pos_from_tw(const GoldilocksField&, u64 x) { return x; }
RONK_DEV u64 pos_from_tw(const MontField& f, u64 x) { return f.redc_mul(x, 1); }

// A constant of the kernel's shared-memory tables.  On the device the load is volatile: the MDS words are the same in
// every round, and a plain load lets the compiler hoist up to 256 of them out of the round loop into registers and spill.
RONK_DEV u64 pos_const(const u64* p) {
#if defined(__CUDA_ARCH__)
  u64 v;
  asm volatile("ld.shared.u64 %0, [%1];" : "=l"(v) : "r"((u32)__cvta_generic_to_shared(p)));
  return v;
#else
  return *p;
#endif
}

// Round structure and S-box exponent of one configuration.
struct PosRounds {
  u32 rounds;       // R = num_f + num_p
  u32 full_lo;      // rounds i < full_lo are full (num_f / 2)
  u32 full_hi;      // rounds i ≥ full_hi are full (num_p + num_f / 2)
  u64 alpha;
};

// s[j] ← s[j]^α for j < N, left to right over α's bits in lockstep (α = 0 gives one, as Field::pow does: 0^0 = 1).
// Any order of the same products gives the same residue, so this is bit-identical to field_pow.
template <class F, int T, int N>
RONK_DEV void pos_sbox(const F& f, u64 (&s)[T], u64 alpha, u64 one) {
  if (alpha == 0) {
#pragma unroll
    for (int j = 0; j < N; j++) s[j] = one;
    return;
  }
  int b = 63;
  while (!((alpha >> b) & 1)) b--;
  u64 x[N];
#pragma unroll
  for (int j = 0; j < N; j++) x[j] = s[j];
  for (b--; b >= 0; b--) {
#pragma unroll
    for (int j = 0; j < N; j++) s[j] = f.mul_tw(s[j], s[j]);
    if ((alpha >> b) & 1) {
#pragma unroll
      for (int j = 0; j < N; j++) s[j] = f.mul_tw(s[j], x[j]);
    }
  }
}

// The permutation of one state in twiddle form.  rc: R·T words, mds: T² words row-major, both
// in twiddle form and, on the device, in shared memory.
template <class F, int T>
RONK_DEV void pos_permute(const F& f, u64 (&s)[T], const PosRounds& r, const u64* rc, const u64* mds, u64 one) {
  for (u32 i = 0; i < r.rounds; i++) {
#pragma unroll
    for (int k = 0; k < T; k++) s[k] = f.add(s[k], pos_const(rc + i * T + k));
    if (i < r.full_lo || i >= r.full_hi) pos_sbox<F, T, T>(f, s, r.alpha, one);
    else pos_sbox<F, T, 1>(f, s, r.alpha, one);
    u64 n[T];
#pragma unroll
    for (int k = 0; k < T; k++) {
      u64 acc = f.mul_tw(s[0], pos_const(mds + k * T));
#pragma unroll
      for (int j = 1; j < T; j++) acc = f.add(acc, f.mul_tw(s[j], pos_const(mds + k * T + j)));
      n[k] = acc;
    }
#pragma unroll
    for (int k = 0; k < T; k++) s[k] = n[k];
  }
}

// One row of ronk_poseidon_sponge_u64: a fresh sponge of capacity T − rate absorbs in[0, len), starts squeezing and
// squeezes n_out words into out (plain residues in and out).  Absorbing any split of the input, then squeezing any split
// of the output, gives the same words as one absorb and one squeeze, so the row's state machine reduces to: add each
// rate-chunk of the input (the last one possibly short) into state[capacity ..] and permute after it; then read rate
// words at a time from state[capacity ..], permuting between chunks.  len == 0 permutes nothing before the first squeeze
// (start_squeezing permutes only when absorb_index != 0, sponge.rs:198-213).
// With rate = T, len = n_out = T this is one permutation of the row in[0, T) into out[0, T) (in may be out): the
// zero state plus the input is the input.  So ronk_poseidon_permute_u64 runs this routine too, and the permutation
// has one call site.
template <class F, int T>
RONK_DEV void pos_sponge_row(const F& f, const PosRounds& r, const u64* rc, const u64* mds, u32 rate, const u64* in,
                             u64 len, u64* out, u64 n_out) {
  const u64 one = f.to_tw(1);
  const int cap = T - (int)rate;
  u64 s[T];
#pragma unroll
  for (int k = 0; k < T; k++) s[k] = 0;
  u64 c = 0, o = 0;  // words absorbed, words squeezed
  for (;;) {
    if (c < len) {
      const u64 left = len - c;
#pragma unroll
      for (int k = 0; k < T; k++)
        if (k >= cap && (u64)(k - cap) < left) s[k] = f.add(s[k], f.to_tw(in[c + (k - cap)]));
      c += rate;
    } else {
      const u64 left = n_out > o ? n_out - o : 0;
#pragma unroll
      for (int k = 0; k < T; k++)
        if (k >= cap && (u64)(k - cap) < left) out[o + (k - cap)] = pos_from_tw(f, s[k]);
      o += rate;
      if (o >= n_out) return;
    }
    pos_permute<F, T>(f, s, r, rc, mds, one);
  }
}

}  // namespace ronk
