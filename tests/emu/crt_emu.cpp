// crt_emu.cpp — the multi-modular product's host-and-device code (ronkathon_b200/csrc/crt.cuh) compiled for the CPU:
// the prime count, Garner's constants and the per-coefficient Garner step of crt_combine_kernel, and the reduction of
// crt_reduce_kernel.  Test infrastructure (tests/test_crt_mul_model.py); the library never runs these on the host.
#include <cstdint>

#include "../../ronkathon_b200/csrc/crt.cuh"

using namespace ronk;

extern "C" {

int emu_crt_prime_count(uint64_t p, uint64_t m) { return crt_prime_count(p, m); }

// out[0..3) = q_i, out[3..6) = the generators
void emu_crt_primes(uint64_t* out) {
  for (int i = 0; i < kCrtPrimes; i++) {
    out[i] = kCrtQ[i];
    out[kCrtPrimes + i] = kCrtG[i];
  }
}

// out = {q1^-1 mod q2, (q1·q2)^-1 mod q3, q1·(q1·q2)^-1 mod q3, 1 mod p, q1 mod p, q1·q2 mod p}, each taken out of the
// form crt_combine_kernel holds it in (Montgomery form, or p's twiddle form) by one multiplication by 1.
void emu_crt_consts(uint64_t p, uint64_t* out) {
  auto plain = [&](const auto& f) {
    const CrtConsts k = crt_consts(f);
    out[0] = k.m2.redc_mul(k.inv1, 1);
    out[1] = k.m3.redc_mul(k.inv12, 1);
    out[2] = k.m3.redc_mul(k.q1inv12, 1);
    out[3] = f.mul_tw(1, k.one_tw);
    out[4] = f.mul_tw(1, k.q1_tw);
    out[5] = f.mul_tw(1, k.q12_tw);
  };
  if (p == GL_P) plain(GoldilocksField());
  else plain(h_mont_field(p));
}

// out[i] = crt_garner<k>(p's policy, c1[i], c2[i], c3[i]): the policy crt_mul_device passes (Goldilocks for GL_P, else
// Montgomery).
int emu_crt_garner(uint64_t p, int k, const uint64_t* c1, const uint64_t* c2, const uint64_t* c3, uint64_t* out, uint64_t n) {
  auto run = [&](const auto& f) {
    const CrtConsts cs = crt_consts(f);
    for (uint64_t i = 0; i < n; i++) {
      if (k == 1) out[i] = crt_garner<1>(f, cs, c1[i], 0, 0);
      else if (k == 2) out[i] = crt_garner<2>(f, cs, c1[i], c2[i], 0);
      else out[i] = crt_garner<3>(f, cs, c1[i], c2[i], c3[i]);
    }
  };
  if (k < 1 || k > 3) return -1;
  if (p == GL_P) run(GoldilocksField());
  else run(h_mont_field(p));
  return 0;
}

void emu_crt_below(uint64_t q, const uint64_t* x, uint64_t* out, uint64_t n) {
  for (uint64_t i = 0; i < n; i++) out[i] = crt_below(x[i], q);
}

}  // extern "C"
