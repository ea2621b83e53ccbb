// batch_inv.cuh — Montgomery's batch inversion of the K values one thread holds: one Fermat inversion and about three
// multiplies per value instead of one inversion (about 64 squarings) each.  __host__ __device__ (RONK_HD), so that
// tests/emu/bary_emu.cpp runs this very code on the CPU under both field policies.
#pragma once
#include "field.cuh"

namespace ronk {

// Values per thread in the barycentric kernels (poly_bary.cu): one Fermat inversion per 16 values.
constexpr int BI_K = 16;

// Hands st(k, v_k^-1) for the K values v_k = ld(k), k < K.  A zero value is skipped: it counts as 1 in the running
// product and its "inverse" is 0.  ld is called twice per index (forward and backward sweep), so the values stay where
// ld reads them (shared memory in the kernels) and only the K exclusive prefix products live in registers.  st(k) is
// called after the last ld(k), in decreasing k, so st may overwrite the value ld(k) read.  Plain residues in and out.
template <int K, class F, class Ld, class St>
RONK_HD void batch_invert(const F& f, Ld&& ld, St&& st) {
  u64 pre[K];  // pre[k] = Π_{k' < k, v_k' != 0} v_k'
  u64 run = 1 % f.modulus();
#pragma unroll
  for (int k = 0; k < K; k++) {
    pre[k] = run;
    const u64 v = ld(k);
    if (v) run = f.mul(run, v);
  }
  u64 inv = field_pow(f, run, f.modulus() - 2);  // (Π v_k)^-1 over the nonzero values
#pragma unroll
  for (int k = K - 1; k >= 0; k--) {
    const u64 v = ld(k);
    st(k, v ? f.mul(inv, pre[k]) : (u64)0);
    if (v) inv = f.mul(inv, v);  // now (Π_{k' < k} v_k')^-1
  }
}

}  // namespace ronk
