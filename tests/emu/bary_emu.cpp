// bary_emu.cpp — TEST INFRASTRUCTURE: compiles batch_invert (ronkathon_b200/csrc/batch_inv.cuh, on field.cuh) for the host
// and runs it the way the barycentric kernels (poly_bary.cu) do: every thread inverts BI_K values in place, chunk by chunk.
// Never linked into libronk_b200.so.
#include <cstddef>
#include <cstdint>

#include "../../ronkathon_b200/csrc/batch_inv.cuh"

using namespace ronk;

namespace {

template <class F>
void run(const F& f, u64* v, size_t count) {
  for (size_t c = 0; c < count; c += BI_K)
    batch_invert<BI_K>(f, [&](int k) { return v[c + k]; }, [&](int k, u64 inv) { v[c + k] = inv; });
}

}  // namespace

extern "C" {

int emu_bi_k() { return BI_K; }

// v[i] ← v[i]^-1 (0 stays 0) in chunks of BI_K words; count must be a multiple of BI_K.  goldilocks != 0 runs the
// Goldilocks policy (p must be Goldilocks), otherwise the run-time Montgomery policy of p.
int emu_batch_invert(uint64_t p, int goldilocks, uint64_t* v, size_t count) {
  if (count % BI_K) return 1;
  if (goldilocks) {
    if (p != GL_P) return 1;
    run(GoldilocksField{}, v, count);
  } else {
    run(h_mont_field(p), v, count);
  }
  return 0;
}

}  // extern "C"
