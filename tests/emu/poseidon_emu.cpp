// poseidon_emu.cpp — TEST INFRASTRUCTURE: compiles the row routine of ronk_poseidon_permute_u64 / ronk_poseidon_sponge_u64
// (ronkathon_b200/csrc/poseidon.cuh) for the host, on both field policies, so the CPU test tier can check it against
// tests/poseidon_oracle.c without a GPU.  What poseidon_rows_kernel does per CTA is repeated here: the constants are
// taken into the policy's twiddle form, and every row runs pos_sponge_row.  Never linked into libronk_b200.so.
#include <cstdint>
#include <vector>

#include "../../ronkathon_b200/csrc/poseidon.cuh"

using namespace ronk;

template <class F, int T>
static void rows(const F& f, const PosRounds& r, const uint64_t* rc_in, const uint64_t* mds_in, uint32_t rate,
                 const uint64_t* in, uint64_t len, uint64_t* out, uint64_t n_out, uint64_t batch) {
  std::vector<u64> rc(r.rounds * T), mds(r.rounds ? T * T : 0);
  for (size_t i = 0; i < rc.size(); i++) rc[i] = f.to_tw(rc_in[i]);
  for (size_t i = 0; i < mds.size(); i++) mds[i] = f.to_tw(mds_in[i]);
  for (uint64_t y = 0; y < batch; y++) pos_sponge_row<F, T>(f, r, rc.data(), mds.data(), rate, in + y * len, len, out + y * n_out, n_out);
}

template <class F>
static int dispatch(const F& f, uint32_t width, const PosRounds& r, const uint64_t* rc, const uint64_t* mds, uint32_t rate,
                    const uint64_t* in, uint64_t len, uint64_t* out, uint64_t n_out, uint64_t batch) {
  switch (width) {
#define RONK_EMU_CASE(T) case T: rows<F, T>(f, r, rc, mds, rate, in, len, out, n_out, batch); return 0;
    RONK_EMU_CASE(2) RONK_EMU_CASE(3) RONK_EMU_CASE(4) RONK_EMU_CASE(5) RONK_EMU_CASE(6) RONK_EMU_CASE(7) RONK_EMU_CASE(8)
    RONK_EMU_CASE(9) RONK_EMU_CASE(10) RONK_EMU_CASE(11) RONK_EMU_CASE(12) RONK_EMU_CASE(13) RONK_EMU_CASE(14)
    RONK_EMU_CASE(15) RONK_EMU_CASE(16)
#undef RONK_EMU_CASE
    default: return 1;
  }
}

extern "C" {

// The sponge rows of ronk_poseidon_sponge_u64 (rate < width) or, with rate = len = n_out = width and in == out, the
// permutation of ronk_poseidon_permute_u64.  goldilocks: the Goldilocks policy (p must be Goldilocks), else MontField.
// Returns 1 for a width outside 2 … 16.
int emu_poseidon_rows(int goldilocks, uint64_t p, uint32_t width, uint64_t alpha, uint32_t num_f, uint32_t num_p,
                      const uint64_t* rc, const uint64_t* mds, uint32_t rate, const uint64_t* in, uint64_t len, uint64_t* out,
                      uint64_t n_out, uint64_t batch) {
  const PosRounds r = {num_f + num_p, num_f / 2, num_p + num_f / 2, alpha};
  if (goldilocks) return dispatch(GoldilocksField{}, width, r, rc, mds, rate, in, len, out, n_out, batch);
  return dispatch(h_mont_field(p), width, r, rc, mds, rate, in, len, out, n_out, batch);
}

}  // extern "C"
