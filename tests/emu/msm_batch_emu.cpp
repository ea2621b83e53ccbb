// msm_batch_emu.cpp — TEST INFRASTRUCTURE: compiles the term test and the scalar check of ronk_msm_pluto_ext_batch's
// kernels (coord_term, scalar4_over in ronkathon_b200/csrc/msm_curve.cuh) for the host, so the CPU test tier can check
// them against the group tables and the oracle without a GPU.  Never linked into libronk_b200.so.
#include <cstdint>

#include "../../ronkathon_b200/csrc/msm_curve.cuh"

using namespace ronk;

extern "C" {

int emu_group_tables(uint32_t* bintab, uint32_t* pttab) { return build_group_tables(bintab, pttab) ? 1 : 0; }

// coord_term over n packed points: on[i] = the point is canonical and on the curve, a[i] / b[i] = its group coordinates
// as msm_coord_pack_kernel stores them (0 when not on the curve)
void emu_coord_terms(const uint32_t* bintab, const uint32_t* points, uint64_t n, uint8_t* on, uint8_t* a, uint8_t* b) {
  for (uint64_t i = 0; i < n; i++) {
    u32 e;
    const bool ok = coord_term(points[i], bintab, e);
    on[i] = ok ? 1 : 0;
    a[i] = ok ? (uint8_t)((e >> 16) & 0xFF) : 0;
    b[i] = ok ? (uint8_t)(e >> 24) : 0;
  }
}

// scalar4_over over n words of four packed scalars: out[i] = 1 when some byte of words[i] is ≥ 17
void emu_scalar4_over(const uint32_t* words, uint64_t n, uint8_t* out) {
  for (uint64_t i = 0; i < n; i++) out[i] = scalar4_over(words[i]) ? 1 : 0;
}

}  // extern "C"
