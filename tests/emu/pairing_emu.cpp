// pairing_emu.cpp — TEST INFRASTRUCTURE: compiles the Miller loop, the pairing-table entry and the per-row check of
// ronk_pairing_pluto_ext / ronk_kzg_check_pluto_ext_batch (ronkathon_b200/csrc/pairing.cuh) for the host, so the CPU test
// tier can check them against tests/pairing_oracle.c without a GPU.  Never linked into libronk_b200.so.
#include <cstdint>

#include "../../ronkathon_b200/csrc/pairing.cuh"

using namespace ronk;

extern "C" {

int emu_group_tables(uint32_t* bintab, uint32_t* pttab) { return build_group_tables(bintab, pttab) ? 1 : 0; }

// What pairing_table_kernel writes: mu[17] and T[289²], one entry per pair as the kernel's threads compute them.
void emu_pairing_table(const uint32_t* pttab, uint16_t* mu, uint8_t* T) {
  mu17_list(mu);
  for (u32 i = 0; i < PAIR_TAB; i++) T[i] = pairing_entry(i / E17_PTS, i % E17_PTS, pttab, mu);
}

// tate_pairing on two packed points: 1 and out = (c0, c1), or 0 where the Miller loop panics
int emu_tate(uint32_t p, uint32_t q, uint8_t* out) {
  Gf v;
  if (!tate_pairing(pt_unpack(p), pt_unpack(q), v)) return 0;
  out[0] = (uint8_t)v.c0;
  out[1] = (uint8_t)v.c1;
  return 1;
}

// P − s·Q in group coordinates, as the check forms B and C′: the packed point pttab[102·a + b], or 0 (with *out
// untouched) when P or Q is rejected by point_coords
int emu_sub_smul(const uint32_t* bintab, const uint32_t* pttab, uint32_t p, uint32_t s, uint32_t q, uint32_t* out) {
  u32 pa, pb, qa, qb;
  if (!point_coords(p, bintab, pa, pb) || !point_coords(q, bintab, qa, qb)) return 0;
  *out = pttab[MSM_EXP * coord_sub_smul(pa, s, qa) + coord_sub_smul(pb, s, qb)];
  return 1;
}

// kzg_check_kernel's rows on the host: ok[i] and bad[i] (1 where the kernel raises its flag for the row)
void emu_kzg_check(const uint32_t* bintab, const uint8_t* T, const uint32_t* c, const uint32_t* q, const uint8_t* z,
                   const uint8_t* v, uint64_t n, uint32_t g1, uint32_t g2, uint8_t* ok, uint8_t* bad) {
  u32 g1a, g1b, g2a, g2b, gena, genb;
  const u32 consts = (u32)!point_coords(g1, bintab, g1a, g1b) | (u32)!point_coords(g2, bintab, g2a, g2b);
  point_coords(PLUTO_EXT_GEN, bintab, gena, genb);
  for (uint64_t i = 0; i < n; i++) {
    u32 b = consts;
    ok[i] = kzg_check_row(c[i], q[i], z[i], v[i], g1a, g1b, g2a, g2b, gena, genb, e17_index(gena, genb), bintab, T, b);
    bad[i] = b ? 1 : 0;
  }
}

}  // extern "C"
