// polymul_emu.cpp — TEST INFRASTRUCTURE: compiles the fused batched product's device phases
// (ronkathon_b200/csrc/polymul_kernel.cuh, on field.cuh and ntt_kernel.cuh) for the host and runs polymul_fused_kernel's
// data flow tile by tile, thread by thread, so the CPU test tier can check it against the oracle.  Never linked into
// libronk_b200.so.
#include <cstdint>
#include <vector>

#include "../../ronkathon_b200/csrc/polymul_kernel.cuh"

using namespace ronk;

namespace {

MontField make_mont(u64 p, u64 g, bool inverse) {  // mirrors make_mont_field() in ntt.cu
  MontField f = h_mont_field(p);
  const u64 r1 = f.w16t[0];
  u32 k = 0;
  while (k < 4 && ((p - 1) >> k) % 2 == 0) k++;
  if (k) {
    u64 w = h_powmod(g, (p - 1) >> k, p);
    if (inverse) w = h_powmod(w, ((u64)1 << k) - 1, p);
    const int stride = 16 >> k;
    for (int e = 0; e < 8; e++)
      if (e % stride == 0) f.w16t[e] = h_mulmod(h_powmod(w, e / stride, p), r1, p);
  }
  return f;
}

// the N-point plan's per-round table of one direction, as build_plan() + tw2d_gather_kernel make it
template <class F>
std::vector<u64> table2d(const F& f, u64 p, u64 g, u32 log_n, bool inverse) {
  const u64 n = (u64)1 << log_n, w = h_powmod(g, (p - 1) / n, p);
  std::vector<u64> tw1d(n);
  for (u64 i = 0; i < n; i++) tw1d[i] = f.to_tw(field_pow(f, w, i));
  u32 off[4];
  const u32 words = ntt_tw2d_layout(log_n, off);
  std::vector<u64> out(words ? words : 2, 0);
  for (u32 w2 = 0; w2 < words; w2++) {
    bool valid;
    const u32 idx = ntt_tw2d_source(log_n, w2, inverse, &valid);
    out[w2] = valid ? tw1d[idx] : 0;
  }
  return out;
}

// polymul_fused_kernel, one CTA after the other; the barriers become the boundaries between the thread loops
template <class F>
void run_fused(const F& ff, const F& fi, u64 p, u64 g, bool gl, const u64* a, u32 da, const u64* b, u32 db, bool shared,
               u64 batch, u64* c, u32 log_n) {
  const u64 n = (u64)1 << log_n, ninv = h_powmod(n % p, p - 2, p);
  const u64 scale = gl ? ninv : h_mulmod(ninv, (u64)((((unsigned __int128)1) << 64) % p), p);
  const std::vector<u64> twf = table2d(ff, p, g, log_n, false), twi = table2d(ff, p, g, log_n, true);
  u64 tiles = 0;
  const PolyMulArgs A = polymul_args(a, da, b, db, shared, batch, c, log_n, twf.data(), twi.data(), scale, &tiles);
  const u32 T = 1u << PM_TILE_LOG, nthr = PM_THREADS;
  std::vector<u64> sa(T), sb(T);
  for (u64 tile = 0; tile < tiles; tile++) {
    for (u32 t = 0; t < nthr; t++) {
      pm_load(sa.data(), A.a, A.da, A.da, A, tile, t, nthr);
      pm_load(sb.data(), A.b, A.db, A.b_stride, A, tile, t, nthr);
    }
    const u32 rounds = pm_round_count(A);
    for (u32 r = 0; r < rounds; r++)
      for (u32 t = 0; t < nthr; t++) {
        pm_round<F, false>(ff, sa.data(), twf.data(), A, r, t, nthr);
        pm_round<F, false>(ff, sb.data(), twf.data(), A, r, t, nthr);
      }
    for (u32 t = 0; t < nthr; t++) pm_pointwise(ff, sa.data(), sb.data(), A, t, nthr);
    for (u32 t = 0; t < nthr; t++) pm_bitrev(sa.data(), sb.data(), A, t, nthr);
    for (u32 r = 0; r < rounds; r++)
      for (u32 t = 0; t < nthr; t++) pm_round<F, true>(fi, sb.data(), twi.data(), A, r, t, nthr);
    for (u32 t = 0; t < nthr; t++) pm_store(fi, sb.data(), A, tile, t, nthr);
  }
}

}  // namespace

extern "C" {

// The fused kernel's data flow over `batch` rows: c (batch × (da + db - 1)) = a (batch × da) · b (batch × db, or db
// words when shared).  Returns 1 where the fused kernel does not apply.
int emu_poly_mul_fused(uint64_t p, uint64_t g, const uint64_t* a, uint32_t da, const uint64_t* b, uint32_t db, int shared,
                       uint64_t batch, uint64_t* c) {
  const u32 L = da + db - 1;
  u32 log_n = 0;
  while ((1u << log_n) < L) log_n++;
  if (!g || log_n == 0 || log_n > PM_MAX_LOG || (p - 1) % ((u64)1 << log_n) != 0) return 1;
  if (p == GL_P && g == 7) {
    GoldilocksField f;
    run_fused(f, f, p, g, true, a, da, b, db, shared != 0, batch, c, log_n);
    return 0;
  }
  run_fused(make_mont(p, g, false), make_mont(p, g, true), p, g, false, a, da, b, db, shared != 0, batch, c, log_n);
  return 0;
}

// Bank-conflict audit of the fused kernel's own shared-memory access patterns, for rows of N = 2^log_n words: the worst
// number of lanes of one half-warp (16 lanes, 16 eight-byte banks) on one bank.  phase 0: the load's row-strided
// scatter of d-word rows; 1: the bit-reversal permutation's writes; 2: the store's un-bit-reversing reads of d-word rows.
int emu_polymul_worst_conflict(uint32_t log_n, uint32_t d, int phase) {
  const u32 T = 1u << PM_TILE_LOG, M = (1u << log_n) - 1u, rows = T >> log_n, nthr = PM_THREADS;
  const u32 run = phase == 1 ? T : rows * d;
  int worst = 1;
  for (u32 w0 = 0; w0 < run; w0 += nthr)
    for (u32 hw = 0; hw < nthr; hw += 16) {
      int cnt[16] = {0};
      for (u32 l = 0; l < 16; l++) {
        const u32 w = w0 + hw + l;
        if (w >= run) continue;
        u32 e;
        if (phase == 1) {
          e = (w & ~M) | bitrev(w & M, log_n);
        } else {
          const u32 j = w / d, k = w - j * d;
          e = (j << log_n) | (phase == 0 ? k : bitrev(k, log_n));
        }
        cnt[swz(e) & 15]++;
      }
      for (int k = 0; k < 16; k++) worst = cnt[k] > worst ? cnt[k] : worst;
    }
  return worst;
}

}  // extern "C"
