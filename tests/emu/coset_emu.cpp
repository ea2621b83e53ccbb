// coset_emu.cpp — TEST INFRASTRUCTURE: compiles the coset-hooked phases of the transform kernels
// (ronkathon_b200/csrc/ntt_kernel.cuh, ntt3_kernel.cuh, on field.cuh) for the host and runs a coset transform thread by
// thread the way ntt.cu launches it: the tile kernels' COSET load (forward) and store (inverse) phases, and the 256-point
// tile passes' COSET round 0 of pass 1 and round 1 of pass 3.  The factor tables are built as coset_table_kernel builds
// them.  Never linked into libronk_b200.so.
#include <cstdint>
#include <vector>

#include "../../ronkathon_b200/csrc/ntt3_kernel.cuh"
#include "../../ronkathon_b200/csrc/ntt_kernel.cuh"

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

template <class F>
std::vector<u64> table(const F& f, u64 w, u64 s, u64 count) {  // pow_table_kernel
  std::vector<u64> t(count);
  for (u64 i = 0; i < count; i++) t[i] = f.to_tw(f.mul(field_pow(f, w, i), s));
  return t;
}

std::vector<u64> table2d(const std::vector<u64>& tw1d, u32 log_m, bool inverse) {  // tw2d_gather_kernel
  u32 off[4];
  const u32 words = ntt_tw2d_layout(log_m, off);
  std::vector<u64> out(words ? words : 2, 0);
  for (u32 w = 0; w < words; w++) {
    bool valid;
    const u32 idx = ntt_tw2d_source(log_m, w, inverse, &valid);
    out[w] = valid ? tw1d[idx] : 0;
  }
  return out;
}

// coset_table_kernel: c^i for i < 2^h, then c^(i·2^h) for i < 2^(log_n - h), twiddle form
template <class F>
std::vector<u64> coset_tables(const F& f, u64 c, u32 log_n) {
  const u32 h = (log_n + 1) / 2, lo = 1u << h;
  std::vector<u64> t(lo + (1u << (log_n - h)));
  for (u32 i = 0; i < t.size(); i++) t[i] = f.to_tw(field_pow(f, c, i < lo ? (u64)i : (u64)(i - lo) << h));
  return t;
}

// ntt_tile_kernel<…, COSET> phase by phase: the hooked load (forward) or store (inverse) where `coset` is set, the plain
// phases elsewhere, each in the formulation RONK_LOAD_V0_MASK / RONK_STORE_V0_MASK choose for the mode
template <class F, int MODE, bool INV>
void run_tiles(const F& f, const NttTileArgs& A, u64 tiles, bool coset) {
  const u32 T = 1u << A.tile_log, nthr = (T / 32 >= 32) ? T / 32 : 32;
  constexpr bool load_v0 = (RONK_LOAD_V0_MASK >> MODE) & 1, store_v0 = (RONK_STORE_V0_MASK >> MODE) & 1;
  std::vector<u64> smem(T);
  for (u64 tile = 0; tile < tiles; tile++) {
    for (u32 t = 0; t < nthr; t++) {
      if constexpr (!INV && MODE != MODE_PASS2) {
        if (coset) {
          if (load_v0) ntt_load_phase_v0<F, MODE, false, true>(smem.data(), A, (u32)tile, t, nthr, &f);
          else ntt_load_phase<F, MODE, false, true>(smem.data(), A, (u32)tile, t, nthr, &f);
          continue;
        }
      }
      if (load_v0) ntt_load_phase_v0<F, MODE>(smem.data(), A, (u32)tile, t, nthr);
      else ntt_load_phase<F, MODE>(smem.data(), A, (u32)tile, t, nthr);
    }
    u32 nst, wb, lcur;
    for (u32 r = 0; ntt_round_plan(A, r, &nst, &wb, &lcur); r++)
      for (u32 t = 0; t < nthr; t++) ntt_round_dispatch<F, INV>(f, smem.data(), A.tw_tile, A, nst, wb, lcur, t, nthr);
    for (u32 t = 0; t < nthr; t++) {
      if constexpr (INV && MODE != MODE_PASS1 && store_v0) {
        if (coset) {
          ntt_store_phase_v0<F, MODE, INV, false, false, true>(f, smem.data(), A, (u32)tile, t, nthr);
          continue;
        }
      }
      if (store_v0) ntt_store_phase_v0<F, MODE, INV>(f, smem.data(), A, (u32)tile, t, nthr);
      else ntt_store_phase<F, MODE, INV>(f, smem.data(), A, (u32)tile, t, nthr);
    }
  }
}

void set_coset(NttTileArgs& A, const std::vector<u64>& ct, u32 log_n) {
  A.coset_h = (log_n + 1) / 2;
  A.coset_lo = ct.data();
  A.coset_hi = ct.data() + (1u << A.coset_h);
}

// run_ntt() of ntt.cu with a coset table: single tile up to 2^13, else the pass pair (preferred tiles 2^14 / 2^13)
template <class F, bool INV>
void run(const F& f, u64 p, u64 g, bool gl, u64* data, u32 log_n, u32 batch, u64 shift) {
  const u64 n = (u64)1 << log_n, w = h_powmod(g, (p - 1) / n, p), ninv = h_powmod(n % p, p - 2, p);
  const u64 scale = gl ? ninv : h_mulmod(ninv, (u64)((((unsigned __int128)1) << 64) % p), p);
  const std::vector<u64> ct = coset_tables(f, INV ? h_powmod(shift, p - 2, p) : shift, log_n);
  const NttShape sh = ntt_shape(log_n);
  u64 tiles = 0;
  if (!sh.two_pass) {
    const auto tw = table2d(table(f, w, 1, n), log_n, INV);
    NttTileArgs A = ntt_args_single(data, nullptr, tw.data(), scale, log_n, (u64)batch << log_n, INV, 12, &tiles);
    set_coset(A, ct, log_n);
    run_tiles<F, MODE_SINGLE, INV>(f, A, tiles, true);
    return;
  }
  const u64 n1 = (u64)1 << sh.log_n1, n2 = (u64)1 << sh.log_n2;
  const auto tw1 = table(f, h_powmod(w, n2, p), 1, n1), tw2 = table(f, h_powmod(w, n1, p), 1, n2);
  const auto tw_lo = table(f, w, 1, n1), tw_hi_inv = table(f, h_powmod(w, n1, p), ninv, n2);
  const auto tw1_2d = table2d(tw1, sh.log_n1, INV), tw2_2d = table2d(tw2, sh.log_n2, INV);
  std::vector<u64> ws((size_t)batch << log_n);
  u32 tile1, tile2;
  ntt_pass_tiles(log_n, 14, 13, &tile1, &tile2);
  NttTileArgs A1 = ntt_args_pass1(data, ws.data(), tw1_2d.data(), tw_lo.data(), INV ? tw_hi_inv.data() : tw2.data(),
                                  tw2.data(), log_n, batch, tile1, tile2, &tiles);
  set_coset(A1, ct, log_n);
  run_tiles<F, MODE_PASS1, INV>(f, A1, tiles, !INV);
  NttTileArgs A2 = ntt_args_pass2(ws.data(), data, nullptr, tw2_2d.data(), log_n, batch, tile2, &tiles);
  set_coset(A2, ct, log_n);
  run_tiles<F, MODE_PASS2, INV>(f, A2, tiles, INV);
}

// ntt3_kernel<…, COSET> over every tile, 128 threads with two groups each
template <int PASS, bool INV, int LOGN, bool COSET>
void run_pass3(const GoldilocksField& f, const Ntt3Args& A) {
  std::vector<u64> smem(N3_TILE_WORDS);
  for (u32 tile = 0; tile < A.batch * (1u << (LOGN - 12)); tile++) {
    u64 in_base, in_row, in_col, out_base, out_row;
    u32 m_base;
    n3_tile_geometry<PASS, LOGN>(tile, &in_base, &in_row, &in_col, &out_base, &out_row, &m_base);
    for (u32 t = 0; t < N3_THREADS; t++)
      n3_round0<GoldilocksField, PASS, INV, false, 2, PASS == 1 ? n3_log_r0(LOGN) : 4, 0, COSET && !INV && PASS == 1>(
          f, smem.data(), A, in_base, in_row, in_col, t, (u64)1 << LOGN);
    for (u32 t = 0; t < N3_THREADS; t++)
      n3_round1<GoldilocksField, PASS, INV, false, LOGN, 2, COSET && INV && PASS == 3>(f, smem.data(), A, out_base, out_row, m_base, t);
  }
}

// run_ntt3<…, COSET> of ntt.cu: Goldilocks with g = 7, the stepped pass-1 twiddles
template <bool INV, int LOGN>
void run3(u64* data, u32 batch, u64 shift) {
  const GoldilocksField f;
  const u64 p = GL_P, n = (u64)1 << LOGN;
  const u64 wf = h_powmod(7, (p - 1) / n, p), w = INV ? h_powmod(wf, p - 2, p) : wf;
  const u32 lo = (u32)(LOGN + 1) / 2u;
  const auto tw256 = table(f, h_powmod(w, n >> 8, p), 1, 256);
  const auto tw_lo = table(f, wf, 1, 1u << lo), tw_hi = table(f, h_powmod(wf, (u64)1 << lo, p), 1, 1u << (LOGN - lo));
  const u64 ninv = INV ? h_powmod(n % p, p - 2, p) : 1, w16 = h_powmod(w, n >> 16, p);
  std::vector<u64> t2(65536);
  for (u32 i = 0; i < 65536; i++) t2[i] = f.to_tw(f.mul(field_pow(f, w16, (u64)((i >> 8) * (i & 255u))), ninv));
  const std::vector<u64> ct = coset_tables(f, INV ? h_powmod(shift, p - 2, p) : shift, LOGN);
  std::vector<u64> ws((size_t)batch << LOGN);
  Ntt3Args A = {};
  A.tw256 = tw256.data(); A.tw_lo = tw_lo.data(); A.tw_hi = tw_hi.data(); A.t2 = t2.data(); A.batch = batch;
  A.src_len = A.dst_len = NTT_UNBOUNDED; A.mul_mask = ~0ULL; A.coset = ct.data();
  A.src = data; A.dst = ws.data();
  run_pass3<1, INV, LOGN, true>(f, A);
  A.src = ws.data();
  run_pass3<2, INV, LOGN, false>(f, A);
  A.dst = data;
  run_pass3<3, INV, LOGN, true>(f, A);
}

}  // namespace

extern "C" {

// ronk_ntt_coset_u64 on the tile kernels (log_n ≥ 1, n ≤ 2^26, shift ≠ 0), on host memory.  Returns 1 if 2^log_n does
// not divide p - 1.
int emu_ntt_coset(uint64_t p, uint64_t g, uint64_t* data, uint32_t log_n, uint32_t batch, uint64_t shift, int inverse) {
  if (log_n == 0 || log_n > 26 || (p - 1) % ((u64)1 << log_n) != 0) return 1;
  if (p == GL_P && g == 7) {
    GoldilocksField f;
    if (inverse) run<GoldilocksField, true>(f, p, g, true, data, log_n, batch, shift);
    else run<GoldilocksField, false>(f, p, g, true, data, log_n, batch, shift);
    return 0;
  }
  const MontField f = make_mont(p, g, inverse != 0);
  if (inverse) run<MontField, true>(f, p, g, false, data, log_n, batch, shift);
  else run<MontField, false>(f, p, g, false, data, log_n, batch, shift);
  return 0;
}

// ronk_ntt_coset_u64 for Goldilocks with g = 7 at 2^21 … 2^24 through the 256-point-tile passes, on host memory
int emu_ntt3_coset(uint64_t* data, uint32_t log_n, uint32_t batch, uint64_t shift, int inverse) {
  switch (log_n * 2 + (inverse ? 1 : 0)) {
    case 42: run3<false, 21>(data, batch, shift); return 0;
    case 43: run3<true, 21>(data, batch, shift); return 0;
    case 44: run3<false, 22>(data, batch, shift); return 0;
    case 45: run3<true, 22>(data, batch, shift); return 0;
    case 46: run3<false, 23>(data, batch, shift); return 0;
    case 47: run3<true, 23>(data, batch, shift); return 0;
    case 48: run3<false, 24>(data, batch, shift); return 0;
    case 49: run3<true, 24>(data, batch, shift); return 0;
    default: return 1;
  }
}

}  // extern "C"
