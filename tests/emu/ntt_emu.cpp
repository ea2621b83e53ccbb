// ntt_emu.cpp — TEST INFRASTRUCTURE: compiles the product's kernel headers
// (ronkathon_b200/csrc/field.cuh, ntt_kernel.cuh) for the host and executes the tile phases thread by
// thread, so the CPU test tier can check the kernel's index maps, round schedule, twiddle tables and
// field arithmetic against the oracle without a GPU.  Never linked into libronk_b200.so and never
// used by the product path.
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../ronkathon_b200/csrc/ntt12_kernel.cuh"
#include "../../ronkathon_b200/csrc/ntt3_kernel.cuh"
#include "../../ronkathon_b200/csrc/ntt_kernel.cuh"

using namespace ronk;

namespace {

struct HostMont {
  MontField f;
};

MontField make_mont(u64 p, u64 g, bool inverse) {  // mirrors make_mont_field() in ntt.cu
  MontField f;
  f.p = p;
  f.pinv = h_inv64(p);
  const u64 r1 = (u64)((((unsigned __int128)1) << 64) % p);
  f.r2 = h_mulmod(r1, r1, p);
  for (int e = 0; e < 8; e++) f.w16t[e] = r1;
  if (g) {
    u32 k = 0;
    while (k < 4 && ((p - 1) >> k) % 2 == 0) k++;
    if (k) {
      u64 w = h_powmod(g, (p - 1) >> k, p);
      if (inverse) w = h_powmod(w, ((u64)1 << k) - 1, p);
      const int stride = 16 >> k;
      for (int e = 0; e < 8; e++)
        if (e % stride == 0) f.w16t[e] = h_mulmod(h_powmod(w, e / stride, p), r1, p);
    }
  }
  return f;
}

template <class F>
std::vector<u64> table(const F& f, u64 w, u64 s, u64 count) {  // pow_table_kernel
  std::vector<u64> t(count);
  for (u64 i = 0; i < count; i++) t[i] = f.to_tw(f.mul(field_pow(f, w, i), s));
  return t;
}

// mirrors tw2d_gather_kernel
std::vector<u64> table2d(const std::vector<u64>& tw1d, u32 log_m, bool inverse) {
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

// 0: the kernel's own per-mode choice (RONK_LOAD_V0_MASK / RONK_STORE_V0_MASK), 1: XOR-composed phases
// everywhere, 2: per-element ("v0") phases everywhere
int g_variant = 0;
// Optional n-word inter-pass twiddle table (NttTileArgs::tw_full) for emu_ntt: 0 = stepped twiddles.
int g_tw_table = 0;
bool use_v0(int mask, int mode) { return g_variant == 0 ? ((mask >> mode) & 1) != 0 : g_variant == 2; }

template <class F, int MODE, bool INV, bool BOUNDED, bool FMUL = false>
void run_tiles_b(const F& f, const NttTileArgs& A, u64 tiles) {
  const u32 T = 1u << A.tile_log, nthr = (T / 32 >= 32) ? T / 32 : 32;
  std::vector<u64> smem(T);
  for (u64 tile = 0; tile < tiles; tile++) {
    for (u32 t = 0; t < nthr; t++) {
      if (use_v0(RONK_LOAD_V0_MASK, MODE)) ntt_load_phase_v0<F, MODE, BOUNDED>(smem.data(), A, (u32)tile, t, nthr);
      else ntt_load_phase<F, MODE, BOUNDED>(smem.data(), A, (u32)tile, t, nthr);
    }
    u32 nst, wb, lcur;
    for (u32 r = 0; ntt_round_plan(A, r, &nst, &wb, &lcur); r++)
      for (u32 t = 0; t < nthr; t++) ntt_round_dispatch<F, INV>(f, smem.data(), A.tw_tile, A, nst, wb, lcur, t, nthr);
    for (u32 t = 0; t < nthr; t++) {
      if (use_v0(RONK_STORE_V0_MASK, MODE)) ntt_store_phase_v0<F, MODE, INV, BOUNDED, FMUL>(f, smem.data(), A, (u32)tile, t, nthr);
      else ntt_store_phase<F, MODE, INV, BOUNDED>(f, smem.data(), A, (u32)tile, t, nthr);
    }
  }
}

// The specialised 4096-point-per-tile kernel (ntt12_kernel.cuh), phase by phase like ntt12_kernel itself.
// g_fast12: 1 = take it wherever ntt.cu's launch_tile would (the product default), 0 = never.
int g_fast12 = 1;
u64 g_fast12_tiles = 0;  // tiles that went through it (so a test can tell the path was really taken)
template <class F, int MODE, bool INV, int LC, bool FMUL>
void run_tiles12(const F& f, const NttTileArgs& A, u64 tiles) {
  using L = N12<LC, MODE>;
  std::vector<u64x2> smem(L::TILE_SLOTS);
  for (u64 tile = 0; tile < tiles; tile++) {
    for (u32 t = 0; t < L::NTHR; t++) n12_round0_load<F, MODE, INV, LC>(f, smem.data(), A.tw_tile, A, (u32)tile, t);
    for (u32 t = 0; t < L::NTHR; t++) n12_round<F, MODE, INV, LC, 1>(f, smem.data(), A.tw_tile, t);
    if constexpr (MODE == MODE_PASS1) {
      for (u32 t = 0; t < L::NTHR; t++) n12_round<F, MODE, INV, LC, 2>(f, smem.data(), A.tw_tile, t);
      for (u32 t = 0; t < L::NTHR; t++) n12_store_pass1<F, LC>(f, smem.data(), A, (u32)tile, t);
    } else {
      // warp-local hand-over from round 1 to round 2: run it warp by warp to mirror the kernel's __syncwarp()
      for (u32 t = 0; t < L::NTHR; t++) n12_round2_store_pass2<F, INV, LC, FMUL>(f, smem.data(), A, (u32)tile, t);
    }
  }
  g_fast12_tiles += tiles;
}
template <class F, int MODE, bool INV>
bool try_tiles12(const F& f, const NttTileArgs& A, u64 tiles) {  // same dispatch as launch12() in ntt.cu
  if constexpr (MODE == MODE_SINGLE) {
    return false;
  } else {
    if (!g_fast12 || !ntt12_applicable(A, MODE) || (INV && (A.flags & NTT_FLAG_MUL))) return false;
    if constexpr (MODE == MODE_PASS1) {
      run_tiles12<F, MODE, INV, 2, false>(f, A, tiles);
    } else {
      if (!INV && (A.flags & NTT_FLAG_MUL)) run_tiles12<F, MODE, INV, 1, !INV>(f, A, tiles);
      else run_tiles12<F, MODE, INV, 1, false>(f, A, tiles);
    }
    return true;
  }
}

// src == nullptr: in place; otherwise the bounded out-of-place form of run_ntt() in ntt.cu (batch 1)
// same choice of instantiation as launch_tile_n() in ntt.cu
template <class F, int MODE, bool INV>
void run_tiles(const F& f, const NttTileArgs& A, u64 tiles) {
  if (try_tiles12<F, MODE, INV>(f, A, tiles)) return;
  const bool bounded = (MODE != MODE_PASS2 && A.src_len != NTT_UNBOUNDED) || (MODE != MODE_PASS1 && A.dst_len != NTT_UNBOUNDED);
  constexpr bool can_fmul = MODE == MODE_PASS2 && !INV;
  if (can_fmul && (A.flags & NTT_FLAG_MUL)) {
    if (bounded) run_tiles_b<F, MODE, INV, true, can_fmul>(f, A, tiles);
    else run_tiles_b<F, MODE, INV, false, can_fmul>(f, A, tiles);
    return;
  }
  if (bounded) run_tiles_b<F, MODE, INV, true>(f, A, tiles);
  else run_tiles_b<F, MODE, INV, false>(f, A, tiles);
}

template <class F, bool INV>
int run(const F& f, u64 p, u64 g, bool fast_gl, u64* data, const u64* mul, u32 log_n, u32 batch, u32 tile_cap,
        u32 pref1, u32 pref2, const u64* src = nullptr, u64 src_len = NTT_UNBOUNDED, u64 dst_len = NTT_UNBOUNDED) {
  if (!src) src = data;
  if (src_len >= ((u64)1 << log_n)) src_len = NTT_UNBOUNDED;
  if (dst_len >= ((u64)1 << log_n)) dst_len = NTT_UNBOUNDED;
  const u64 n = (u64)1 << log_n;
  const u64 w = h_powmod(g, (p - 1) / n, p);
  const u64 ninv = h_powmod(n % p, p - 2, p);
  const u64 scale = fast_gl ? ninv : h_mulmod(ninv, (u64)((((unsigned __int128)1) << 64) % p), p);
  const NttShape sh = ntt_shape(log_n);
  u64 tiles = 0;
  if (!sh.two_pass) {
    auto tw1d = table(f, w, 1, n);
    auto tw = table2d(tw1d, log_n, INV);
    NttTileArgs A = ntt_args_single(data, mul, tw.data(), scale, log_n, (u64)batch << log_n, INV, tile_cap, &tiles);
    A.src = src;
    A.src_len = src_len;
    A.dst_len = dst_len;
    run_tiles<F, MODE_SINGLE, INV>(f, A, tiles);
    return 0;
  }
  const u64 n1 = (u64)1 << sh.log_n1, n2 = (u64)1 << sh.log_n2;
  auto tw1 = table(f, h_powmod(w, n2, p), 1, n1);
  auto tw2 = table(f, h_powmod(w, n1, p), 1, n2);
  auto tw_lo = table(f, w, 1, n1);
  auto tw_hi_inv = table(f, h_powmod(w, n1, p), ninv, n2);
  std::vector<u64> ws((size_t)batch << log_n);
  u32 tile1, tile2;
  ntt_pass_tiles(log_n, pref1, pref2, &tile1, &tile2);
  auto tw1_2d = table2d(tw1, sh.log_n1, INV);
  auto tw2_2d = table2d(tw2, sh.log_n2, INV);
  NttTileArgs A1 = ntt_args_pass1(src, ws.data(), tw1_2d.data(), tw_lo.data(), INV ? tw_hi_inv.data() : tw2.data(),
                                  tw2.data(), log_n, batch, tile1, tile2, &tiles);
  A1.src_len = src_len;
  std::vector<u64> tw_full;
  if (g_tw_table) {  // mirrors interpass_table_kernel
    tw_full.resize(n);
    const u64* thi = INV ? tw_hi_inv.data() : tw2.data();
    for (u64 i = 0; i < n; i++) {
      const u32 k1_in = (u32)i & ((1u << A1.log_c2) - 1u);
      const u32 j2 = (u32)(i >> A1.log_c2) & ((1u << sh.log_n2) - 1u);
      const u32 k1 = ((u32)(i >> (sh.log_n2 + A1.log_c2)) << A1.log_c2) | k1_in;
      const u32 nmask = (log_n >= 32) ? 0xFFFFFFFFu : ((1u << log_n) - 1u);
      u32 ex = (j2 * k1) & nmask;
      if (INV) ex = (0u - ex) & nmask;
      tw_full[i] = f.mul_tw(tw_lo[ex & ((1u << A1.log_lo) - 1u)], thi[ex >> A1.log_lo]);
    }
    A1.tw_full = tw_full.data();
  }
  run_tiles<F, MODE_PASS1, INV>(f, A1, tiles);
  NttTileArgs A2 = ntt_args_pass2(ws.data(), data, mul, tw2_2d.data(), log_n, batch, tile2, &tiles);
  A2.dst_len = dst_len;
  run_tiles<F, MODE_PASS2, INV>(f, A2, tiles);
  return 0;
}

unsigned long long g_ntt3_mul_mask = ~0ULL;  // n - 1: the multiplier is ONE n-word table shared by the whole batch
int g_ntt3_ng1 = 0;  // 1: the 256-thread (one group per thread) flavour of the 2^16 / 2^20 tile passes
// The three-pass 2^24 transform (ntt3_kernel.cuh), phase by phase like ntt3_kernel; tables as run_ntt3() builds them.
template <class F, int PASS, bool INV, int LOGN, bool BOUNDED = false, int LI = 0>
void run_pass3(const F& f, const Ntt3Args& A) {
  std::vector<u64> smem(N3_TILE_WORDS);
  for (u32 tile = 0; tile < A.batch * (LOGN >= 21 ? (1u << (LOGN - 12)) : LOGN == 20 ? 256u : 16u); tile++) {
    u64 in_base, in_row, in_col, out_base, out_row;
    u32 m_base;
    n3_tile_geometry<PASS, LOGN, LI>(tile, &in_base, &in_row, &in_col, &out_base, &out_row, &m_base);
    if (g_ntt3_ng1 && LOGN != 24 && LI == 0) {   // one group per thread, 256 threads per tile (grids that do not fill the GPU)
      for (u32 t = 0; t < 2 * N3_THREADS; t++) n3_round0<F, PASS, INV, false, 1>(f, smem.data(), A, in_base, in_row, in_col, t);
      for (u32 t = 0; t < 2 * N3_THREADS; t++) n3_round1<F, PASS, INV, false, LOGN, 1>(f, smem.data(), A, out_base, out_row, m_base, t);
      continue;
    }
    for (u32 t = 0; t < N3_THREADS; t++)
      n3_round0<F, PASS, INV, BOUNDED && PASS == (LOGN >= 21 ? 1 : 2), 2, (PASS == 1 && LOGN >= 21) ? n3_log_r0(LOGN) : 4, LI>(
          f, smem.data(), A, in_base, in_row, in_col, t, (u64)1 << LOGN);
    for (u32 t = 0; t < N3_THREADS; t++) n3_round1<F, PASS, INV, BOUNDED, LOGN>(f, smem.data(), A, out_base, out_row, m_base, t);
  }
}
int g_ntt3_t1 = 0;  // 1: pass-1 twiddles from the n-word table
template <class F, bool INV, int LOGN, bool BOUNDED = false, int LI = 0>
int run3(const F& f, u64 p, u64 g, u64* data, const u64* mul, u32 batch, const u64* src = nullptr, u64 src_len = ~0ULL,
         u64 dst_len = ~0ULL) {
  if (LI > 0) {   // split transform n = 2^LI·2^LOGN: the register first pass with the n-point plan's two-level tables, in place
    const u32 log_n = LOGN + LI, lo = (log_n + 1) / 2;
    const u64 nn = (u64)1 << log_n;
    const u64 wn = h_powmod(g, (p - 1) / nn, p);
    auto o_lo = table(f, wn, 1, 1u << lo);
    auto o_hi = table(f, h_powmod(wn, (u64)1 << lo, p), 1, 1u << (log_n - lo));
    Ntt3Args P = {};
    P.src = data; P.dst = data; P.tw_lo = o_lo.data(); P.tw_hi = o_hi.data(); P.batch = batch;
    P.scale_tw = INV ? f.to_tw(h_powmod((u64)1 << LI, p - 2, p)) : 0;
    const u32 log_per = LOGN - (4 - LI);
    for (u64 i = 0; i < ((u64)batch << log_per); i++)
      n3p_columns<F, INV, LI>(f, P, (i >> log_per) << log_n, i & (((u64)1 << log_per) - 1), LOGN, lo);
    batch <<= LI;
  }
  const u64 n = (u64)1 << LOGN;
  u64 w = h_powmod(g, (p - 1) / n, p);
  const u64 wf = w;
  if (INV) w = h_powmod(w, p - 2, p);
  auto tw256 = table(f, h_powmod(w, n >> 8, p), 1, 256);
  std::vector<u64> tw_lo, tw_hi, t1;
  if (LOGN >= 21) {                                      // the plan's two-level tables, split at ceil(LOGN / 2)
    const u32 lo = (u32)(LOGN + 1) / 2u, mask = (1u << LOGN) - 1u;
    tw_lo = table(f, wf, 1, 1u << lo);                   // forward tables; the kernel negates exponents for INV
    tw_hi = table(f, h_powmod(wf, (u64)1 << lo, p), 1, 1u << (LOGN - lo));
    if (g_ntt3_t1) {                                     // mirrors ntt3_t1_kernel
      t1.resize(n);
      for (u64 i = 0; i < n; i++) {
        u32 ex = (u32)((i >> 16) * (i & 0xFFFFu)) & mask;
        if (INV) ex = (0u - ex) & mask;
        t1[i] = f.mul_tw(tw_lo[ex & ((1u << lo) - 1u)], tw_hi[ex >> lo]);
      }
    }
  }
  if (LOGN == 20) {                                      // the plan's 10 / 10 split of the two-level tables
    tw_lo = table(f, wf, 1, 1024);
    tw_hi = table(f, h_powmod(wf, 1024, p), 1, 1024);
    if (g_ntt3_t1) {                                     // mirrors ntt3_t1_20_kernel
      t1.resize(n);
      for (u64 i = 0; i < n; i++) {
        u32 ex = (u32)((i >> 4) * (i & 15u)) & 0xFFFFFu;
        if (INV) ex = (0u - ex) & 0xFFFFFu;
        t1[i] = f.mul_tw(tw_lo[ex & 1023u], tw_hi[ex >> 10]);
      }
    }
  }
  const u64 ninv = INV ? h_powmod(n % p, p - 2, p) : 1;
  std::vector<u64> t2(65536);
  const u64 w16 = h_powmod(w, n >> 16, p);
  for (u32 i = 0; i < 65536; i++) t2[i] = f.to_tw(f.mul(field_pow(f, w16, (u64)((i >> 8) * (i & 255u))), ninv));
  std::vector<u64> ws((size_t)batch << LOGN);
  Ntt3Args A = {};
  A.tw256 = tw256.data(); A.tw_lo = tw_lo.data(); A.tw_hi = tw_hi.data(); A.t2 = t2.data(); A.batch = batch;
  A.t1 = t1.empty() ? nullptr : t1.data();
  A.src_len = src_len; A.dst_len = dst_len; A.mul_mask = g_ntt3_mul_mask;
  A.src = src ? src : data; A.dst = ws.data();          // the flow of run_ntt3(): src → ws, ws in place, ws → data
  if constexpr (LOGN == 20) {                            // A1 src → data, A2 data → ws, C ws → data
    A.dst = data;
    run_pass3<F, 2, INV, 20>(f, A);
    A.src = data; A.dst = ws.data();
    run_pass3<F, 1, INV, 20>(f, A);
    A.src = ws.data(); A.dst = data; A.mul_src = mul; A.flags = mul ? NTT_FLAG_MUL : 0;
    for (u64 b = 0; b < batch; b++)
      for (u64 k2 = 0; k2 < 65536; k2++) n3c_point<F, INV>(f, A, b, k2);
    return 0;
  }
  if (LOGN >= 21) {
    run_pass3<F, 1, INV, LOGN, BOUNDED>(f, A);
    A.src = ws.data();
  }
  run_pass3<F, 2, INV, LOGN, BOUNDED && LOGN == 16>(f, A);
  A.src = ws.data(); A.dst = data; A.mul_src = mul; A.flags = mul ? NTT_FLAG_MUL : 0;
  run_pass3<F, 3, INV, LOGN, BOUNDED, LI>(f, A);
  return 0;
}

// ntt16c_kernel on the host: the sixteen CTAs of a cluster one after the other, phase by phase (both cluster barriers
// become the boundary between the loops); each CTA's receive buffer is a host array the others write through `remote`.
struct HostRemote {
  u64* const* bufs;
  u64* operator()(u32 rank) const { return bufs[rank]; }
};
template <class F, bool INV>
int run16_cluster(const F& f, u64 p, u64 g, u64* data, const u64* mul, u32 batch) {
  const u64 n = 65536;
  u64 w = h_powmod(g, (p - 1) / n, p);
  if (INV) w = h_powmod(w, p - 2, p);
  auto tw256 = table(f, h_powmod(w, n >> 8, p), 1, 256);
  const u64 ninv = INV ? h_powmod(n % p, p - 2, p) : 1;
  std::vector<u64> t2(65536);
  for (u32 i = 0; i < 65536; i++) t2[i] = f.to_tw(f.mul(field_pow(f, w, (u64)((i >> 8) * (i & 255u))), ninv));
  Ntt3Args A = {};
  A.tw256 = tw256.data(); A.t2 = t2.data(); A.batch = batch; A.src_len = A.dst_len = ~0ULL; A.mul_mask = ~0ULL;
  A.src = data; A.dst = data; A.mul_src = mul; A.flags = mul ? NTT_FLAG_MUL : 0;
  for (u32 b = 0; b < batch; b++) {
    std::vector<std::vector<u64>> tile(16, std::vector<u64>(N3_TILE_WORDS)), recv(16, std::vector<u64>(N3_RECV_WORDS));
    u64* bufs[16];
    for (int r = 0; r < 16; r++) bufs[r] = recv[r].data();
    u64 in_base, in_row, in_col, out_base, out_row;
    u32 m_base;
    for (u32 r = 0; r < 16; r++) {  // up to the first cluster barrier: every input of the transform is in shared memory
      n3_tile_geometry<2, 16>(16 * b + r, &in_base, &in_row, &in_col, &out_base, &out_row, &m_base);
      for (u32 t = 0; t < 2 * N3_THREADS; t++) n3_round0<F, 2, INV, false, 1>(f, tile[r].data(), A, in_base, in_row, in_col, t);
    }
    for (u32 r = 0; r < 16; r++)    // between the barriers: remote stores
      for (u32 t = 0; t < 2 * N3_THREADS; t++) n3_round1_cluster<F, INV, 1>(f, tile[r].data(), A, r, t, HostRemote{bufs});
    for (u32 r = 0; r < 16; r++) {  // after the second barrier: pass 3 out of the receive buffer, in place on the data
      Ntt3Args B = A;
      B.src = recv[r].data();
      for (u32 t = 0; t < 2 * N3_THREADS; t++) n3_round0<F, 3, INV, false, 1>(f, tile[r].data(), B, 0, 1, N3_RECV_STRIDE, t);
      n3_tile_geometry<3, 16>(16 * b + r, &in_base, &in_row, &in_col, &out_base, &out_row, &m_base);
      for (u32 t = 0; t < 2 * N3_THREADS; t++) n3_round1<F, 3, INV, false, 16, 1>(f, tile[r].data(), A, out_base, out_row, m_base, t);
    }
  }
  return 0;
}

template <int S>
void gl_pow2_n(const u64* a, u64* out, u64 n) {
  GoldilocksField f;
  for (u64 i = 0; i < n; i++) out[i] = f.mul_pow2<S>(a[i]);
}
template <int E, bool INV>
void gl_w16_sub_n(const u64* a, const u64* b, u64* out, u64 n) {
  GoldilocksField f;
  for (u64 i = 0; i < n; i++) out[i] = f.w16_sub<E, INV>(a[i], b[i]);
}
template <int... S>
void gl_pow2_dispatch(int s, const u64* a, u64* out, u64 n, std::integer_sequence<int, S...>) {
  static void (*const table[])(const u64*, u64*, u64) = {&gl_pow2_n<S>...};
  table[s](a, out, n);
}
template <int... E>
void gl_w16_sub_dispatch(int e, bool inv, const u64* a, const u64* b, u64* out, u64 n, std::integer_sequence<int, E...>) {
  static void (*const fwd[])(const u64*, const u64*, u64*, u64) = {&gl_w16_sub_n<E, false>...};
  static void (*const bwd[])(const u64*, const u64*, u64*, u64) = {&gl_w16_sub_n<E, true>...};
  (inv ? bwd : fwd)[e](a, b, out, n);
}

}  // namespace


// Bank-conflict audit of the additive layout of ntt12_kernel.cuh: worst multiplicity of a bank within one
// shared-memory transaction over every access of every phase; 1 = conflict-free.  128-bit accesses are served 8
// lanes at a time against eight 16-byte banks (slot mod 8); the 64-bit reads of the pass-1 store 16 lanes at a
// time against sixteen 8-byte banks.  Also checks that word() is injective and stays inside TILE_SLOTS (-1 if not).
template <int LC, int MODE>
static int layout12_worst() {
  using L = N12<LC, MODE>;
  std::vector<int> seen(L::TILE_SLOTS, 0);
  for (u32 e = 0; e < L::PAIRS; e++)
    if (L::word(e) >= L::TILE_SLOTS || seen[L::word(e)]++) return -1;
  int worst = 1;
  auto account = [&](const std::vector<u32>& banks, int nb) {
    std::vector<int> cnt(nb, 0);
    for (u32 w : banks) cnt[w % nb]++;
    for (int k = 0; k < nb; k++) worst = cnt[k] > worst ? cnt[k] : worst;
  };
  for (u32 q8 = 0; q8 < L::NTHR / 8; q8++) {
    for (int R = 0; R < 3; R++) {
      const u32 wb = L::LP + 8 - 4 * R;
      for (u32 q = 0; q < 16; q++) {
        std::vector<u32> w;
        for (u32 l = 0; l < 8; l++) {
          const u32 t = q8 * 8 + l;
          const u32 e0 = ((t >> wb) << (wb + 4)) | (t & ((1u << wb) - 1u));
          w.push_back(L::word(e0 | (q << wb)));
        }
        account(w, 8);
      }
    }
  }
  if (MODE == MODE_PASS1) {  // 64-bit reads: 16 lanes, bank = 2·slot + half
    for (u32 hw = 0; hw < L::NTHR / 16; hw++)
      for (u32 j = 0; j < 16; j++)
        for (u32 h = 0; h < 2; h++) {
          std::vector<u32> w;
          for (u32 l = 0; l < 16; l++) {
            const u32 g = hw * 16 + l + (j << L::KK);
            const u32 c = g & (L::C - 1u), blk = g >> LC;
            const u32 e = (bitrev12c(2 * blk + h) << L::LP) | (c >> 1);
            w.push_back(2 * L::word(e) + (c & 1u));
          }
          account(w, 16);
        }
  }
  return worst;
}

extern "C" {

// Same contract as ronk_ntt_u64 / ronk_ntt_mul_u64, on host memory.
int emu_ntt(uint64_t p, uint64_t g, uint64_t* data, const uint64_t* mul, uint32_t log_n, uint32_t batch, int inverse,
            uint32_t tile_cap, uint32_t pref1, uint32_t pref2) {
  if (log_n == 0 || log_n > 26 || (p - 1) % ((u64)1 << log_n) != 0) return 1;
  if (p == GL_P && g == 7) {
    GoldilocksField f;
    return inverse ? run<GoldilocksField, true>(f, p, g, true, data, mul, log_n, batch, tile_cap, pref1, pref2)
                   : run<GoldilocksField, false>(f, p, g, true, data, mul, log_n, batch, tile_cap, pref1, pref2);
  }
  MontField f = make_mont(p, g, inverse != 0);
  return inverse ? run<MontField, true>(f, p, g, false, data, mul, log_n, batch, tile_cap, pref1, pref2)
                 : run<MontField, false>(f, p, g, false, data, mul, log_n, batch, tile_cap, pref1, pref2);
}
// Goldilocks (g = 7) 2^24- or 2^16-point transforms through the 256-point-tile kernel functions.
int emu_ntt3(uint64_t* data, const uint64_t* mul, uint32_t log_n, uint32_t batch, int inverse, int t1_table) {
  GoldilocksField f;
  g_ntt3_t1 = t1_table & 1;
  g_ntt3_ng1 = (t1_table >> 1) & 1;   // bit 1 of the switch word: one group per thread
  if (log_n == 24)
    return inverse ? run3<GoldilocksField, true, 24>(f, GL_P, 7, data, mul, batch) : run3<GoldilocksField, false, 24>(f, GL_P, 7, data, mul, batch);
  if (log_n == 16)
    return inverse ? run3<GoldilocksField, true, 16>(f, GL_P, 7, data, mul, batch) : run3<GoldilocksField, false, 16>(f, GL_P, 7, data, mul, batch);
  if (log_n == 20)
    return inverse ? run3<GoldilocksField, true, 20>(f, GL_P, 7, data, mul, batch) : run3<GoldilocksField, false, 20>(f, GL_P, 7, data, mul, batch);
  if (log_n == 21)
    return inverse ? run3<GoldilocksField, true, 21>(f, GL_P, 7, data, mul, batch) : run3<GoldilocksField, false, 21>(f, GL_P, 7, data, mul, batch);
  if (log_n == 22)
    return inverse ? run3<GoldilocksField, true, 22>(f, GL_P, 7, data, mul, batch) : run3<GoldilocksField, false, 22>(f, GL_P, 7, data, mul, batch);
  if (log_n == 23)
    return inverse ? run3<GoldilocksField, true, 23>(f, GL_P, 7, data, mul, batch) : run3<GoldilocksField, false, 23>(f, GL_P, 7, data, mul, batch);
  // split transforms: 2^17 … 2^19 over 2^16, 2^25 over 2^24 (2^26 runs the same code with LI = 2: too slow for the CPU tier)
  if (log_n == 17)
    return inverse ? run3<GoldilocksField, true, 16, false, 1>(f, GL_P, 7, data, mul, batch) : run3<GoldilocksField, false, 16, false, 1>(f, GL_P, 7, data, mul, batch);
  if (log_n == 18)
    return inverse ? run3<GoldilocksField, true, 16, false, 2>(f, GL_P, 7, data, mul, batch) : run3<GoldilocksField, false, 16, false, 2>(f, GL_P, 7, data, mul, batch);
  if (log_n == 19)
    return inverse ? run3<GoldilocksField, true, 16, false, 3>(f, GL_P, 7, data, mul, batch) : run3<GoldilocksField, false, 16, false, 3>(f, GL_P, 7, data, mul, batch);
  if (log_n == 25)
    return inverse ? run3<GoldilocksField, true, 24, false, 1>(f, GL_P, 7, data, mul, batch) : run3<GoldilocksField, false, 24, false, 1>(f, GL_P, 7, data, mul, batch);
  return 1;
}
// forward transforms ⊙ ONE n-word multiplier shared by the batch (the twiddle column of the distributed transform)
int emu_ntt3_shared_mul(uint64_t* data, const uint64_t* mul_n_words, uint32_t log_n, uint32_t batch) {
  g_ntt3_mul_mask = ((unsigned long long)1 << log_n) - 1;
  const int rc = emu_ntt3(data, mul_n_words, log_n, batch, 0, 1);
  g_ntt3_mul_mask = ~0ULL;
  return rc;
}
// a batch of 2^16-point transforms through the cluster formulation (ntt16c_kernel), in place
int emu_ntt16_cluster(uint64_t* data, const uint64_t* mul, uint32_t batch, int inverse) {
  GoldilocksField f;
  return inverse ? run16_cluster<GoldilocksField, true>(f, GL_P, 7, data, mul, batch)
                 : run16_cluster<GoldilocksField, false>(f, GL_P, 7, data, mul, batch);
}
// one bounded 2^24 transform, as the polynomial product uses it: dst[0, dst_len) = NTT(src[0, src_len) zero-extended) [⊙ mul]
int emu_ntt3_bounded(const uint64_t* src, uint64_t src_len, uint64_t* dst, uint64_t dst_len, const uint64_t* mul, int inverse) {
  GoldilocksField f;
  g_ntt3_t1 = 0;
  return inverse ? run3<GoldilocksField, true, 24, true>(f, GL_P, 7, dst, mul, 1, src, src_len, dst_len)
                 : run3<GoldilocksField, false, 24, true>(f, GL_P, 7, dst, mul, 1, src, src_len, dst_len);
}
// worst bank multiplicity of the three-pass tile layout over all accesses of all passes (1 = conflict-free)
int emu_layout3_worst_conflict(void) {
  int worst = 1;
  auto account = [&](u32 (&w)[16]) {
    int cnt[16] = {0};
    for (int l = 0; l < 16; l++) cnt[w[l] & 15]++;
    for (int k = 0; k < 16; k++) worst = cnt[k] > worst ? cnt[k] : worst;
  };
  std::vector<int> seen(N3_TILE_WORDS, 0);
  for (u32 d1 = 0; d1 < 16; d1++) for (u32 d0 = 0; d0 < 16; d0++) for (u32 c = 0; c < 16; c++)
    if (n3_word(d1, d0, c) >= N3_TILE_WORDS || seen[n3_word(d1, d0, c)]++) return -1;
  for (int pass = 1; pass <= 3; pass++)
    for (u32 hw = 0; hw < 16; hw++)      // half-warp = 16 consecutive groups
      for (u32 q = 0; q < 16; q++) {
        u32 w0[16], w1[16];
        for (u32 l = 0; l < 16; l++) {
          const u32 g = hw * 16 + l;
          const u32 d0 = pass == 3 ? (g & 15u) : (g >> 4), c = pass == 3 ? (g >> 4) : (g & 15u);
          w0[l] = n3_word(q, d0, c);                 // round-0 write of register q
          w1[l] = n3_word(g >> 4, q, g & 15u);       // round-1 read of register q
        }
        account(w0);
        account(w1);
      }
  return worst;
}

void emu_set_variant(int v) { g_variant = v; }
void emu_set_fast12(int on) { g_fast12 = on; }
uint64_t emu_fast12_tiles(void) { return g_fast12_tiles; }

void emu_set_tw_table(int on) { g_tw_table = on; }
int emu_layout12_worst_conflict(int mode, int lc) {
  if (mode == MODE_PASS1 && lc == 2) return layout12_worst<2, MODE_PASS1>();
  if (mode == MODE_PASS2 && lc == 1) return layout12_worst<1, MODE_PASS2>();
  if (mode == MODE_PASS2 && lc == 2) return layout12_worst<2, MODE_PASS2>();
  return -2;
}

// Bounded out-of-place transform (ntt_device_bounded): dst[0, dst_len) = NTT(src[0, src_len) ‖ zeros) [⊙ mul].
int emu_ntt_bounded(uint64_t p, uint64_t g, const uint64_t* src, uint64_t src_len, uint64_t* dst, uint64_t dst_len,
                    const uint64_t* mul, uint32_t log_n, int inverse, uint32_t tile_cap, uint32_t pref1, uint32_t pref2) {
  if (log_n == 0 || log_n > 26 || (p - 1) % ((u64)1 << log_n) != 0) return 1;
  if (p == GL_P && g == 7) {
    GoldilocksField f;
    return inverse ? run<GoldilocksField, true>(f, p, g, true, dst, mul, log_n, 1, tile_cap, pref1, pref2, src, src_len, dst_len)
                   : run<GoldilocksField, false>(f, p, g, true, dst, mul, log_n, 1, tile_cap, pref1, pref2, src, src_len, dst_len);
  }
  MontField f = make_mont(p, g, inverse != 0);
  return inverse ? run<MontField, true>(f, p, g, false, dst, mul, log_n, 1, tile_cap, pref1, pref2, src, src_len, dst_len)
                 : run<MontField, false>(f, p, g, false, dst, mul, log_n, 1, tile_cap, pref1, pref2, src, src_len, dst_len);
}

// Field-policy arithmetic, element-wise, for cross-checks against the oracle.
// op: 0 add, 1 sub, 2 mul, 3 neg(a), 4 a·2^b (Goldilocks only, b in the supported set)
int emu_field_op(uint64_t p, int op, const uint64_t* a, const uint64_t* b, uint64_t* out, uint64_t n, int force_mont) {
  if (p == GL_P && !force_mont) {
    GoldilocksField f;
    for (u64 i = 0; i < n; i++) {
      switch (op) {
        case 0: out[i] = f.add(a[i], b[i]); break;
        case 1: out[i] = f.sub(a[i], b[i]); break;
        case 2: out[i] = f.mul(a[i], b[i]); break;
        case 3: out[i] = f.neg(a[i]); break;
        default: return 1;
      }
    }
    return 0;
  }
  MontField f = make_mont(p, 0, false);
  for (u64 i = 0; i < n; i++) {
    switch (op) {
      case 0: out[i] = f.add(a[i], b[i]); break;
      case 1: out[i] = f.sub(a[i], b[i]); break;
      case 2: out[i] = f.mul(a[i], b[i]); break;
      case 3: out[i] = f.neg(a[i]); break;
      default: return 1;
    }
  }
  return 0;
}

// out[e] = a · ω16^e (e = 0..7) then a · ω16^-e (e = 0..7): the Goldilocks shift twiddles.
void emu_gl_w16(uint64_t a, uint64_t out[16]) {
  GoldilocksField f;
  out[0] = f.w16<0, false>(a); out[1] = f.w16<1, false>(a); out[2] = f.w16<2, false>(a); out[3] = f.w16<3, false>(a);
  out[4] = f.w16<4, false>(a); out[5] = f.w16<5, false>(a); out[6] = f.w16<6, false>(a); out[7] = f.w16<7, false>(a);
  out[8] = f.w16<0, true>(a); out[9] = f.w16<1, true>(a); out[10] = f.w16<2, true>(a); out[11] = f.w16<3, true>(a);
  out[12] = f.w16<4, true>(a); out[13] = f.w16<5, true>(a); out[14] = f.w16<6, true>(a); out[15] = f.w16<7, true>(a);
}

// The host twins of the Goldilocks shift primitives, element-wise, on the inputs the device harness gets
// (tests/cuda/field_harness.cu).  op 0: out = mul_pow2<k>(a), k in [0, 192); op 1: out = w16_sub<k, inv>(a, b),
// k in [0, 8).
int emu_gl_shift_op(int op, int k, int inv, const uint64_t* a, const uint64_t* b, uint64_t* out, uint64_t n) {
  if (op == 0 && k >= 0 && k < 192) {
    gl_pow2_dispatch(k, a, out, n, std::make_integer_sequence<int, 192>{});
    return 0;
  }
  if (op == 1 && k >= 0 && k < 8) {
    gl_w16_sub_dispatch(k, inv != 0, a, b, out, n, std::make_integer_sequence<int, 8>{});
    return 0;
  }
  return 1;
}

// Bank-conflict audit of the shared-memory swizzle: worst number of distinct 8-byte banks hit
// twice by any half-warp in a window read at base bit `wb` for a tile of 2^tile_log elements.
int emu_swizzle_worst_conflict(uint32_t tile_log, uint32_t wb) {
  const u32 nthr = (1u << tile_log) / 16;
  int worst = 1;
  for (u32 hw = 0; hw < nthr / 16; hw++)
    for (u32 q = 0; q < 16; q++) {
      int cnt[16] = {0};
      for (u32 l = 0; l < 16; l++) {
        const u32 t = hw * 16 + l;
        const u32 e0 = ((t >> wb) << (wb + 4)) | (t & ((1u << wb) - 1u));
        cnt[swz(e0 | (q << wb)) & 15]++;
      }
      for (int k = 0; k < 16; k++) worst = cnt[k] > worst ? cnt[k] : worst;
    }
  return worst;
}
}
