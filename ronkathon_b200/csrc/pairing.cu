// pairing.cu — the reference's Tate pairing on E[17] (src/curve/pairing.rs:33-54) and kzg::check (src/kzg/setup.rs:81-103)
// as table lookups in group coordinates.
//
// E(F_101²) ≅ (Z/102)² (msm_curve.cuh, build_group_tables): every point is a·G1 + b·G2, and the 17-torsion E[17] is the
// 289 points with 6 | a and 6 | b.  The pairing only accepts points of E[17], so it has at most 289² inputs:
//   pairing_table_kernel  once per context, one thread per pair (P, Q) of E[17]: the literal Miller loop and final
//                         exponentiation (pairing.cuh) → T[289·idx(P) + idx(Q)] = the index of the value in the 17-entry
//                         list of μ17, or PAIR_PANIC where the reference panics (Infinity in either argument, P == Q)
//   kzg_check_kernel      one thread per row: the (a, b) of the commitment and the proof by one bintab lookup each, then
//                         B = g2 − z·GEN and C′ = C − v·g1 by arithmetic mod 102, then T[proof][B] == T[C′][GEN]
//   pairing_kernel        the same lookups for explicit pairs, decoded to (c0, c1)
// Both tables (81.6 KB bintab, 83.5 KB T) sit in the check kernel's shared memory, one CTA per SM.
#include "pairing.cuh"
#include "ronk_internal.h"

namespace ronk {

constexpr int PAIR_TAB_THREADS = 256;
constexpr int KZG_CHECK_THREADS = 1024;
constexpr int PAIRING_THREADS = 256;
// ctx->pairing_tab: T[PAIR_TAB] padded to a multiple of 16 bytes | mu[17] (c0 | c1 << 8)
constexpr size_t kPairTabBytes = (PAIR_TAB + 15) / 16 * 16;

__global__ void __launch_bounds__(PAIR_TAB_THREADS) pairing_table_kernel(const u32* __restrict__ pttab, const uint16_t* __restrict__ mu,
                                                                        uint8_t* __restrict__ T) {
  const u32 i = blockIdx.x * PAIR_TAB_THREADS + threadIdx.x;
  if (i < PAIR_TAB) T[i] = pairing_entry(i / E17_PTS, i % E17_PTS, pttab, mu);
}

// Built once per context on first use by either entry, after the group tables it takes its basis from.
static int pairing_tables(ronk_ctx* ctx) {
  if (ctx->pairing_tab) return RONK_OK;
  RONK_TRY(msm_coord_tables(ctx));
  uint16_t mu[PAIR_R];
  mu17_list(mu);
  const u32* pttab = ctx->msm_coord.get() + kTabWords;
  return build_table(ctx, &ctx->pairing_tab, kPairTabBytes + sizeof(mu), [&](uint8_t* tab) {
    cudaError_t e = cudaMemcpyAsync(tab + kPairTabBytes, mu, sizeof(mu), cudaMemcpyHostToDevice, ctx->stream);
    if (e != cudaSuccess) return set_err(ctx, RONK_ECUDA, std::string("pairing table upload: ") + cudaGetErrorString(e));
    RONK_TRY(launch(ctx, "pairing_table", pairing_table_kernel, (PAIR_TAB + PAIR_TAB_THREADS - 1) / PAIR_TAB_THREADS,
                    PAIR_TAB_THREADS, 0, false, pttab, (const uint16_t*)(tab + kPairTabBytes), tab));
    if ((e = cudaStreamSynchronize(ctx->stream)) != cudaSuccess)  // mu is on this stack frame
      return set_err(ctx, RONK_ECUDA, std::string("pairing table build: ") + cudaGetErrorString(e));
    return RONK_OK;
  });
}

__global__ void __launch_bounds__(KZG_CHECK_THREADS, 1)
kzg_check_kernel(const u32* __restrict__ commitments, const u32* __restrict__ proofs, const uint8_t* __restrict__ points,
                 const uint8_t* __restrict__ values, size_t n, const u32* __restrict__ g1_srs, const u32* __restrict__ g2_srs,
                 const u32* __restrict__ bintab_g, const uint8_t* __restrict__ T_g, volatile u32* flag, uint8_t* __restrict__ ok) {
  extern __shared__ __align__(16) u32 pair_smem[];
  u32* bintab = pair_smem;                                            // [kTabWords]
  uint8_t* T = reinterpret_cast<uint8_t*>(pair_smem + kTabWords);     // [kPairTabBytes]
  const u32 t = threadIdx.x;
  {
    const uint4* src = reinterpret_cast<const uint4*>(bintab_g);
    uint4* dst = reinterpret_cast<uint4*>(bintab);
    for (u32 i = t; i < kTabWords / 4; i += KZG_CHECK_THREADS) dst[i] = src[i];
    const uint4* tsrc = reinterpret_cast<const uint4*>(T_g);
    uint4* tdst = reinterpret_cast<uint4*>(T);
    for (u32 i = t; i < kPairTabBytes / 16; i += KZG_CHECK_THREADS) tdst[i] = tsrc[i];
  }
  __syncthreads();
  // the SRS points the reference reads (g1_srs[0], g2_srs[1]) and GEN, once per thread
  u32 g1a, g1b, g2a, g2b, gena, genb;
  u32 bad = (u32)!point_coords(g1_srs[0], bintab, g1a, g1b) | (u32)!point_coords(g2_srs[1], bintab, g2a, g2b);
  point_coords(PLUTO_EXT_GEN, bintab, gena, genb);
  const u32 gen_idx = e17_index(gena, genb);
  const size_t stride = (size_t)gridDim.x * KZG_CHECK_THREADS;
  for (size_t i = (size_t)blockIdx.x * KZG_CHECK_THREADS + t; i < n; i += stride)
    ok[i] = kzg_check_row(commitments[i], proofs[i], points[i], values[i], g1a, g1b, g2a, g2b, gena, genb, gen_idx, bintab, T, bad);
  if (bad) *flag = 1u;
}

__global__ void __launch_bounds__(PAIRING_THREADS)
pairing_kernel(const u32* __restrict__ p, const u32* __restrict__ q, size_t n, const u32* __restrict__ bintab,
               const uint8_t* __restrict__ T, const uint16_t* __restrict__ mu, volatile u32* flag, uint8_t* __restrict__ out) {
  const size_t stride = (size_t)gridDim.x * PAIRING_THREADS;
  u32 bad = 0;
  for (size_t i = (size_t)blockIdx.x * PAIRING_THREADS + threadIdx.x; i < n; i += stride) {
    u32 pa, pb, qa, qb;
    bad |= (u32)!point_coords(p[i], bintab, pa, pb) | (u32)!point_coords(q[i], bintab, qa, qb);
    bad |= (u32)!e17_finite(pa, pb) | (u32)!e17_finite(qa, qb);
    const u32 k = T[E17_PTS * e17_index(pa, pb) + e17_index(qa, qb)];
    bad |= (u32)(k == PAIR_PANIC);
    const u32 v = mu[k < PAIR_R ? k : 0];
    out[2 * i] = (uint8_t)(v & 0xFFu);
    out[2 * i + 1] = (uint8_t)(v >> 8);
  }
  if (bad) *flag = 1u;
}

// Step (1) of both entries' errors, the checks that read no memory.  The _host twins skip the alignment check, which
// concerns the device buffers their staging provides.
static int pairing_args(ronk_ctx* ctx, const uint8_t* p, const uint8_t* q, size_t n, const uint8_t* out, bool device) {
  if (!ctx) return RONK_EINVAL;
  if (n && (!p || !q || !out)) return set_err(ctx, RONK_EINVAL, "null argument");
  if (device && (((uintptr_t)p | (uintptr_t)q) & 3) != 0) return set_err(ctx, RONK_EINVAL, "p and q must be 4-byte aligned");
  if (n >> 32) return set_err(ctx, RONK_EUNSUPPORTED, "n at or above 2^32");
  return RONK_OK;
}

static int check_args(ronk_ctx* ctx, const uint8_t* commitments, const uint8_t* proofs, const uint8_t* points, const uint8_t* values,
                      size_t n, const uint8_t* g1_srs, size_t n_g1, const uint8_t* g2_srs, size_t n_g2, const uint8_t* ok, bool device) {
  if (!ctx) return RONK_EINVAL;
  if (n && (!commitments || !proofs || !points || !values || !g1_srs || !g2_srs || !ok))
    return set_err(ctx, RONK_EINVAL, "null argument");
  if (n_g1 == 0) return set_err(ctx, RONK_EINVAL, "has g1 srs (kzg/setup.rs:89)");
  if (n_g2 < 2) return set_err(ctx, RONK_EINVAL, "g2_srs[1] out of bounds (kzg/setup.rs:92)");
  if (device && (((uintptr_t)commitments | (uintptr_t)proofs | (uintptr_t)g1_srs | (uintptr_t)g2_srs) & 3) != 0)
    return set_err(ctx, RONK_EINVAL, "point arrays must be 4-byte aligned");
  if (n >> 32) return set_err(ctx, RONK_EUNSUPPORTED, "n at or above 2^32");
  return RONK_OK;
}

}  // namespace ronk

using namespace ronk;

extern "C" {

int ronk_pairing_pluto_ext(ronk_ctx* ctx, const uint8_t* p, const uint8_t* q, size_t n, uint8_t* out) {
  ronk::DeviceGuard _dg(ctx);
  RONK_TRY(pairing_args(ctx, p, q, n, out, true));
  if (bytes_overlap(out, 2 * n, p, 4 * n) || bytes_overlap(out, 2 * n, q, 4 * n)) return set_err(ctx, RONK_EINVAL, "out overlaps p or q");
  if (n == 0) return RONK_OK;
  RONK_TRY(pairing_tables(ctx));
  volatile u32* flag = nullptr;
  RONK_TRY(clear_flag(ctx, &flag));
  const u32* bintab = ctx->msm_coord.get();
  const uint8_t* T = ctx->pairing_tab.get();
  RONK_TRY(launch(ctx, "pairing", pairing_kernel, grid_for(ctx, n, PAIRING_THREADS), PAIRING_THREADS, 0, false, (const u32*)p,
                  (const u32*)q, n, bintab, T, (const uint16_t*)(T + kPairTabBytes), flag, out));
  RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (ctx->h_flag[0]) return set_err(ctx, RONK_EINVAL, "off-curve or non-canonical point, a point outside E[17] or Infinity, or P == Q");
  return RONK_OK;
}

int ronk_pairing_pluto_ext_host(ronk_ctx* ctx, const uint8_t* p, const uint8_t* q, size_t n, uint8_t* out) {
  ronk::DeviceGuard _dg(ctx);
  RONK_TRY(pairing_args(ctx, p, q, n, out, false));
  if (n == 0) return RONK_OK;
  Staged s[] = {{4 * n, p}, {4 * n, q}, {2 * n, nullptr, out}};
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  return stage_out(ctx, ronk_pairing_pluto_ext(ctx, (const uint8_t*)s[0].dev, (const uint8_t*)s[1].dev, n, (uint8_t*)s[2].dev), s);
}

int ronk_kzg_check_pluto_ext_batch(ronk_ctx* ctx, const uint8_t* commitments, const uint8_t* proofs, const uint8_t* points,
                                   const uint8_t* values, size_t n, const uint8_t* g1_srs, size_t n_g1, const uint8_t* g2_srs,
                                   size_t n_g2, uint8_t* ok) {
  ronk::DeviceGuard _dg(ctx);
  RONK_TRY(check_args(ctx, commitments, proofs, points, values, n, g1_srs, n_g1, g2_srs, n_g2, ok, true));
  if (bytes_overlap(ok, n, commitments, 4 * n) || bytes_overlap(ok, n, proofs, 4 * n) || bytes_overlap(ok, n, points, n) ||
      bytes_overlap(ok, n, values, n) || bytes_overlap(ok, n, g1_srs, 4) || bytes_overlap(ok, n, g2_srs, 8))
    return set_err(ctx, RONK_EINVAL, "ok overlaps an input");
  if (n == 0) return RONK_OK;
  constexpr size_t kSmem = kTabWords * sizeof(u32) + kPairTabBytes;
  RONK_TRY(pairing_tables(ctx));
  RONK_TRY(ensure_smem_attr(ctx, kzg_check_kernel, (int)kSmem));
  volatile u32* flag = nullptr;
  RONK_TRY(clear_flag(ctx, &flag));
  // a CTA is worth its 165 KB of tables once every thread sees ≥ 4 rows
  RONK_TRY(launch(ctx, "kzg_check", kzg_check_kernel, grid_for(ctx, n, KZG_CHECK_THREADS * 4, 1), KZG_CHECK_THREADS, kSmem, false,
                  (const u32*)commitments, (const u32*)proofs, points, values, n, (const u32*)g1_srs, (const u32*)g2_srs,
                  (const u32*)ctx->msm_coord.get(), (const uint8_t*)ctx->pairing_tab.get(), flag, ok));
  RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (ctx->h_flag[0])
    return set_err(ctx, RONK_EINVAL, "off-curve or non-canonical point, scalar >= 17, or a pairing argument the reference panics on");
  return RONK_OK;
}

// Ships only the SRS points the check reads: g1_srs[0] and g2_srs[0..2).
int ronk_kzg_check_pluto_ext_batch_host(ronk_ctx* ctx, const uint8_t* commitments, const uint8_t* proofs, const uint8_t* points,
                                        const uint8_t* values, size_t n, const uint8_t* g1_srs, size_t n_g1, const uint8_t* g2_srs,
                                        size_t n_g2, uint8_t* ok) {
  ronk::DeviceGuard _dg(ctx);
  RONK_TRY(check_args(ctx, commitments, proofs, points, values, n, g1_srs, n_g1, g2_srs, n_g2, ok, false));
  if (n == 0) return RONK_OK;
  Staged s[] = {{4 * n, commitments}, {4 * n, proofs}, {n, points}, {n, values}, {4, g1_srs}, {8, g2_srs}, {n, nullptr, ok}};
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  return stage_out(ctx,
                   ronk_kzg_check_pluto_ext_batch(ctx, (const uint8_t*)s[0].dev, (const uint8_t*)s[1].dev, (const uint8_t*)s[2].dev,
                                                  (const uint8_t*)s[3].dev, n, (const uint8_t*)s[4].dev, 1, (const uint8_t*)s[5].dev, 2,
                                                  (uint8_t*)s[6].dev),
                   s);
}

}  // extern "C"
