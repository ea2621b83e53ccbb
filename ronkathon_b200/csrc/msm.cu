// msm.cu — GF(101²) / AffinePoint<PlutoExtendedCurve> arithmetic and kzg::commit as a Pippenger
// bucket MSM.  Mirrors src/algebra/field/extension/gf_101_2.rs (inverse :35-47, Mul :86-100),
// src/curve/mod.rs (Add :178-213, Neg :225-235, Mul<ScalarField> :157-172, is_on_curve :130-139),
// src/curve/pluto_curve.rs:40-51 (y² = x³ + 3) and src/kzg/setup.rs:48-60 (commit).
//
// Points travel as one packed 32-bit word x0 | x1<<8 | y0<<16 | y1<<24 (x = x0 + x1·t);
// 0xFFFFFFFF is Infinity.  Scalars are F17 residues, one byte each, so a single 5-bit Pippenger
// window with 16 non-trivial buckets covers the whole scalar.
//
//   msm_bucket_kernel   every thread streams its share of (point, scalar) pairs into 16 private
//                       buckets held in shared memory ([bucket][thread], conflict-free), then the
//                       CTA tree-reduces the 16 × 128 partials with ALL threads sharing the
//                       (bucket, pair) work of each level → partial[cta][17].
//   msm_finish_kernel   one CTA, 64 threads per bucket: tree over the partials, then
//                       Σ s·B_s = Σ_{k=1..16} (B_16 + … + B_k) as a suffix scan + tree sum in one warp.
// The whole computation is a chain of dependent affine adds, so it is latency-bound: what matters is
// the number of SEQUENTIAL adds (≈ 16 stream + 18 tree + 8 + 6 + 8 for 2^20 terms) and the latency of
// one add.  The field is so small that an affine add costs one F101 inversion, cheaper than projective
// formulas, and it keeps the reference's exceptional-case structure verbatim; in the MSM kernels the
// inverse comes from a 101-entry table in shared memory (built per CTA with the x^99 chain) instead of
// nine dependent multiplies per add.
#include "msm_curve.cuh"
#include "ronk_internal.h"

namespace ronk {

constexpr int MSM_THREADS = 128;
constexpr int MSM_TERMS = 16;       // terms per thread the grid is sized for
constexpr int MSM_FIN_LANES = 64;   // finishing threads per bucket

__global__ void __launch_bounds__(MSM_THREADS) msm_bucket_kernel(const u32* __restrict__ points,
                                                                 const uint8_t* __restrict__ scalars, size_t n,
                                                                 u32* __restrict__ partial, int* flag) {
  __shared__ u32 bucket[16][MSM_THREADS];  // bucket[s-1][thread]
  __shared__ uint8_t inv[104];
  const u32 t = threadIdx.x;
  build_inv_table(inv, t, MSM_THREADS);
#pragma unroll
  for (int s = 0; s < 16; s++) bucket[s][t] = PT_INF;
  __syncthreads();
  const size_t stride = (size_t)gridDim.x * MSM_THREADS;
  bool bad = false;
  // the loads of the next pair are issued before the current one is processed: the add chain below is
  // latency-bound and would otherwise wait a full memory
  // latency per term
  size_t i = (size_t)blockIdx.x * MSM_THREADS + t;
  u32 w_next = (i < n) ? points[i] : PT_INF, s_next = (i < n) ? scalars[i] : 0u;
  for (; i < n; i += stride) {
    const u32 w = w_next, s = s_next;
    if (i + stride < n) { w_next = points[i + stride]; s_next = scalars[i + stride]; }
    if (s >= 17 || !pt_valid(w)) { bad = true; continue; }
    if (s == 0 || w == PT_INF) continue;  // g1 * 0 = Infinity (curve/mod.rs:163-165)
    bucket[s - 1][t] = pt_add_t(bucket[s - 1][t], w, inv);
  }
  if (bad) atomicExch(flag, 1);
  __syncthreads();
  // 16 × len partial sums → 16 × len/2, every thread takes (bucket, pair) items: 8, 4, 2, 1, 1, 1, 1
  // sequential adds instead of 16 per level on the surviving threads
  for (u32 half = MSM_THREADS / 2; half > 0; half >>= 1) {
    for (u32 idx = t; idx < 16u * half; idx += MSM_THREADS) {
      const u32 s = idx / half, j = idx - s * half;
      bucket[s][j] = pt_add_t(bucket[s][j], bucket[s][j + half], inv);
    }
    __syncthreads();
  }
  if (t < 17) partial[(size_t)blockIdx.x * 17 + t] = (t == 0) ? PT_INF : bucket[t - 1][0];
}

// partial[sets][17] → buckets_out[17], result.  blockDim = 16 buckets × MSM_FIN_LANES.
__global__ void __launch_bounds__(16 * MSM_FIN_LANES) msm_finish_kernel(const u32* __restrict__ partial, u32 sets,
                                                                        u32* __restrict__ buckets_out,
                                                                        u32* __restrict__ result) {
  __shared__ u32 red[16][MSM_FIN_LANES];
  __shared__ uint8_t inv[104];
  const u32 tid = threadIdx.x, s = tid / MSM_FIN_LANES, lane = tid % MSM_FIN_LANES;  // bucket s + 1
  build_inv_table(inv, tid, blockDim.x);
  __syncthreads();
  u32 acc = PT_INF;
  for (u32 g = lane; g < sets; g += MSM_FIN_LANES) acc = pt_add_t(acc, partial[(size_t)g * 17 + s + 1], inv);
  red[s][lane] = acc;
  __syncthreads();
  for (u32 half = MSM_FIN_LANES / 2; half > 0; half >>= 1) {
    if (lane < half) red[s][lane] = pt_add_t(red[s][lane], red[s][lane + half], inv);
    __syncthreads();
  }
  if (tid < 17) buckets_out[tid] = (tid == 0) ? PT_INF : red[tid - 1][0];
  if (tid < 32) {
    // lane k < 16 holds B_{k+1}.  run_k = B_{k+1} + … + B_16 (suffix scan), result = Σ_k run_k:
    // every B_s is counted s times.  8 sequential adds instead of the 32 of the serial running sum.
    u32 v = (tid < 16) ? red[tid][0] : PT_INF;
#pragma unroll
    for (int off = 1; off < 16; off <<= 1) {
      const u32 other = __shfl_down_sync(0xFFFFFFFFu, v, off);
      if (tid + off < 16) v = pt_add_t(v, other, inv);
    }
#pragma unroll
    for (int off = 8; off > 0; off >>= 1) {
      const u32 other = __shfl_down_sync(0xFFFFFFFFu, v, off);
      if (tid < (u32)off) v = pt_add_t(v, other, inv);
    }
    if (tid == 0) result[0] = v;
  }
}

// ---------------------------------------------------------------------------------------------------
// kzg::commit as a point-indexed histogram (round 2).  E(F_101²): y² = x³ + 3 has 102² = 10 404 points and
// exponent 102, so Σ s_i·P_i = Σ_P (c_P mod 102)·P with c_P = Σ_{i: P_i = P} s_i.  Each term then costs one
// table lookup (validation) and one shared-memory atomicAdd — the kernel streams the 5 B/term once and is
// HBM / atomic-bound instead of a chain of dependent affine additions (round 1: 73 GB/s at 2^20 terms).
//   bin(P) = 2·(x0 + 101·x1) + ybit(y),  ybit(y) = y0 ? (y0 > 50) : (y1 > 50)   (y and -y get different bits)
//   ytab[bin] = y0 | y1 << 8 of the curve point in that bin, 0xFFFF when the bin holds no point: a term is
//               on the curve (curve/mod.rs:130-139) iff its coordinates are canonical and ytab[bin] == its y.
//   msm_hist_kernel     per-CTA histogram in shared memory → partial[cta][MSM_BINS] (plain coalesced store)
//   msm_hist_finish     one thread per bin: column sum mod 102, c·P by double-and-add with the reference's
//                       addition law, CTA tree; the last CTA to finish reduces the CTA sums and writes result
//                       and error flag straight into mapped pinned host memory (no memset / memcpy launches).
// (MSM_XS, MSM_BINS, MSM_EXP, y_bit, pt_bin: msm_curve.cuh)
constexpr int MSM_HIST_THREADS = 1024;
constexpr int MSM_FIN_THREADS = 256;   // bins per finishing CTA
constexpr u32 MSM_FIN_GROUPS = 4;      // thread groups sharing the column sum of those bins (blockDim = 1024)

// sq[idx(y²)] = y (either root), for every y in F_101²
__global__ void msm_sqrt_table_kernel(uint16_t* sq) {
  const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= MSM_XS) return;
  const Gf y = {i % Q101, i / Q101};
  const Gf y2 = gf_mul(y, y);
  sq[y2.c0 + Q101 * y2.c1] = (uint16_t)(y.c0 | (y.c1 << 8));  // the two roots race; either is fine
}
__global__ void msm_ytab_kernel(const uint16_t* __restrict__ sq, uint16_t* __restrict__ ytab) {
  const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= MSM_XS) return;
  const Gf x = {i % Q101, i / Q101};
  const Gf rhs = gf_add(gf_mul(gf_mul(x, x), x), Gf{3, 0});
  const u32 r = sq[rhs.c0 + Q101 * rhs.c1];
  uint16_t e0 = 0xFFFF, e1 = 0xFFFF;
  if (r != 0xFFFFu) {
    const Gf y = {r & 0xFF, r >> 8}, ny = gf_neg(y);
    const uint16_t wy = (uint16_t)(y.c0 | (y.c1 << 8)), wn = (uint16_t)(ny.c0 | (ny.c1 << 8));
    (y_bit(y.c0, y.c1) ? e1 : e0) = wy;
    if (wn != wy) (y_bit(ny.c0, ny.c1) ? e1 : e0) = wn;
  }
  ytab[2 * i] = e0;
  ytab[2 * i + 1] = e1;
}

__global__ void __launch_bounds__(MSM_HIST_THREADS, 1)
msm_hist_kernel(const u32* __restrict__ points, const uint8_t* __restrict__ scalars, size_t n,
                const uint16_t* __restrict__ ytab_g, u32* __restrict__ partial, u32* __restrict__ ghist,
                volatile int* host_flag) {
  extern __shared__ __align__(16) u32 msm_smem[];
  u32* hist = msm_smem;                                      // [MSM_BINS]
  uint16_t* ytab = reinterpret_cast<uint16_t*>(hist + MSM_BINS);  // [MSM_BINS]
  const u32 t = threadIdx.x;
  asm volatile("griddepcontrol.launch_dependents;");  // the finishing kernel may set up while this one runs (PDL)
  for (u32 i = t; i < MSM_BINS; i += MSM_HIST_THREADS) hist[i] = 0u;
  {  // 40 804 bytes of table, 4 at a time
    const u32* src = reinterpret_cast<const u32*>(ytab_g);
    u32* dst = reinterpret_cast<u32*>(ytab);
    for (u32 i = t; i < MSM_BINS / 2; i += MSM_HIST_THREADS) dst[i] = src[i];
  }
  __syncthreads();
  const size_t stride = (size_t)gridDim.x * MSM_HIST_THREADS;
  bool bad = false;
  constexpr int U = 4;  // loads in flight per thread
  for (size_t i0 = (size_t)blockIdx.x * MSM_HIST_THREADS + t; i0 < n; i0 += stride * U) {
    u32 w[U], s[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const size_t i = i0 + (size_t)u * stride;
      w[u] = (i < n) ? points[i] : PT_INF;
      s[u] = (i < n) ? (u32)scalars[i] : 0u;
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      if (s[u] >= 17u) { bad = true; continue; }            // not an F17 residue
      if (w[u] == PT_INF) continue;                         // Infinity · s = Infinity
      if (__vcmpgeu4(w[u], 0x65656565u)) { bad = true; continue; }  // a coordinate ≥ 101
      const u32 bin = 2u * ((w[u] & 0xFF) + Q101 * ((w[u] >> 8) & 0xFF)) + y_bit((w[u] >> 16) & 0xFF, w[u] >> 24);
      if ((u32)ytab[bin] != (w[u] >> 16)) { bad = true; continue; }  // not on y² = x³ + 3
      if (!s[u]) continue;                                  // g1 * 0 = Infinity (curve/mod.rs:163-165)
      // Shared-memory atomics retire about one lane per clock per SM.  RONK_MSM_SPLIT=1 sends every other term to an
      // L2-resident global histogram with a fire-and-forget RED instead; that was several times SLOWER (the 20 k hot
      // L2 lines serialise), so it is off by default and kept only as a recorded
      // negative result.
      if (ghist && (u & 1)) atomicAdd(&ghist[bin], s[u]);
      else atomicAdd(&hist[bin], s[u]);
    }
  }
  if (bad) *host_flag = 1;
  __syncthreads();
  u32* out = partial + (size_t)blockIdx.x * MSM_BINS;
  for (u32 i = t; i < MSM_BINS; i += MSM_HIST_THREADS) out[i] = hist[i];
}

// CTA tree over one point per thread (len = blockDim.x, a power of two); result in red[0].
// Five levels inside each warp by shuffles (no barrier), then one warp folds the per-warp sums.
RONK_DEV void msm_cta_tree(u32* red, u32 t, u32 len, const uint8_t* inv) {
#if defined(__CUDA_ARCH__)
  u32 v = red[t];
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const u32 o = __shfl_down_sync(0xFFFFFFFFu, v, off);
    if ((t & 31u) < (u32)off) v = pt_add_t(v, o, inv);
  }
  __syncthreads();
  if ((t & 31u) == 0) red[t >> 5] = v;
  __syncthreads();
  if (t < 32) {
    const u32 warps = len >> 5;  // ≤ 32
    v = (t < warps) ? red[t] : 0xFFFFFFFFu;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const u32 o = __shfl_down_sync(0xFFFFFFFFu, v, off);
      if (t < (u32)off) v = pt_add_t(v, o, inv);
    }
    if (t == 0) red[0] = v;
  }
  __syncthreads();
#endif
}

__global__ void __launch_bounds__(MSM_FIN_THREADS * MSM_FIN_GROUPS)
msm_hist_finish_kernel(const u32* __restrict__ partial, u32 sets, u32* __restrict__ ghist,
                       const uint16_t* __restrict__ ytab, u32* __restrict__ cta_sum, u32* __restrict__ done_counter,
                       volatile u32* host_result) {
  __shared__ u32 red[MSM_FIN_THREADS];
  __shared__ u32 colsum[MSM_FIN_GROUPS][MSM_FIN_THREADS];
  __shared__ uint8_t inv[104];
  __shared__ u32 is_last;
  const u32 t = threadIdx.x & (MSM_FIN_THREADS - 1u), grp = threadIdx.x / MSM_FIN_THREADS;
  build_inv_table(inv, threadIdx.x, MSM_FIN_THREADS * MSM_FIN_GROUPS);
  const u32 bin = blockIdx.x * MSM_FIN_THREADS + t;
  asm volatile("griddepcontrol.wait;" ::: "memory");  // the histogram kernel has completed and its stores are visible
  // Column sum over the partial histograms: the kernel's long pole (ncu: long_scoreboard 35 of 48 stall cycles per
  // instruction).  MSM_FIN_GROUPS thread groups take every MSM_FIN_GROUPS-th histogram with 16 loads in flight each,
  // so 132 histograms are 3 dependent steps instead of 9.
  {
    u32 acc16[16];
#pragma unroll
    for (int k = 0; k < 16; k++) acc16[k] = 0u;
    if (bin < MSM_BINS) {
      u32 g = grp;
      for (; g + 15u * MSM_FIN_GROUPS < sets; g += 16u * MSM_FIN_GROUPS) {
#pragma unroll
        for (int k = 0; k < 16; k++) acc16[k] += partial[(size_t)(g + (u32)k * MSM_FIN_GROUPS) * MSM_BINS + bin];
      }
      for (; g < sets; g += MSM_FIN_GROUPS) acc16[0] += partial[(size_t)g * MSM_BINS + bin];
    }
    u32 part = 0;
#pragma unroll
    for (int k = 0; k < 16; k++) part += acc16[k];
    colsum[grp][t] = part;
  }
  __syncthreads();
  if (grp) return;  // the remaining work is one thread per bin
  u32 c = 0;
  if (bin < MSM_BINS) {
#pragma unroll
    for (u32 k = 0; k < MSM_FIN_GROUPS; k++) c += colsum[k][t];
    if (ghist) {
      c += ghist[bin];
      ghist[bin] = 0u;  // self-cleaning: ready for the next call
    }
  }
  c %= MSM_EXP;
  __syncthreads();
  u32 acc = PT_INF;
  if (c) {  // the bin holds a curve point (only validated terms were counted)
    const u32 xi = bin >> 1;
    const u32 base = (xi % Q101) | ((xi / Q101) << 8) | ((u32)ytab[bin] << 16);
    // c·P, most significant bit first: ≤ 6 doublings + ≤ 6 additions of the reference's affine law
    for (int b = 31 - __clz(c); b >= 0; b--) {
      acc = pt_add_t(acc, acc, inv);
      if ((c >> b) & 1u) acc = pt_add_t(acc, base, inv);
    }
  }
  red[t] = acc;
  __syncthreads();
  msm_cta_tree(red, t, MSM_FIN_THREADS, inv);
  if (t == 0) {
    cta_sum[blockIdx.x] = red[0];
    __threadfence();
    is_last = (atomicAdd(done_counter, 1u) == gridDim.x - 1) ? 1u : 0u;
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  u32 mine = 0xFFFFFFFFu;  // Infinity
  if (t < gridDim.x) mine = reinterpret_cast<volatile u32*>(cta_sum)[t];  // gridDim.x ≤ MSM_FIN_THREADS
  red[t] = mine;
  __syncthreads();
  msm_cta_tree(red, t, MSM_FIN_THREADS, inv);
  if (t == 0) {
    host_result[0] = red[0];
    *done_counter = 0u;  // ready for the next call
  }
}

// ---------------------------------------------------------------------------------------------------
// kzg::commit in group coordinates (round 2, default).  E(F_101²) ≅ (Z/102)² (msm_curve.cuh, build_group_tables):
// with P_i = a_i·G1 + b_i·G2,  Σ s_i·P_i = (Σ s_i a_i mod 102)·G1 + (Σ s_i b_i mod 102)·G2.  Per term: one 4-byte and
// one 1-byte load (16 + 4 bytes per four terms on the vector path), the same validation as the histogram kernel (the
// table entry carries the y of the bin's curve point: is_on_curve, curve/mod.rs:130-139), ONE shared-memory load and
// two integer multiply-adds into registers — no atomics, no dependent point additions.  One launch: the last CTA to
// finish (atomic counter) looks the result up in pttab and writes it, with the error flag, into mapped pinned host
// memory.  Bound by HBM at 5 B/term once the 82 KB table per CTA is amortised.
constexpr int MSM_COORD_THREADS = 1024;
constexpr int MSM_COORD_U = 2;  // 16-byte point loads per thread and batch; two batches (16 terms) are in flight

// Branch-free: a rejected term only raises `bad` (the call then fails and the sums are discarded).
__device__ __forceinline__ void msm_coord_term(u32 w, u32 s, const u32* __restrict__ tab, u32& acc_a, u32& acc_b, u32& bad) {
  u32 e;
  const bool on = coord_term(w, tab, e);                 // Infinity contributes nothing
  bad |= (u32)(s >= 17u) | (u32)(!on && w != PT_INF);    // not an F17 residue / off the curve / non-canonical
  const u32 sv = on ? s : 0u;                            // s = 0 adds nothing: g1 * 0 = Infinity (curve/mod.rs:163-165)
  acc_a += sv * ((e >> 16) & 0xFFu);
  acc_b += sv * (e >> 24);
}

struct MsmQuads {
  uint4 w[MSM_COORD_U];
  u32 s[MSM_COORD_U];
};
__device__ __forceinline__ void msm_coord_load(MsmQuads& b, const uint4* __restrict__ p4, const u32* __restrict__ s4, size_t q0,
                                               size_t step, size_t quads) {
#pragma unroll
  for (int u = 0; u < MSM_COORD_U; u++) {
    const size_t q = q0 + (size_t)u * step;
    if (q < quads) { b.w[u] = p4[q]; b.s[u] = s4[q]; }
    else { b.w[u] = make_uint4(PT_INF, PT_INF, PT_INF, PT_INF); b.s[u] = 0u; }
  }
}

__global__ void __launch_bounds__(MSM_COORD_THREADS, 1)
msm_coord_kernel(const u32* __restrict__ points, const uint8_t* __restrict__ scalars, size_t n, int vec,
                 const u32* __restrict__ bintab_g, const u32* __restrict__ pttab,
                 unsigned long long* __restrict__ gacc /* arrivals << 48 | Σa << 24 | Σb */, volatile u32* host /*[0] flag, [1] result*/) {
  extern __shared__ __align__(16) u32 msm_smem[];
  u32* tab = msm_smem;  // [MSM_BINS]
  __shared__ u32 wsum[2][MSM_COORD_THREADS / 32];
  const u32 t = threadIdx.x;
  const size_t gthreads = (size_t)gridDim.x * MSM_COORD_THREADS, gtid = (size_t)blockIdx.x * MSM_COORD_THREADS + t;
  const size_t quads = vec ? (n >> 2) : 0;
  const uint4* p4 = reinterpret_cast<const uint4*>(points);
  const u32* s4 = reinterpret_cast<const u32*>(scalars);
  const size_t step = gthreads * MSM_COORD_U;
  // the first batch of terms is requested before the table: its HBM latency hides behind the 82 KB table copy
  MsmQuads cur;
  msm_coord_load(cur, p4, s4, gtid, gthreads, quads);
  {
    const uint4* src = reinterpret_cast<const uint4*>(bintab_g);  // MSM_BINS padded to a multiple of 4 words
    uint4* dst = reinterpret_cast<uint4*>(tab);
    for (u32 i = t; i < (MSM_BINS + 3) / 4; i += MSM_COORD_THREADS) dst[i] = src[i];
  }
  __syncthreads();
  u32 acc_a = 0, acc_b = 0, bad = 0;
  {
    u32 it = 0;
    for (size_t q0 = gtid; q0 < quads; q0 += step) {
      MsmQuads nxt;
      msm_coord_load(nxt, p4, s4, q0 + step, gthreads, quads);
#pragma unroll
      for (int u = 0; u < MSM_COORD_U; u++) {
        msm_coord_term(cur.w[u].x, cur.s[u] & 0xFFu, tab, acc_a, acc_b, bad);
        msm_coord_term(cur.w[u].y, (cur.s[u] >> 8) & 0xFFu, tab, acc_a, acc_b, bad);
        msm_coord_term(cur.w[u].z, (cur.s[u] >> 16) & 0xFFu, tab, acc_a, acc_b, bad);
        msm_coord_term(cur.w[u].w, cur.s[u] >> 24, tab, acc_a, acc_b, bad);
      }
      cur = nxt;
      // 8 terms ≤ 8·16·101 per pass: fold long before 32 bits fill (any n)
      if ((++it & 0x3FFFu) == 0u) { acc_a %= MSM_EXP; acc_b %= MSM_EXP; }
    }
  }
  {
    u32 it = 0;
    for (size_t i = (quads << 2) + gtid; i < n; i += gthreads) {  // tail of the vector path, or everything when unaligned
      msm_coord_term(points[i], (u32)scalars[i], tab, acc_a, acc_b, bad);
      if ((++it & 0xFFFFFu) == 0u) { acc_a %= MSM_EXP; acc_b %= MSM_EXP; }
    }
  }
  if (bad) host[0] = 1u;
  acc_a %= MSM_EXP;
  acc_b %= MSM_EXP;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    acc_a += __shfl_down_sync(0xFFFFFFFFu, acc_a, off);
    acc_b += __shfl_down_sync(0xFFFFFFFFu, acc_b, off);
  }
  if ((t & 31u) == 0) { wsum[0][t >> 5] = acc_a; wsum[1][t >> 5] = acc_b; }
  __syncthreads();
  if (t < 32) {
    u32 a = wsum[0][t], b = wsum[1][t];  // MSM_COORD_THREADS / 32 = 32 warps
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      a += __shfl_down_sync(0xFFFFFFFFu, a, off);
      b += __shfl_down_sync(0xFFFFFFFFu, b, off);
    }
    if (t == 0) {
      // ONE atomic per CTA carries both sums and the arrival; the CTA that sees all others' arrivals holds the totals
      const unsigned long long mine = (1ull << 48) | ((unsigned long long)(a % MSM_EXP) << 24) | (unsigned long long)(b % MSM_EXP);
      const unsigned long long old = atomicAdd(gacc, mine);
      if ((old >> 48) == (unsigned long long)(gridDim.x - 1)) {
        const unsigned long long tot = old + mine;
        const u32 sa = (u32)((tot >> 24) & 0xFFFFFFull) % MSM_EXP, sb = (u32)(tot & 0xFFFFFFull) % MSM_EXP;
        *gacc = 0ull;  // self-cleaning: the next call is ordered behind this kernel on the stream
        host[1] = pttab[MSM_EXP * sa + sb];
      }
    }
  }
}

// ctx->msm_coord: bintab[kTabWords] | pttab[102²] | counter, Σa, Σb — built once per context, on first use by either commit
// entry or by the pairing table (basis search + tables on the host, ≈ 3·10⁴ affine additions)
int msm_coord_tables(ronk_ctx* ctx) {
  if (ctx->msm_coord) return RONK_OK;
  std::vector<u32> tabs(kTabWords + MSM_EXP * MSM_EXP + 4, 0xFFFFFFFFu);
  if (!build_group_tables(tabs.data(), tabs.data() + kTabWords)) return set_err(ctx, RONK_ECUDA, "internal: no basis of E(F_101^2) found");
  tabs[kTabWords + MSM_EXP * MSM_EXP + 0] = tabs[kTabWords + MSM_EXP * MSM_EXP + 1] = tabs[kTabWords + MSM_EXP * MSM_EXP + 2] = 0u;
  return build_table(ctx, &ctx->msm_coord, tabs.size(), [&](u32* tab) {
    RONK_CUDA(ctx, cudaMemcpyAsync(tab, tabs.data(), tabs.size() * sizeof(u32), cudaMemcpyHostToDevice, ctx->stream));
    RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // tabs is pageable and goes out of scope
    return RONK_OK;
  });
}

static int msm_coord_device(ronk_ctx* ctx, const uint8_t* points, size_t n_points, const uint8_t* scalars, size_t n_scalars,
                            u32* h_result) {
  if (!ctx || (n_scalars && (!points || !scalars))) return set_err(ctx, RONK_EINVAL, "null argument");
  if (n_points < n_scalars) return set_err(ctx, RONK_EINVAL, "srs shorter than coefficients (kzg/setup.rs:53)");
  if (((uintptr_t)points & 3) != 0) return set_err(ctx, RONK_EINVAL, "points must be 4-byte aligned");
  if (n_scalars == 0) { *h_result = PT_INF; return RONK_OK; }   // empty sum = Infinity (curve/mod.rs:219-223)
  constexpr size_t kSmem = kTabWords * sizeof(u32);
  RONK_TRY(msm_coord_tables(ctx));
  RONK_TRY(ensure_smem_attr(ctx, msm_coord_kernel, (int)kSmem));
  const u32* bintab = ctx->msm_coord.get();
  const u32* pttab = bintab + kTabWords;
  static_assert((kTabWords + MSM_EXP * MSM_EXP) % 2 == 0, "the 64-bit accumulator must be 8-byte aligned");
  unsigned long long* gacc = (unsigned long long*)(ctx->msm_coord.get() + kTabWords + MSM_EXP * MSM_EXP);
  // a CTA is worth its 82 KB table load once every thread sees ≥ 4 terms
  const int ctas = grid_for(ctx, n_scalars, MSM_COORD_THREADS * 4, 1);
  const int vec = (((uintptr_t)points & 15) == 0 && ((uintptr_t)scalars & 3) == 0) ? 1 : 0;
  volatile u32* host = (volatile u32*)ctx->h_flag;  // mapped pinned: [0] = flag, [1] = result
  host[0] = 0u;
  host[1] = PT_INF;
  u32* host_dev = nullptr;
  RONK_CUDA(ctx, cudaHostGetDevicePointer((void**)&host_dev, (void*)ctx->h_flag, 0));
  RONK_TRY(launch(ctx, "msm_coord", msm_coord_kernel, ctas, MSM_COORD_THREADS, kSmem, false, (const u32*)points, scalars,
                  n_scalars, vec, bintab, pttab, gacc, host_dev));
  RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (host[0]) return set_err(ctx, RONK_EINVAL, "off-curve point, non-canonical coordinate or scalar >= 17");
  *h_result = host[1];
  return RONK_OK;
}

// ---------------------------------------------------------------------------------------------------
// kzg::commit of `batch` scalar rows against one SRS (ronk_msm_pluto_ext_batch).  The rows share the points, so each
// point's group coordinates (a_i, b_i) are looked up and checked once per call, not once per row and point; a row is then
// two byte dot products mod 102, four terms per __dp4a (scalars < 17, coordinates < 102).  Three launches whatever the
// batch:
//   msm_coord_pack_kernel   the first n points → byte planes A[i] = a_i, B[i] = b_i, zero-padded to a multiple of 16 bytes
//                           (Infinity and rejected points: 0); raises the error flag for a bad point
//   msm_rows_kernel         one warp per item of MSM_ROWS_R rows × one column of MSM_ROWS_CHUNK scalar words: each row's
//                           (Σ s·a, Σ s·b) mod 102 over the column → partial[row][column]; raises the flag for a scalar
//                           ≥ 17.  A plane word is loaded once per item and serves all its rows; the planes (2n bytes)
//                           stay in L2 across rows, so the kernel streams the batch·n scalar bytes once
//   msm_rows_finish_kernel  one warp per row: the row's partials mod 102 in a fixed order, then pttab[102·Σa + Σb] →
//                           out[row], unless the flag is raised
constexpr int MSM_PACK_THREADS = 256;
constexpr int MSM_ROWS_THREADS = 256;
constexpr int MSM_ROWS_R = 4;                      // rows per warp item
constexpr int MSM_ROWS_U = 16;                     // scalar words per lane and row in one item
constexpr u64 MSM_ROWS_CHUNK = 32 * MSM_ROWS_U;    // scalar words per column
// Each __dp4a adds at most 4·16·101 = 6464 (four scalars < 17 times coordinates < 102); a lane's accumulators start at 0
// in every item and are folded mod 102 at its end, after at most MSM_ROWS_U steps.
static_assert((u64)MSM_ROWS_U * 6464u < (1ull << 32), "msm_rows_kernel's accumulators must not overflow between folds");

__global__ void __launch_bounds__(MSM_PACK_THREADS)
msm_coord_pack_kernel(const u32* __restrict__ points, size_t n, size_t plane_words, const u32* __restrict__ bintab,
                      u32* __restrict__ A, u32* __restrict__ B, volatile u32* flag) {
  const size_t stride = (size_t)gridDim.x * MSM_PACK_THREADS;
  u32 bad = 0;
  for (size_t k = (size_t)blockIdx.x * MSM_PACK_THREADS + threadIdx.x; k < plane_words; k += stride) {
    u32 a4 = 0, b4 = 0;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const size_t i = 4 * k + j;
      if (i >= n) break;
      const u32 w = points[i];
      u32 e;
      const bool on = coord_term(w, bintab, e);
      bad |= (u32)(!on && w != PT_INF);   // off the curve / non-canonical
      if (on) {
        a4 |= ((e >> 16) & 0xFFu) << (8 * j);
        b4 |= (e >> 24) << (8 * j);
      }
    }
    A[k] = a4;
    B[k] = b4;
  }
  if (bad) *flag = 1u;
}

__global__ void __launch_bounds__(MSM_ROWS_THREADS, 4)
msm_rows_kernel(const uint8_t* __restrict__ scalars, size_t n, u32 batch, const u32* __restrict__ A, const u32* __restrict__ B,
                u64 cols, u32* __restrict__ partial, volatile u32* flag) {
  const u32 lane = threadIdx.x & 31u;
  const u64 items = ((u64)batch + MSM_ROWS_R - 1) / MSM_ROWS_R * cols;
  const u64 warps = (u64)gridDim.x * (MSM_ROWS_THREADS / 32);
  const u64 full = n >> 2, words = (n + 3) >> 2;   // whole scalar words of a row; with its byte tail
  u32 bad = 0;
  for (u64 item = (u64)blockIdx.x * (MSM_ROWS_THREADS / 32) + (threadIdx.x >> 5); item < items; item += warps) {
    const u64 grp = item / cols, col = item - grp * cols;
    const u64 r0 = grp * MSM_ROWS_R;
    u32 acc_a[MSM_ROWS_R], acc_b[MSM_ROWS_R];
#pragma unroll
    for (int j = 0; j < MSM_ROWS_R; j++) acc_a[j] = acc_b[j] = 0u;
#pragma unroll 4
    for (int u = 0; u < MSM_ROWS_U; u++) {
      const u64 k = col * MSM_ROWS_CHUNK + (u64)u * 32u + lane;
      if (k >= words) break;
      const u32 a4 = A[k], b4 = B[k];
#pragma unroll
      for (int j = 0; j < MSM_ROWS_R; j++) {
        if (r0 + j >= batch) break;
        // row r starts at byte r·n, so most rows are not 4-byte aligned: word k of the row is the funnel shift of the two
        // aligned words it straddles.  The upper one holds a byte of the row whenever the shift is nonzero, so no load
        // leaves the scalar block.  The row's last n mod 4 scalars are read as bytes.
        const uint8_t* row = scalars + (r0 + j) * n;
        u32 s4 = 0;
        if (k < full) {
          const uintptr_t at = (uintptr_t)(row + 4 * k);
          const u32 sh = (u32)(at & 3u);
          const u32* wp = reinterpret_cast<const u32*>(at - sh);
          s4 = __funnelshift_r(wp[0], sh ? wp[1] : 0u, 8u * sh);
        } else {
          for (u32 t = 0; t < (u32)(n & 3u); t++) s4 |= (u32)row[4 * k + t] << (8u * t);
        }
        bad |= scalar4_over(s4);
        acc_a[j] = __dp4a(s4, a4, acc_a[j]);
        acc_b[j] = __dp4a(s4, b4, acc_b[j]);
      }
    }
#pragma unroll
    for (int j = 0; j < MSM_ROWS_R; j++) {
      u32 a = acc_a[j] % MSM_EXP, b = acc_b[j] % MSM_EXP;
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) {
        a += __shfl_down_sync(0xFFFFFFFFu, a, off);
        b += __shfl_down_sync(0xFFFFFFFFu, b, off);
      }
      if (lane == 0 && r0 + j < batch) partial[(r0 + j) * cols + col] = (a % MSM_EXP) | ((b % MSM_EXP) << 16);
    }
  }
  if (bad) *flag = 1u;
}

__global__ void __launch_bounds__(MSM_ROWS_THREADS)
msm_rows_finish_kernel(const u32* __restrict__ partial, u64 cols, u32 batch, const u32* __restrict__ pttab,
                       const volatile u32* flag, u32* __restrict__ out) {
  __shared__ u32 raised;
  if (threadIdx.x == 0) raised = *flag;   // the earlier launches of the call have completed: one read per CTA
  __syncthreads();
  if (raised) return;                     // a rejected call leaves out as it was
  const u32 lane = threadIdx.x & 31u;
  const u64 warps = (u64)gridDim.x * (MSM_ROWS_THREADS / 32);
  for (u64 r = (u64)blockIdx.x * (MSM_ROWS_THREADS / 32) + (threadIdx.x >> 5); r < batch; r += warps) {
    u32 sa = 0, sb = 0;
    for (u64 c = lane; c < cols; c += 32) {
      const u32 v = partial[r * cols + c];
      sa += v & 0xFFFFu;
      sb += v >> 16;
      sa = sa >= MSM_EXP ? sa - MSM_EXP : sa;
      sb = sb >= MSM_EXP ? sb - MSM_EXP : sb;
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      sa += __shfl_down_sync(0xFFFFFFFFu, sa, off);
      sb += __shfl_down_sync(0xFFFFFFFFu, sb, off);
    }
    if (lane == 0) out[r] = pttab[MSM_EXP * (sa % MSM_EXP) + sb % MSM_EXP];
  }
}

// Step (1) of ronk_msm_pluto_ext_batch's errors: the checks that read no memory.  The _host twin skips the alignment
// check, which concerns the device buffers its staging provides.
static int msm_batch_args(ronk_ctx* ctx, const uint8_t* points, size_t n_points, const uint8_t* scalars, size_t n_scalars,
                          u32 batch, const uint8_t* out, bool device) {
  if (!ctx) return RONK_EINVAL;
  if ((batch && n_scalars && (!points || !scalars)) || (batch && !out)) return set_err(ctx, RONK_EINVAL, "null argument");
  if (n_points < n_scalars) return set_err(ctx, RONK_EINVAL, "srs shorter than coefficients (kzg/setup.rs:53)");
  if (device && ((((uintptr_t)points | (uintptr_t)out) & 3) != 0))
    return set_err(ctx, RONK_EINVAL, "points and out must be 4-byte aligned");
  if (batch && n_scalars > ((size_t)1 << 40) / batch) return set_err(ctx, RONK_EUNSUPPORTED, "batch * n_scalars above 2^40 bytes");
  return RONK_OK;
}

static int msm_batch_device(ronk_ctx* ctx, const uint8_t* points, size_t n_points, const uint8_t* scalars, size_t n_scalars,
                            u32 batch, uint8_t* out) {
  RONK_TRY(msm_batch_args(ctx, points, n_points, scalars, n_scalars, batch, out, true));
  if (bytes_overlap(out, (size_t)batch * 4, points, n_scalars * 4) || bytes_overlap(out, (size_t)batch * 4, scalars, (size_t)batch * n_scalars))
    return set_err(ctx, RONK_EINVAL, "out overlaps the points or the scalars");
  if (batch == 0) return RONK_OK;
  if (n_scalars == 0) {  // every row is the empty sum, Infinity (curve/mod.rs:219-223)
    RONK_CUDA(ctx, cudaMemsetAsync(out, 0xFF, (size_t)batch * 4, ctx->stream));
    return RONK_OK;
  }
  RONK_TRY(msm_coord_tables(ctx));
  const u32* bintab = ctx->msm_coord.get();
  const u32* pttab = bintab + kTabWords;
  const size_t plane_words = (n_scalars + 15) / 16 * 4;   // each plane: ⌈n/16⌉·16 bytes
  const u64 cols = ((n_scalars + 3) / 4 + MSM_ROWS_CHUNK - 1) / MSM_ROWS_CHUNK;
  const u64 items = ((u64)batch + MSM_ROWS_R - 1) / MSM_ROWS_R * cols;
  Frame fr(ctx);
  u32 *A = nullptr, *partial = nullptr;
  RONK_TRY(fr.take(&A, 2 * plane_words));
  RONK_TRY(fr.take(&partial, (size_t)batch * cols));
  u32* B = A + plane_words;
  volatile u32* host = (volatile u32*)ctx->h_flag;  // mapped pinned: [0] = flag
  host[0] = 0u;
  u32* flag = nullptr;
  RONK_CUDA(ctx, cudaHostGetDevicePointer((void**)&flag, (void*)ctx->h_flag, 0));
  RONK_TRY(launch(ctx, "msm_coord_pack", msm_coord_pack_kernel, grid_for(ctx, plane_words, MSM_PACK_THREADS), MSM_PACK_THREADS, 0,
                  false, (const u32*)points, n_scalars, plane_words, bintab, A, B, (volatile u32*)flag));
  RONK_TRY(launch(ctx, "msm_rows", msm_rows_kernel, grid_for(ctx, items, MSM_ROWS_THREADS / 32, 4), MSM_ROWS_THREADS, 0, false,
                  scalars, n_scalars, batch, (const u32*)A, (const u32*)B, cols, partial, (volatile u32*)flag));
  RONK_TRY(launch(ctx, "msm_rows_finish", msm_rows_finish_kernel, grid_for(ctx, batch, MSM_ROWS_THREADS / 32), MSM_ROWS_THREADS, 0,
                  false, (const u32*)partial, cols, batch, pttab, (const volatile u32*)flag, (u32*)out));
  RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (host[0]) return set_err(ctx, RONK_EINVAL, "off-curve point, non-canonical coordinate or scalar >= 17");
  return RONK_OK;
}

// element-wise curve ops (host API support). op: 0 add, 1 neg, 2 scalar-mul by repeated addition
__global__ void point_op_kernel(int op, const u32* a, const u32* b, const uint8_t* sc, u32* out, size_t n, int* flag) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const u32 wa = a[i];
    if (!pt_valid(wa)) { atomicExch(flag, 1); out[i] = PT_INF; continue; }
    if (op == 0) {
      const u32 wb = b[i];
      if (!pt_valid(wb)) { atomicExch(flag, 1); out[i] = PT_INF; continue; }
      out[i] = pt_add_w(wa, wb);
    } else if (op == 1) {
      Pt p = pt_unpack(wa);
      if (!p.inf) p.y = gf_neg(p.y);  // curve/mod.rs:228-231
      out[i] = pt_pack(p);
    } else {
      const u32 s = sc[i];
      if (s >= 17) { atomicExch(flag, 1); out[i] = PT_INF; continue; }
      u32 val = PT_INF;              // rhs == 0 → Infinity
      if (s) {
        val = wa;
        for (u32 k = 1; k < s; k++) val = pt_add_w(val, wa);  // (s-1) repeated `+=`
      }
      out[i] = val;
    }
  }
}

// Histogram path: result of the first n_scalars terms (kzg::commit).  Two launches, no memset, no memcpy:
// the kernels write the error flag and the result into mapped pinned host memory.
static int msm_hist_device(ronk_ctx* ctx, const uint8_t* points, size_t n_points, const uint8_t* scalars, size_t n_scalars,
                           u32* h_result) {
  if (!ctx || (n_scalars && (!points || !scalars))) return set_err(ctx, RONK_EINVAL, "null argument");
  if (n_points < n_scalars) return set_err(ctx, RONK_EINVAL, "srs shorter than coefficients (kzg/setup.rs:53)");
  if (((uintptr_t)points & 3) != 0) return set_err(ctx, RONK_EINVAL, "points must be 4-byte aligned");
  if (n_scalars == 0) { *h_result = PT_INF; return RONK_OK; }   // empty sum = Infinity (curve/mod.rs:219-223)
  constexpr size_t kSmem = MSM_BINS * sizeof(u32) + MSM_BINS * sizeof(uint16_t);
  if (!ctx->msm_ytab) {  // one-time per context: curve tables, completion counter
    DevBuf<uint16_t> sq, ytab;
    DevBuf<u32> done;
    RONK_TRY(build_tables(ctx, [&] {
      RONK_TRY(sq.alloc(ctx, MSM_XS));
      RONK_TRY(ytab.alloc(ctx, MSM_BINS));
      RONK_TRY(done.alloc(ctx, 1 + MSM_BINS));  // counter + global histogram
      RONK_CUDA(ctx, cudaMemsetAsync(sq.get(), 0xFF, MSM_XS * sizeof(uint16_t), ctx->stream));
      RONK_CUDA(ctx, cudaMemsetAsync(done.get(), 0, (1 + MSM_BINS) * sizeof(u32), ctx->stream));
      {
        LaunchScope ls(ctx, "msm_tables");
        msm_sqrt_table_kernel<<<(MSM_XS + 255) / 256, 256, 0, ctx->stream>>>(sq.get());
        msm_ytab_kernel<<<(MSM_XS + 255) / 256, 256, 0, ctx->stream>>>(sq.get(), ytab.get());
      }
      RONK_TRY(check_launch(ctx, "msm table kernels"));
      RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
      return RONK_OK;
    }));
    ctx->msm_ytab = std::move(ytab);
    ctx->msm_done = std::move(done);
  }
  RONK_TRY(ensure_smem_attr(ctx, msm_hist_kernel, (int)kSmem));
  // one CTA per SM at most; each thread should see ≥ 8 terms before another CTA (its table load and its 82 KB of
  // partial histogram) is worth it (≥ 32 terms per thread made 2^20 terms slower)
  const size_t ctas = grid_for(ctx, n_scalars, MSM_HIST_THREADS * 8, 1);
  constexpr u32 fin_ctas = (MSM_BINS + MSM_FIN_THREADS - 1) / MSM_FIN_THREADS;  // 80
  static_assert(fin_ctas <= MSM_FIN_THREADS, "final tree assumes one CTA sum per thread");
  Frame fr(ctx);
  u32* partial = nullptr;
  RONK_TRY(fr.take(&partial, ctas * MSM_BINS + fin_ctas));
  u32* cta_sum = partial + ctas * MSM_BINS;
  // the split between shared-memory and L2 atomics pays once the SM's atomic unit is the limiter
  u32* ghist = (n_scalars >= ((size_t)1 << 22) && ctx->tune.msm_split) ? ctx->msm_done.get() + 1 : nullptr;
  volatile u32* host = (volatile u32*)ctx->h_flag;  // mapped pinned: [0] = flag, [1] = result
  host[0] = 0u;
  host[1] = PT_INF;
  u32* host_dev = nullptr;
  RONK_CUDA(ctx, cudaHostGetDevicePointer((void**)&host_dev, (void*)ctx->h_flag, 0));
  RONK_TRY(launch(ctx, "msm_hist", msm_hist_kernel, (unsigned)ctas, MSM_HIST_THREADS, kSmem, false, (const u32*)points, scalars,
                  n_scalars, (const uint16_t*)ctx->msm_ytab.get(), partial, ghist, (volatile int*)host_dev));
  RONK_TRY(launch(ctx, "msm_hist_finish", msm_hist_finish_kernel, fin_ctas, MSM_FIN_THREADS * MSM_FIN_GROUPS, 0, ctx->tune.pdl,
                  partial, (u32)ctas, ghist, (const uint16_t*)ctx->msm_ytab.get(), cta_sum, ctx->msm_done.get(), host_dev + 1));
  RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (host[0]) return set_err(ctx, RONK_EINVAL, "off-curve point, non-canonical coordinate or scalar >= 17");
  *h_result = host[1];
  return RONK_OK;
}

// Bucket path (the 17 Pippenger bucket sums a rank contributes to a distributed commit, and the round-1 kernel
// pair): device buckets[17] + result[1] for the first n_scalars terms
static int msm_device(ronk_ctx* ctx, const uint8_t* points, size_t n_points, const uint8_t* scalars, size_t n_scalars,
                      u32* h_buckets /*17 or null*/, u32* h_result) {
  if (!ctx || (n_scalars && (!points || !scalars))) return set_err(ctx, RONK_EINVAL, "null argument");
  if (n_points < n_scalars) return set_err(ctx, RONK_EINVAL, "srs shorter than coefficients (kzg/setup.rs:53)");
  if (((uintptr_t)points & 3) != 0) return set_err(ctx, RONK_EINVAL, "points must be 4-byte aligned");
  const int ctas = grid_for(ctx, n_scalars, MSM_THREADS * MSM_TERMS);
  // device block [flag | 17 buckets | result]: one memset, and one copy into pinned host memory at the end
  // (two copies into pageable memory cost a large share of a small call)
  Frame fr(ctx);
  u32* partial = nullptr;
  RONK_TRY(fr.take(&partial, (size_t)ctas * 17 + 1 + 17 + 1));
  u32* d_mflag = partial + (size_t)ctas * 17;
  u32* d_buckets = d_mflag + 1;
  u32* d_result = d_buckets + 17;
  RONK_CUDA(ctx, cudaMemsetAsync(d_mflag, 0, sizeof(u32), ctx->stream));
  RONK_TRY(launch(ctx, "msm_bucket", msm_bucket_kernel, ctas, MSM_THREADS, 0, false, (const u32*)points, scalars, n_scalars,
                  partial, (int*)d_mflag));
  RONK_TRY(launch(ctx, "msm_finish", msm_finish_kernel, 1, 16 * MSM_FIN_LANES, 0, false, partial, (u32)ctas, d_buckets,
                  d_result));
  u32* host = (u32*)ctx->h_flag;  // pinned, 32 words
  RONK_CUDA(ctx, cudaMemcpyAsync(host, d_mflag, 19 * sizeof(u32), cudaMemcpyDeviceToHost, ctx->stream));
  RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (host[0]) return set_err(ctx, RONK_EINVAL, "off-curve point, non-canonical coordinate or scalar >= 17");
  if (h_buckets) std::memcpy(h_buckets, host + 1, 17 * sizeof(u32));
  if (h_result) *h_result = host[18];
  return RONK_OK;
}

static void unpack_to_bytes(u32 w, uint8_t out[4]) {
  out[0] = (uint8_t)(w & 0xFF);
  out[1] = (uint8_t)((w >> 8) & 0xFF);
  out[2] = (uint8_t)((w >> 16) & 0xFF);
  out[3] = (uint8_t)(w >> 24);
}

}  // namespace ronk

using namespace ronk;

extern "C" {

int ronk_msm_pluto_ext(ronk_ctx* ctx, const uint8_t* points, size_t n_points, const uint8_t* scalars, size_t n_scalars,
                       uint8_t out[4]) {
  ronk::DeviceGuard _dg(ctx);
  if (!out) return set_err(ctx, RONK_EINVAL, "null argument");
  u32 res = PT_INF;
  if (ctx && ctx->tune.msm_coord) RONK_TRY(msm_coord_device(ctx, points, n_points, scalars, n_scalars, &res));
  else if (ctx && ctx->tune.msm_hist) RONK_TRY(msm_hist_device(ctx, points, n_points, scalars, n_scalars, &res));
  else RONK_TRY(msm_device(ctx, points, n_points, scalars, n_scalars, nullptr, &res));
  unpack_to_bytes(res, out);
  return RONK_OK;
}

int ronk_msm_pluto_ext_buckets(ronk_ctx* ctx, const uint8_t* points, size_t n_points, const uint8_t* scalars,
                               size_t n_scalars, uint8_t buckets[68]) {
  ronk::DeviceGuard _dg(ctx);
  if (!buckets) return set_err(ctx, RONK_EINVAL, "null argument");
  u32 b[17];
  RONK_TRY(msm_device(ctx, points, n_points, scalars, n_scalars, b, nullptr));
  for (int s = 0; s < 17; s++) unpack_to_bytes(b[s], buckets + 4 * s);
  return RONK_OK;
}

// Checked before staging: a null argument, which cannot be uploaded, and the srs length, which the staged call (it
// passes n_scalars points) no longer sees.
int ronk_msm_pluto_ext_host(ronk_ctx* ctx, const uint8_t* points, size_t n_points, const uint8_t* scalars,
                            size_t n_scalars, uint8_t out[4]) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx || !out || (n_scalars && (!points || !scalars))) return set_err(ctx, RONK_EINVAL, "null argument");
  if (n_points < n_scalars) return set_err(ctx, RONK_EINVAL, "srs shorter than coefficients (kzg/setup.rs:53)");
  Staged s[] = {{n_scalars * 4, points}, {n_scalars, scalars}};
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  return stage_out(
      ctx, ronk_msm_pluto_ext(ctx, (const uint8_t*)s[0].dev, n_scalars, (const uint8_t*)s[1].dev, n_scalars, out), s);
}

int ronk_msm_pluto_ext_batch(ronk_ctx* ctx, const uint8_t* points, size_t n_points, const uint8_t* scalars, size_t n_scalars,
                             uint32_t batch, uint8_t* out) {
  ronk::DeviceGuard _dg(ctx);
  return msm_batch_device(ctx, points, n_points, scalars, n_scalars, batch, out);
}

// Ships only the first n_scalars points, as ronk_msm_pluto_ext_host does.
int ronk_msm_pluto_ext_batch_host(ronk_ctx* ctx, const uint8_t* points, size_t n_points, const uint8_t* scalars,
                                  size_t n_scalars, uint32_t batch, uint8_t* out) {
  ronk::DeviceGuard _dg(ctx);
  RONK_TRY(msm_batch_args(ctx, points, n_points, scalars, n_scalars, batch, out, false));
  if (batch == 0) return RONK_OK;
  Staged s[] = {{n_scalars * 4, points}, {(size_t)batch * n_scalars, scalars}, {(size_t)batch * 4, nullptr, out}};
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  return stage_out(ctx,
                   ronk_msm_pluto_ext_batch(ctx, (const uint8_t*)s[0].dev, n_scalars, (const uint8_t*)s[1].dev, n_scalars, batch,
                                            (uint8_t*)s[2].dev),
                   s);
}

int ronk_msm_combine_buckets_host(ronk_ctx* ctx, const uint8_t* buckets, size_t n_sets, uint8_t out[4]) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx || !out || (n_sets && !buckets)) return set_err(ctx, RONK_EINVAL, "null argument");
  if (n_sets > (1u << 20)) return set_err(ctx, RONK_EUNSUPPORTED, "too many bucket sets");
  u32 res;
  Staged s[] = {{n_sets * 17 * 4, buckets}, {17 * 4}, {4, nullptr, &res}};  // bucket sets, combined buckets, result
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  RONK_TRY(stage_out(ctx, launch(ctx, "msm_finish", msm_finish_kernel, 1, 16 * MSM_FIN_LANES, 0, false, (const u32*)s[0].dev,
                                 (u32)n_sets, (u32*)s[1].dev, (u32*)s[2].dev), s));
  unpack_to_bytes(res, out);
  return RONK_OK;
}

static int point_op_host(ronk_ctx* ctx, int op, const uint8_t* a, const uint8_t* b, const uint8_t* sc, uint8_t* out,
                         size_t n) {
  if (!ctx || (n && (!a || !out)) || (n && op == 0 && !b) || (n && op == 2 && !sc))
    return set_err(ctx, RONK_EINVAL, "null argument");
  if (n == 0) return RONK_OK;
  // a, b (add only), the scalars (smul only), out
  Staged s[] = {{n * 4, a}, {op == 0 ? n * 4 : 0, b}, {op == 2 ? n : 0, sc}, {n * 4, nullptr, out}};
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  RONK_TRY(reset_flag(ctx));
  RONK_TRY(launch(ctx, "point_op", point_op_kernel, grid_for(ctx, n, 128), 128, 0, false, op, (const u32*)s[0].dev,
                  (const u32*)s[1].dev, (const uint8_t*)s[2].dev, (u32*)s[3].dev, n, ctx->d_flag.get()));
  int v = 0;
  RONK_TRY(read_flag(ctx, &v));
  if (v) return set_err(ctx, RONK_EINVAL, "Point is not on curve / scalar out of range");
  return stage_out(ctx, RONK_OK, s);
}

int ronk_point_add_pluto_ext_host(ronk_ctx* ctx, const uint8_t* a, const uint8_t* b, uint8_t* out, size_t n) {
  ronk::DeviceGuard _dg(ctx);
  return point_op_host(ctx, 0, a, b, nullptr, out, n);
}
int ronk_point_neg_pluto_ext_host(ronk_ctx* ctx, const uint8_t* a, uint8_t* out, size_t n) {
  ronk::DeviceGuard _dg(ctx);
  return point_op_host(ctx, 1, a, nullptr, nullptr, out, n);
}
int ronk_point_smul_pluto_ext_host(ronk_ctx* ctx, const uint8_t* a, const uint8_t* scalars, uint8_t* out, size_t n) {
  ronk::DeviceGuard _dg(ctx);
  return point_op_host(ctx, 2, a, nullptr, scalars, out, n);
}

}  // extern "C"
