// rs.cu — Reed–Solomon encoding (Message::encode, src/codes/reed_solomon.rs:42-52) and errors-and-erasures decoding
// of batches of codewords, positions i < n at ω_n^i.  With m = n - k, per row:
//   Y = n^-1 · (inverse transform of the row); S_j = Y[k + j], j < m (zero for a codeword);
//   Γ(z) = Π_{i erased} (1 - ω^-i z); Berlekamp–Massey seeded with Γ (Blahut's form, inversion-free:
//   Ψ ← b·Ψ - d·z^s·B, which scales Ψ and Ω by one constant) gives the errata locator Ψ; fail unless
//   2·deg Ψ - ε ≤ m; Ω = S·Ψ mod z^m;
//   forward transforms of Ψ, Ψ', Ω: the roots of Ψ among the ω^i and, there, the errata values (Forney)
//   e_i = -n · ω^(i(k-1)) · Ω(ω^i) / Ψ'(ω^i);
//   C = n^-1 · inverse transform of (row - e); fail unless |roots| = deg Ψ and C[k..n) = 0; the message is C[0..k).
// The last check is what keeps the decoder bounded-distance: it never returns a codeword outside the radius.
// tests/test_rs_decode_model.py is a Python model of the same steps.
//
// Launches per decode (none depends on the batch): the inverse transform of the rows, rs_locator (one CTA per row,
// Ψ in registers, S and B in shared memory), one forward transform of 3·batch rows (Ψ, Ψ', Ω), rs_correct
// (element-wise), the inverse transform, rs_finish.  The transforms are ronk_ntt_any_u64's (anyntt_device) on its
// power-of-two and Bluestein paths; on its literal path (n below the crossover, not a power of two) they are
// rs_dft_kernel, one O(n²) launch over all rows, in place of ntt_any's per-row evaluation launches.
#include <algorithm>

#include "ntt_kernel.cuh"
#include "ronk_internal.h"

namespace ronk {

// Ψ has m + 1 ≤ 8192 coefficients, RS_LOC_PER in registers of each of ≤ 1024 threads.  Shared memory: S (m words)
// and the two buffers of B (m + 1 words each), 24·m + 16 bytes: 196 600 bytes at the cap, under the H100's 227 KiB.
constexpr int RS_LOC_PER = 8;
constexpr int RS_LOC_MAX_THREADS = 1024;
constexpr u64 kRsMaxParity = (u64)RS_LOC_PER * RS_LOC_MAX_THREADS - 1;  // 8191
constexpr int RS_THREADS = 256;

// Per-row results of the locator, completed by rs_correct.
struct RsRow {
  u32 deg;    // deg Ψ
  u32 eps;    // erasures
  u32 fail;   // nonzero: the row is uncorrectable
  u32 roots;  // roots of Ψ among the ω^i (rs_correct)
};

template <class F>
__device__ __forceinline__ u64 rs_warp_sum(const F& f, u64 v) {
  for (int o = 16; o > 0; o >>= 1) v = f.add(v, __shfl_xor_sync(0xFFFFFFFFu, v, o));
  return v;
}

// The locator of one row per CTA, for both decoders.  AT = false (ronk_rs_decode_u64): the syndromes are
// Y[b·n + k + j] of the rows' scaled inverse transforms, the erasure at position i contributes (1 - ω^-i z), and the
// outputs are Ψ, Ψ', Ω with rows[b].deg = deg Ψ.  AT = true (ronk_rs_decode_at_u64): the syndromes are Y[b·sld + j],
// the erasure at position i contributes (1 - xs[i]·z), and the outputs are the reversed forms σ = X^L·Ψ(1/X), σ' and
// Ω̂ = X^(L-1)·Ω(1/X) with rows[b].deg = L, Berlekamp–Massey's length: a point at 0 adds the factor 1 to Ψ but a root
// at 0 to σ, so deg Ψ would miss it.  Either way the outputs are zero-padded to `ld` words at out + b·ld,
// + plane + b·ld, + 2·plane + b·ld (all zero for a failed row).  Thread t owns the coefficients i = t + j·blockDim.x,
// j < RS_LOC_PER.
template <class F, bool AT>
__device__ __forceinline__ void rs_locator_body(const F& f, const u64* __restrict__ Y, u64 sld, const u64* __restrict__ xs,
                                                const uint8_t* __restrict__ erased, u64 n, u64 k, u64 winv,
                                                u64* __restrict__ out, u64 ld, u64 plane, RsRow* __restrict__ rows) {
  extern __shared__ u64 sm[];
  __shared__ u64 red[2][RS_LOC_MAX_THREADS / 32];
  __shared__ u32 count;
  __shared__ int top;
  const u64 m = n - k;
  const u32 t = threadIdx.x, T = blockDim.x, lane = t & 31, warp = t >> 5, nwarps = T >> 5;
  const u64 b = blockIdx.x;
  u64* S = sm;
  const auto Bb = [&](int c) { return sm + m + (u64)c * (m + 1); };  // the two buffers of B
  if (t == 0) {
    count = 0;
    top = 0;
  }
  __syncthreads();
  // the erasures' ω^-i (x_i), in any order (Γ is a product), into S's space: S is loaded after Γ is built
  if (erased)
    for (u64 i = t; i < n; i += T)
      if (erased[b * n + i]) {
        const u32 at = atomicAdd(&count, 1u);
        if constexpr (AT) {
          if (at < m) S[at] = xs[i];
        } else {
          if (at < m) S[at] = field_pow(f, winv, i);
        }
      }
  for (u64 i = t; i <= m; i += T) Bb(0)[i] = i == 0 ? 1 % f.modulus() : 0;
  __syncthreads();
  const u32 eps = count;
  bool fail = eps > m;
  u64 psi[RS_LOC_PER];
  int cur = 0;
  if (!fail) {
    for (u32 l = 0; l < eps; l++) {  // Γ ← Γ · (1 - x z)
      const u64 x = S[l];
      const u64* src = Bb(l & 1);
      u64* dst = Bb((l & 1) ^ 1);
      for (u64 i = t; i <= m; i += T) dst[i] = i ? f.sub(src[i], f.mul(x, src[i - 1])) : src[0];
      __syncthreads();
    }
    cur = eps & 1;
  }
#pragma unroll
  for (int j = 0; j < RS_LOC_PER; j++) {
    const u64 i = t + (u64)j * T;
    psi[j] = !fail && i <= m ? Bb(cur)[i] : 0;
  }
  __syncthreads();  // the erasure list is read; S may be loaded
  if constexpr (AT) {
    for (u64 j = t; j < m; j += T) S[j] = Y[b * sld + j];
  } else {
    for (u64 j = t; j < m; j += T) S[j] = Y[b * n + k + j];
  }
  __syncthreads();
  if (!fail) {
    // Berlekamp–Massey, one barrier per step: Ψ stays in registers, B is read at Bb(cur) and a new B written to the
    // other buffer, which nobody reads before the next step's barrier; red is double-buffered the same way.
    // hi, hb: upper bounds of deg Ψ and deg B (uniform), so that the work of a step stops at the coefficients that can
    // be nonzero.  A new B is written in full, zeros included, so reads past hb see zeros.
    u64 L = eps, bb = 1 % f.modulus(), s = 1, hi = eps, hb = eps;
    for (u64 r = eps; r < m; r++) {
      u64 part = 0;
#pragma unroll
      for (int j = 0; j < RS_LOC_PER; j++) {
        const u64 i = t + (u64)j * T;
        if (i <= r && i <= hi) part = f.add(part, f.mul(psi[j], S[r - i]));
      }
      part = rs_warp_sum(f, part);
      if (lane == 0) red[r & 1][warp] = part;
      __syncthreads();
      const u64 d = rs_warp_sum(f, lane < nwarps ? red[r & 1][lane] : 0);
      if (d == 0) {
        s++;
        continue;
      }
      const u64* Bc = Bb(cur);
      const bool grow = 2 * L <= r + eps;
      const u64 nh = s + hb < hi ? hi : (s + hb < m ? s + hb : m);
#pragma unroll
      for (int j = 0; j < RS_LOC_PER; j++) {
        const u64 i = t + (u64)j * T;
        if (i <= m) {
          const u64 old = psi[j];
          if (i <= nh) psi[j] = f.sub(f.mul(bb, old), i >= s ? f.mul(d, Bc[i - s]) : 0);
          if (grow) Bb(cur ^ 1)[i] = old;
        }
      }
      if (grow) hb = hi;
      hi = nh;
      if (grow) {
        cur ^= 1;
        L = r + 1 + eps - L;
        bb = d;
        s = 1;
      } else {
        s++;
      }
    }
    if constexpr (AT) {
      if (t == 0) top = (int)L;
    } else {
#pragma unroll
      for (int j = 0; j < RS_LOC_PER; j++) {
        const u64 i = t + (u64)j * T;
        if (i <= m && psi[j]) atomicMax(&top, (int)i);
      }
    }
  }
  __syncthreads();
  const u32 deg = (u32)top;
  fail = fail || 2 * (u64)deg > m + eps;
  u64* P = Bb(0);  // Ψ, for its derivative and Ω
#pragma unroll
  for (int j = 0; j < RS_LOC_PER; j++) {
    const u64 i = t + (u64)j * T;
    if (i <= m) P[i] = fail ? 0 : psi[j];
  }
  __syncthreads();
  u64* o = out + b * ld;
  if constexpr (AT) {
    // σ[i] = Ψ[L - i], σ'[i] = (i + 1)·Ψ[L - 1 - i], Ω̂[i] = Ω[L - 1 - i]; L ≤ m on a row that has not failed
    const u64 L = fail ? 0 : deg;
    for (u64 i = t; i < ld; i += T) {
      u64 sg = 0, ds = 0, om = 0;
      if (i <= L) sg = P[L - i];
      if (i < L) {
        const u64 e = L - 1 - i;
        ds = f.mul((i + 1) % f.modulus(), P[e]);
        for (u64 l = 0; l <= e; l++) om = f.add(om, f.mul(P[l], S[e - l]));
      }
      o[i] = sg;
      o[plane + i] = ds;
      o[2 * plane + i] = om;
    }
  } else {
    for (u64 i = t; i < ld; i += T) {
      u64 om = 0;
      if (i < m)
        for (u64 l = 0; l <= i; l++) om = f.add(om, f.mul(P[l], S[i - l]));
      o[i] = i <= m ? P[i] : 0;
      o[plane + i] = i < m ? f.mul((i + 1) % f.modulus(), P[i + 1]) : 0;
      o[2 * plane + i] = om;
    }
  }
  if (t == 0) rows[b] = RsRow{deg, eps, fail ? 1u : 0u, 0u};
}

// Y: the rows' scaled inverse transforms (batch × n); erased: batch × n bytes or null; winv = ω^-1.
template <class F>
__global__ void __launch_bounds__(RS_LOC_MAX_THREADS)
rs_locator_kernel(const F f, const u64* __restrict__ Y, const uint8_t* __restrict__ erased, u64 n, u64 k, u64 winv,
                  u64* __restrict__ out, u64 ld, u64 plane, RsRow* __restrict__ rows) {
  rs_locator_body<F, false>(f, Y, 0, nullptr, erased, n, k, winv, out, ld, plane, rows);
}

// S: the rows' syndromes, m = n - k words at S + b·sld; xs: the n points; erased: batch × n bytes or null.
template <class F>
__global__ void __launch_bounds__(RS_LOC_MAX_THREADS)
rs_locator_at_kernel(const F f, const u64* __restrict__ S, u64 sld, const u64* __restrict__ xs,
                     const uint8_t* __restrict__ erased, u64 n, u64 k, u64* __restrict__ out, u64 ld, u64 plane,
                     RsRow* __restrict__ rows) {
  rs_locator_body<F, true>(f, S, sld, xs, erased, n, k, 0, out, ld, plane, rows);
}

// out[r·n + i] = scale · Σ_{j<len} a[r·lda + j] · ω^(±ij), r < rows: the literal transform of every row in one launch,
// ω^(ij mod n) read from nodes (ω^i, plain).  scale2 = to_tw(to_tw(scale)): the sum is accumulated in twiddle products.
template <class F, bool INV>
__global__ void __launch_bounds__(RS_THREADS)
rs_dft_kernel(const F f, const u64* __restrict__ a, u64 len, u64 lda, const u64* __restrict__ nodes, u64 n, u64 rows,
              u64 scale2, u64* __restrict__ out) {
  const u64 total = rows * n, stride = (u64)gridDim.x * blockDim.x;
  for (u64 at = (u64)blockIdx.x * blockDim.x + threadIdx.x; at < total; at += stride) {
    const u64 r = at / n, i = at - r * n;
    const u64 step = INV ? (i ? n - i : 0) : i;
    const u64* src = a + r * lda;
    u64 acc = 0, e = 0;
    for (u64 j = 0; j < len; j++) {
      acc = f.add(acc, f.mul_tw(src[j], nodes[e]));
      e += step;
      if (e >= n) e -= n;
    }
    out[at] = f.mul_tw(acc, scale2);
  }
}

// codeword[b·n + i] = msg[b·k + i] for i < k, else 0
__global__ void __launch_bounds__(RS_THREADS)
rs_pad_kernel(const u64* __restrict__ msg, u64 k, u64 n, u64 total, u64* __restrict__ cw) {
  const u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 at = (u64)blockIdx.x * blockDim.x + threadIdx.x; at < total; at += stride) {
    const u64 b = at / n, i = at - b * n;
    cw[at] = i < k ? msg[b * k + i] : 0;
  }
}

// R = received - e over batch × n: at a root ω^i of Ψ (P: its values, plane words before those of Ψ' and Ω), the
// Forney value; counts the roots per row (at most deg Ψ ≤ m of them: Ψ(0) ≠ 0), and a root where Ψ' vanishes fails.
template <class F>
__global__ void __launch_bounds__(RS_THREADS)
rs_correct_kernel(const F f, const u64* __restrict__ received, const u64* __restrict__ P, u64 plane, u64 n, u64 k, u64 w,
                  u64 neg_n, RsRow* rows, u64* __restrict__ R) {
  const u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 at = (u64)blockIdx.x * blockDim.x + threadIdx.x; at < plane; at += stride) {
    const u64 b = at / n, i = at - b * n;
    u64 v = received[at];
    if (!rows[b].fail && P[at] == 0) {
      atomicAdd(&rows[b].roots, 1u);
      const u64 dv = P[plane + at];
      if (dv == 0) {
        atomicOr(&rows[b].fail, 1u);
      } else {
        const u64 x = f.mul(field_pow(f, w, i * (k - 1) % n), f.mul(neg_n, P[2 * plane + at]));
        v = f.sub(v, f.mul(x, field_pow(f, dv, f.modulus() - 2)));
      }
    }
    R[at] = v;
  }
}

// out = received with its erased positions set to 0, over total words: the erased values are never read after this.
__global__ void __launch_bounds__(RS_THREADS)
rs_mask_kernel(const u64* __restrict__ received, const uint8_t* __restrict__ erased, u64 total, u64* __restrict__ out) {
  const u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 at = (u64)blockIdx.x * blockDim.x + threadIdx.x; at < total; at += stride) out[at] = erased[at] ? 0 : received[at];
}

// rs_correct_kernel at any points: R = row - e over batch × n.  At a root x_i of σ (E: σ's values, plane words before
// those of σ' and Ω̂), e_i = Ω̂(x_i)·M'(x_i) / σ'(x_i), W[i] = M'(x_i); counts the roots per row (at most L: deg σ = L,
// and σ's roots among distinct points are distinct), and a root where σ' vanishes fails.
template <class F>
__global__ void __launch_bounds__(RS_THREADS)
rs_forney_kernel(const F f, const u64* __restrict__ row, const u64* __restrict__ E, u64 plane, const u64* __restrict__ W, u64 n,
                 RsRow* rows, u64* __restrict__ R) {
  const u64 stride = (u64)gridDim.x * blockDim.x;
  for (u64 at = (u64)blockIdx.x * blockDim.x + threadIdx.x; at < plane; at += stride) {
    const u64 b = at / n, i = at - b * n;
    u64 v = row[at];
    if (!rows[b].fail && E[at] == 0) {
      atomicAdd(&rows[b].roots, 1u);
      const u64 dv = E[plane + at];
      if (dv == 0) {
        atomicOr(&rows[b].fail, 1u);
      } else {
        const u64 x = f.mul(E[2 * plane + at], W[i]);
        v = f.sub(v, f.mul(x, field_pow(f, dv, f.modulus() - 2)));
      }
    }
    R[at] = v;
  }
}

// Grid (row, chunk), RS_FIN_CHUNK message words per CTA: the row decodes when the locator did not fail, Ψ has deg Ψ roots
// and C[k..n) = 0 (m ≤ kRsMaxParity words, checked by every CTA of the row); then msg = C[0..k) and status = deg Ψ - ε,
// else msg = 0 and status = -1.
constexpr u64 RS_FIN_CHUNK = (u64)RS_THREADS * 32;
__global__ void __launch_bounds__(RS_THREADS)
rs_finish_kernel(const u64* __restrict__ C, u64 n, u64 k, const RsRow* __restrict__ rows, u64* __restrict__ msg,
                 int32_t* __restrict__ status) {
  __shared__ int bad;
  const u64 b = blockIdx.x;
  const RsRow rw = rows[b];
  if (threadIdx.x == 0) bad = rw.fail || rw.roots != rw.deg;
  __syncthreads();
  const u64* c = C + b * n;
  for (u64 i = k + threadIdx.x; i < n; i += blockDim.x)
    if (c[i]) bad = 1;
  __syncthreads();
  const bool ok = !bad;
  const u64 end = std::min(k, (blockIdx.y + 1) * RS_FIN_CHUNK);
  for (u64 j = blockIdx.y * RS_FIN_CHUNK + threadIdx.x; j < end; j += blockDim.x) msg[b * k + j] = ok ? c[j] : 0;
  if (blockIdx.y == 0 && threadIdx.x == 0) status[b] = ok ? (int32_t)(rw.deg - rw.eps) : -1;
}

// Checks shared by encode and decode, after the null checks: *path set on RONK_OK.  `rows` transforms of n points
// run in one call; 3·batch·n < 2^31 is within what every transform path takes.
static int rs_args(ronk_ctx* ctx, u64 p, u64 g, const void* in, u64 n, u64 k, u64 rows, AnyNttPath* path) {
  if (n == 0 || k == 0 || k > n) return set_err(ctx, RONK_EINVAL, "need 0 < k <= n");
  RONK_TRY(anyntt_args(ctx, p, g, in, n, path));
  if (!root_has_order(h_powmod(g, (p - 1) / n, p), n, p))  // n ≤ 2^26 here
    return set_err(ctx, RONK_EINVAL, "ω_n has order below n (two positions share a point)");
  if (rows * n > 0x7FFFFFFFULL) return set_err(ctx, RONK_EUNSUPPORTED, "batch too large");
  return RONK_OK;
}

template <class F>
static int rs_dft(ronk_ctx* ctx, const F& f, const u64* a, u64 len, u64 lda, const u64* nodes, u64 n, u64 rows, bool inverse,
                  u64* out) {
  const u64 p = f.modulus();
  const u64 scale = inverse ? h_powmod(n % p, p - 2, p) : 1 % p;
  const int grid = grid_for(ctx, rows * n, RS_THREADS);
  if (inverse)
    return launch(ctx, "rs_dft", rs_dft_kernel<F, true>, grid, RS_THREADS, 0, false, f, a, len, lda, nodes, n, rows,
                  f.to_tw(f.to_tw(scale)), out);
  return launch(ctx, "rs_dft", rs_dft_kernel<F, false>, grid, RS_THREADS, 0, false, f, a, len, lda, nodes, n, rows,
                f.to_tw(f.to_tw(scale)), out);
}

static int rs_encode_device(ronk_ctx* ctx, u64 p, u64 g, const u64* msg, u64 k, u64 n, u32 batch, u64* cw) {
  if (!ctx || !msg || !cw) return set_err(ctx, RONK_EINVAL, "null argument");
  AnyNttPath path;
  RONK_TRY(rs_args(ctx, p, g, msg, n, k, batch, &path));
  if (bytes_overlap(msg, (size_t)batch * k * 8, cw, (size_t)batch * n * 8)) return set_err(ctx, RONK_EINVAL, "output overlaps input");
  if (batch == 0) return RONK_OK;
  if (path != AN_LITERAL) {
    RONK_TRY(launch(ctx, "rs_pad", rs_pad_kernel, grid_for(ctx, (size_t)batch * n, RS_THREADS), RS_THREADS, 0, false, msg, k,
                    n, (u64)batch * n, cw));
    return anyntt_device(ctx, p, g, cw, n, batch, 0);
  }
  Frame fr(ctx);
  u64* nodes = nullptr;
  RONK_TRY(fr.take(&nodes, n));
  RONK_TRY(roots_table(ctx, p, g, n, nodes));
  return with_field(ctx, p, 0, false, [&](const auto& f) { return rs_dft(ctx, f, msg, k, k, nodes, n, batch, false, cw); });
}

static int rs_decode_args(ronk_ctx* ctx, u64 p, u64 g, const void* received, const void* erased, u64 n, u64 k, u32 batch,
                          const void* msg, const void* status, AnyNttPath* path) {
  if (!ctx || !received || !msg || !status) return set_err(ctx, RONK_EINVAL, "null argument");
  RONK_TRY(rs_args(ctx, p, g, received, n, k, 3 * (u64)batch, path));
  const size_t nr = (size_t)batch * n * 8, ne = (size_t)batch * n, nm = (size_t)batch * k * 8, ns = (size_t)batch * 4;
  if (bytes_overlap(msg, nm, received, nr) || bytes_overlap(msg, nm, erased, ne) || bytes_overlap(status, ns, received, nr) ||
      bytes_overlap(status, ns, erased, ne) || bytes_overlap(msg, nm, status, ns))
    return set_err(ctx, RONK_EINVAL, "output overlaps input");
  if (n - k > kRsMaxParity) return set_err(ctx, RONK_EUNSUPPORTED, "n - k above kRsMaxParity = 8191");
  return RONK_OK;
}

static int rs_decode_device(ronk_ctx* ctx, u64 p, u64 g, const u64* received, const uint8_t* erased, u64 n, u64 k,
                            u32 batch, u64* msg, int32_t* status) {
  AnyNttPath path;
  RONK_TRY(rs_decode_args(ctx, p, g, received, erased, n, k, batch, msg, status, &path));
  if (batch == 0) return RONK_OK;
  const u64 m = n - k, plane = (u64)batch * n;
  const bool literal = path == AN_LITERAL;
  Frame fr(ctx);
  u64 *Y = nullptr, *P = nullptr, *compact = nullptr, *nodes = nullptr;
  RsRow* rows = nullptr;
  RONK_TRY(fr.take(&Y, plane));
  RONK_TRY(fr.take(&P, 3 * plane));
  RONK_TRY(fr.take(&rows, batch));
  if (literal) {
    RONK_TRY(fr.take(&nodes, n));
    RONK_TRY(fr.take(&compact, 3 * (size_t)batch * (m + 1)));
    RONK_TRY(roots_table(ctx, p, g, n, nodes));
  }
  const u64 w = h_powmod(g, (p - 1) / n, p), winv = h_powmod(w, p - 2, p);
  return with_field(ctx, p, 0, false, [&](const auto& f) {
    using F = std::decay_t<decltype(f)>;
    // Y = n^-1 · inverse transform of the rows: S_j = Y[k + j]
    if (literal) {
      RONK_TRY(rs_dft(ctx, f, received, n, n, nodes, n, batch, true, Y));
    } else {
      RONK_CUDA(ctx, cudaMemcpyAsync(Y, received, plane * 8, cudaMemcpyDeviceToDevice, ctx->stream));
      RONK_TRY(anyntt_device(ctx, p, g, Y, n, batch, 1));
    }
    // Ψ, Ψ', Ω: zero-padded to n words in P for the in-place transforms, m + 1 words for rs_dft
    const u64 ld = literal ? m + 1 : n;
    const u32 threads = (u32)std::min<u64>(RS_LOC_MAX_THREADS, std::max<u64>(32, ((m + 1 + RS_LOC_PER - 1) / RS_LOC_PER + 31) / 32 * 32));
    const size_t smem = (3 * m + 2) * sizeof(u64);
    RONK_TRY(ensure_smem_attr(ctx, rs_locator_kernel<F>, (int)((3 * kRsMaxParity + 2) * sizeof(u64))));
    RONK_TRY(launch(ctx, "rs_locator", rs_locator_kernel<F>, batch, threads, smem, false, f, (const u64*)Y, erased, n, k,
                    winv, literal ? compact : P, ld, (u64)batch * ld, rows));
    if (literal)
      RONK_TRY(rs_dft(ctx, f, compact, m + 1, m + 1, nodes, n, 3 * (u64)batch, false, P));
    else
      RONK_TRY(anyntt_device(ctx, p, g, P, n, 3 * batch, 0));
    // R = row - e into Y, then C = n^-1 · inverse transform of R
    RONK_TRY(launch(ctx, "rs_correct", rs_correct_kernel<F>, grid_for(ctx, plane, RS_THREADS), RS_THREADS, 0, false, f,
                    received, (const u64*)P, plane, n, k, w, (p - n % p) % p, rows, Y));
    u64* C = Y;
    if (literal) {
      RONK_TRY(rs_dft(ctx, f, Y, n, n, nodes, n, batch, true, P));
      C = P;
    } else {
      RONK_TRY(anyntt_device(ctx, p, g, Y, n, batch, 1));
    }
    return launch(ctx, "rs_finish", rs_finish_kernel, dim3(batch, (unsigned)((k + RS_FIN_CHUNK - 1) / RS_FIN_CHUNK)), RS_THREADS,
                  0, false, (const u64*)C, n, k, (const RsRow*)rows, msg, status);
  });
}

// ---- decoding at any distinct points (ronk_rs_decode_at_u64) ---------------------------------------------------------
// With m = n - k, M = Π (X - x_i), and I_b the interpolant of row b with its erasures zeroed:
//   S_b(z) = Ĩ_b(z)·T(z) mod z^m, Ĩ_b[t] = I_b[n - 1 - t], T = 1 / (z^n·M(1/z)) mod z^m, the reversal of
//   quo(X^(n+m-1), M); that is S_j = Σ_i r_i·x_i^j / M'(x_i), zero for a codeword (deg f·X^j ≤ n - 2);
//   the locator above (AT) gives σ, σ', Ω̂ and L; one multieval of the 3·batch rows over xs, and M'(x_i) once;
//   rs_forney corrects the roots of σ; C_b = interpolant of (row - e); rs_finish as for ronk_rs_decode_u64.
// Every step is an existing batched entry point or kernel on its own path rule, and none picks its launches by the
// batch save where those entry points do.

// Checks that read no pointer's contents, in the documented order.
static int rs_decode_at_args(ronk_ctx* ctx, u64 p, u64 g, const void* xs, const void* received, const void* erased, u64 n,
                             u64 k, u32 batch, const void* msg, const void* status) {
  if (!ctx || !xs || !received || !msg || !status) return set_err(ctx, RONK_EINVAL, "null argument");
  RONK_TRY(validate_modulus(ctx, p));
  if (g >= p) return set_err(ctx, RONK_EINVAL, "generator out of range");
  if (n == 0 || k == 0 || k > n) return set_err(ctx, RONK_EINVAL, "need 0 < k <= n");
  const u64 m = n - k;
  if (m > kRsMaxParity) return set_err(ctx, RONK_EUNSUPPORTED, "n - k above kRsMaxParity = 8191");
  if (n > kTreeMaxLeaves) return set_err(ctx, RONK_EUNSUPPORTED, "more than 2^24 points");
  if (3 * (u64)batch > 0xFFFFFFFFULL) return set_err(ctx, RONK_EUNSUPPORTED, "3·batch rows above 2^32 - 1");
  bool tree = false;
  if (batch) {  // the path rules divide by the batch
    RONK_TRY(interpolate_path(ctx, p, g, n, batch, &tree));
    RONK_TRY(multieval_path(ctx, p, g, m + 1, 3 * batch, n, &tree));
  }
  if (m && ((u64)batch << log2_ceil(2 * m - 1)) > ((u64)1 << 32))
    return set_err(ctx, RONK_EUNSUPPORTED, "more than 2^32 words of syndrome products");
  const size_t nx = n * 8, nr = (size_t)batch * n * 8, ne = (size_t)batch * n, nm = (size_t)batch * k * 8, ns = (size_t)batch * 4;
  if (bytes_overlap(msg, nm, xs, nx) || bytes_overlap(msg, nm, received, nr) || bytes_overlap(msg, nm, erased, ne) ||
      bytes_overlap(status, ns, xs, nx) || bytes_overlap(status, ns, received, nr) || bytes_overlap(status, ns, erased, ne) ||
      bytes_overlap(msg, nm, status, ns))
    return set_err(ctx, RONK_EINVAL, "output overlaps input");
  return RONK_OK;
}

static int rs_decode_at_device(ronk_ctx* ctx, u64 p, u64 g, const u64* xs, const u64* received, const uint8_t* erased, u64 n,
                               u64 k, u32 batch, u64* msg, int32_t* status) {
  RONK_TRY(rs_decode_at_args(ctx, p, g, xs, received, erased, n, k, batch, msg, status));
  if (batch == 0) return RONK_OK;
  const u64 m = n - k, plane = (u64)batch * n, lp = (u64)batch * (m + 1), ls = m ? 2 * m - 1 : 0;
  // Z: the masked rows, then C | I: the interpolants, then row - e | M, M', M'(x_i) | X^(n+m-1), its quotient and
  // remainder by M, T | Ĩ, S | σ, σ', Ω̂ | their values | rows
  Frame fr(ctx);
  u64* Z = nullptr;
  RONK_TRY(fr.take(&Z, 2 * plane + 3 * n + 1 + (m ? 3 * (n + m) + m : 0) + (u64)batch * (m + ls) + 3 * lp + 3 * plane + 2 * (u64)batch));
  u64* I = Z + plane;
  u64* M = I + plane;
  u64* Mp = M + n + 1;
  u64* W = Mp + n;
  u64* A = W + n;
  u64* Q = A + (m ? n + m : 0);
  u64* Rm = Q + (m ? n + m : 0);
  u64* T = Rm + (m ? n + m : 0);
  u64* IR = T + m;
  u64* S = IR + (u64)batch * m;
  u64* P = S + (u64)batch * ls;
  u64* E = P + 3 * lp;
  RsRow* rows = (RsRow*)(E + 3 * plane);
  const u64* row = received;
  if (erased) {
    RONK_TRY(launch(ctx, "rs_mask", rs_mask_kernel, grid_for(ctx, plane, RS_THREADS), RS_THREADS, 0, false, received, erased,
                    plane, Z));
    row = Z;
  }
  // synchronises; RONK_EINVAL for a repeated point, before anything is written to msg or status
  RONK_TRY(ronk_poly_interpolate_batch_u64(ctx, p, g, xs, row, n, batch, I));
  RONK_TRY(ronk_poly_from_roots_u64(ctx, p, g, xs, n, M));
  RONK_TRY(poly_deriv(ctx, p, M, n, Mp));
  RONK_TRY(ronk_poly_multieval_batch_u64(ctx, p, g, Mp, n, 1, xs, n, W));
  if (m) {
    const u64 one = 1;  // X^(n+m-1) (pageable source: staged before cudaMemcpyAsync returns)
    RONK_CUDA(ctx, cudaMemsetAsync(A, 0, (n + m - 1) * sizeof(u64), ctx->stream));
    RONK_CUDA(ctx, cudaMemcpyAsync(A + n + m - 1, &one, sizeof(u64), cudaMemcpyHostToDevice, ctx->stream));
    RONK_TRY(ronk_poly_divrem_u64(ctx, p, g, A, n + m, M, n + 1, Q, Rm));
    RONK_TRY(reverse_words(ctx, "rs_reverse", Q, m - 1, m, T, m));
    RONK_TRY(reverse_rows(ctx, I, n, n - 1, m, IR, m, m, batch));
    RONK_TRY(ronk_poly_mul_batch_u64(ctx, p, g, IR, m, T, m, 1, batch, S));
  }
  return with_field(ctx, p, 0, false, [&](const auto& f) {
    using F = std::decay_t<decltype(f)>;
    const u32 threads = (u32)std::min<u64>(RS_LOC_MAX_THREADS, std::max<u64>(32, ((m + 1 + RS_LOC_PER - 1) / RS_LOC_PER + 31) / 32 * 32));
    RONK_TRY(ensure_smem_attr(ctx, rs_locator_at_kernel<F>, (int)((3 * kRsMaxParity + 2) * sizeof(u64))));
    RONK_TRY(launch(ctx, "rs_locator_at", rs_locator_at_kernel<F>, batch, threads, (3 * m + 2) * sizeof(u64), false, f,
                    (const u64*)S, ls, xs, erased, n, k, P, m + 1, lp, rows));
    RONK_TRY(ronk_poly_multieval_batch_u64(ctx, p, g, P, m + 1, 3 * batch, xs, n, E));
    RONK_TRY(launch(ctx, "rs_forney", rs_forney_kernel<F>, grid_for(ctx, plane, RS_THREADS), RS_THREADS, 0, false, f, row,
                    (const u64*)E, plane, (const u64*)W, n, rows, I));
    RONK_TRY(ronk_poly_interpolate_batch_u64(ctx, p, g, xs, I, n, batch, Z));
    return launch(ctx, "rs_finish", rs_finish_kernel, dim3(batch, (unsigned)((k + RS_FIN_CHUNK - 1) / RS_FIN_CHUNK)), RS_THREADS,
                  0, false, (const u64*)Z, n, k, (const RsRow*)rows, msg, status);
  });
}

}  // namespace ronk

using namespace ronk;

extern "C" int ronk_rs_decode_at_u64(ronk_ctx* ctx, uint64_t p, uint64_t g, const uint64_t* xs, const uint64_t* received,
                                     const uint8_t* erased, uint64_t n, uint64_t k, uint32_t batch, uint64_t* msg,
                                     int32_t* status) {
  ronk::DeviceGuard _dg(ctx);
  return rs_decode_at_device(ctx, p, g, (const u64*)xs, (const u64*)received, erased, n, k, batch, (u64*)msg, status);
}

extern "C" int ronk_rs_decode_at_u64_host(ronk_ctx* ctx, uint64_t p, uint64_t g, const uint64_t* xs, const uint64_t* received,
                                          const uint8_t* erased, uint64_t n, uint64_t k, uint32_t batch, uint64_t* msg,
                                          int32_t* status) {
  ronk::DeviceGuard _dg(ctx);
  RONK_TRY(rs_decode_at_args(ctx, p, g, xs, received, erased, n, k, batch, msg, status));  // before staging
  for (u64 i = 0; i < n; i++)
    if (xs[i] >= p) return set_err(ctx, RONK_EINVAL, "point out of range (x >= p)");
  if (batch == 0) return RONK_OK;
  Staged s[] = {{n * 8, xs},
                {(size_t)batch * n * 8, received},
                {erased ? (size_t)batch * n : 0, erased},
                {(size_t)batch * k * 8, nullptr, msg},
                {(size_t)batch * 4, nullptr, status}};
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  return stage_out(ctx,
                   rs_decode_at_device(ctx, p, g, s[0].dev, s[1].dev, erased ? (const uint8_t*)s[2].dev : nullptr, n, k, batch,
                                       s[3].dev, (int32_t*)s[4].dev),
                   s);
}

extern "C" int ronk_rs_encode_u64(ronk_ctx* ctx, uint64_t p, uint64_t g, const uint64_t* msg, uint64_t k, uint64_t n,
                                  uint32_t batch, uint64_t* codeword) {
  ronk::DeviceGuard _dg(ctx);
  return rs_encode_device(ctx, p, g, (const u64*)msg, k, n, batch, (u64*)codeword);
}

extern "C" int ronk_rs_decode_u64(ronk_ctx* ctx, uint64_t p, uint64_t g, const uint64_t* received, const uint8_t* erased,
                                  uint64_t n, uint64_t k, uint32_t batch, uint64_t* msg, int32_t* status) {
  ronk::DeviceGuard _dg(ctx);
  return rs_decode_device(ctx, p, g, (const u64*)received, erased, n, k, batch, (u64*)msg, status);
}

extern "C" int ronk_rs_decode_u64_host(ronk_ctx* ctx, uint64_t p, uint64_t g, const uint64_t* received,
                                       const uint8_t* erased, uint64_t n, uint64_t k, uint32_t batch, uint64_t* msg,
                                       int32_t* status) {
  ronk::DeviceGuard _dg(ctx);
  AnyNttPath path;
  RONK_TRY(rs_decode_args(ctx, p, g, received, erased, n, k, batch, msg, status, &path));  // before staging
  if (batch == 0) return RONK_OK;
  Staged s[] = {{(size_t)batch * n * 8, received, nullptr},
                {erased ? (size_t)batch * n : 0, erased, nullptr},
                {(size_t)batch * k * 8, nullptr, msg},
                {(size_t)batch * 4, nullptr, status}};
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  return stage_out(ctx,
                   rs_decode_device(ctx, p, g, s[0].dev, erased ? (const uint8_t*)s[1].dev : nullptr, n, k, batch, s[2].dev,
                                    (int32_t*)s[3].dev),
                   s);
}
