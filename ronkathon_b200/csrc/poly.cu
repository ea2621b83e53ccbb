// poly.cu — Polynomial<Monomial|Lagrange, F, D> operations other than the transforms.
// Mirrors src/polynomial/arithmetic.rs (Add :16-35, Sub :49-68, Mul :97-119, Div/Rem :121-146) and
// src/polynomial/mod.rs (evaluate :133-139, quotient_and_remainder :170-225, dft :240-258,
// Lagrange evaluate :382-415).
#include "ntt_kernel.cuh"
#include "ronk_internal.h"

namespace ronk {

// out[i] = a[i] ± (i < db ? b[i] : 0), i < da   (arithmetic.rs:23-34 / :56-67)
template <class F, bool SUB>
__global__ void poly_addsub_kernel(const F f, const u64* a, size_t da, const u64* b, size_t db, u64* out) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < da; i += stride) {
    const u64 y = (i < db) ? b[i] : 0ULL;
    out[i] = SUB ? f.sub(a[i], y) : f.add(a[i], y);
  }
}

// Schoolbook product (arithmetic.rs:110-118) of `total / L` contiguous rows: c[r] = a[r]·b[r] (b_stride = db) or
// a[r]·b (b_stride = 0), one thread per output coefficient.  A single product is one row (total = L).
template <class F>
__global__ void poly_mul_schoolbook_kernel(const F f, const u64* a, size_t da, const u64* b, size_t db, size_t b_stride,
                                           u64* c, u64 total) {
  const size_t L = da + db - 1;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (u64 o = (size_t)blockIdx.x * blockDim.x + threadIdx.x; o < total; o += stride) {
    const u64 r = total == L ? 0 : (total >> 32) ? o / L : (u32)o / (u32)L;
    const size_t k = o - r * L;
    const u64* ar = a + r * da;
    const u64* br = b + r * b_stride;
    const size_t lo = (k >= db) ? k - db + 1 : 0, hi = (k < da) ? k : da - 1;
    u64 acc = 0;
    for (size_t i = lo; i <= hi; i++) acc = f.add(acc, f.mul(ar[i], br[k - i]));
    c[o] = acc;
  }
}

// evaluate (mod.rs:133-139): out[b·m + pt] = Σ_j c[b·d + j] x^j, m = gridDim.x, for the rows b < rows (blockIdx.y,
// stepping by gridDim.y).  One CTA per point; thread t owns the coefficients j ≡ t (mod 256) (coalesced), Horner in
// x^256, then a shared-memory tree sum.  The powers of x are formed once for all the CTA's rows.
template <class F>
__global__ void poly_eval_kernel(const F f, const u64* c, size_t d, const u64* xs, u32 rows, u64* out) {
  __shared__ u64 red[256];
  const u32 t = threadIdx.x;
  const u64 x = xs[blockIdx.x];
  const u64 y = field_pow(f, x, 256);
  const u64 xt = t < d ? field_pow(f, x, (u64)t) : 0ULL;
  for (u64 b = blockIdx.y; b < rows; b += gridDim.y) {
    const u64* cb = c + b * d;
    u64 acc = 0;
    if (t < d) {
      const size_t kmax = (d - 1 - t) / 256;
      for (size_t k = kmax + 1; k-- > 0;) acc = f.add(f.mul(acc, y), cb[t + 256 * k]);
      acc = f.mul(acc, xt);
    }
    red[t] = acc;
    __syncthreads();
    for (u32 s = 128; s > 0; s >>= 1) {
      if (t < s) red[t] = f.add(red[t], red[t + s]);
      __syncthreads();
    }
    if (t == 0) out[b * gridDim.x + blockIdx.x] = red[0];
  }
}

// Lagrange-basis evaluate (mod.rs:382-415), literal fold semantics: the closure's early
// `return c` replaces the accumulator, and l(x) multiplies the fold afterwards.
template <class F>
__global__ void lagrange_eval_kernel(const F f, const u64* c, const u64* nodes, u32 n, u64 x, u64* out, int* flag) {
  __shared__ u64 red[256];
  __shared__ u64 lred[256];
  __shared__ u32 hit;  // index j* with nodes[j*] == x, or n
  const u32 t = threadIdx.x;
  if (t == 0) hit = n;
  __syncthreads();
  for (u32 j = t; j < n; j += blockDim.x)
    if (nodes[j] == x) hit = j;
  __syncthreads();
  const u32 jstar = hit;
  u64 acc = 0, lx = 1 % f.modulus();
  for (u32 j = t; j < n; j += blockDim.x) {
    lx = f.mul(lx, f.sub(x, nodes[j]));
    // The reference builds EVERY weight first (mod.rs:386-393), so a repeated node panics in F::ONE.div
    // whatever x is — also for the terms the fold later discards.
    u64 wden = 1 % f.modulus();  // w_j^-1 = Π_{m≠j} (x_j - x_m)
    for (u32 m = 0; m < n; m++)
      if (m != j) wden = f.mul(wden, f.sub(nodes[j], nodes[m]));
    if (wden == 0) { atomicExch(flag, 1); continue; }
    if (jstar < n && j <= jstar) {
      if (j == jstar) acc = f.add(acc, c[j]);
      continue;
    }
    const u64 den = f.mul(wden, f.sub(x, nodes[j]));
    if (den == 0) { atomicExch(flag, 1); continue; }
    acc = f.add(acc, f.mul(c[j], field_pow(f, den, f.modulus() - 2)));
  }
  red[t] = acc;
  lred[t] = lx;
  __syncthreads();
  for (u32 s = blockDim.x / 2; s > 0; s >>= 1) {
    if (t < s) {
      red[t] = f.add(red[t], red[t + s]);
      lred[t] = f.mul(lred[t], lred[t + s]);
    }
    __syncthreads();
  }
  if (t == 0) out[0] = f.mul(lred[0], red[0]);
}

// quotient_and_remainder (mod.rs:170-225) of one row by the whole CTA; q and r have da terms.
// flag: 1 = all-zero divisor / non-invertible, 2 = index out of range (the reference panics).
template <class F>
__device__ __forceinline__ void divrem_row(const F& f, const u64* a, u32 da, const u64* b, u32 db, u64* q, u64* r, int* flag) {
  __shared__ u32 s_deg, s_ok;
  __shared__ u64 s_s;
  const u32 t = threadIdx.x, nt = blockDim.x;
  for (u32 i = t; i < da; i += nt) { q[i] = 0; r[i] = a[i]; }
  __shared__ u32 s_rdeg, s_rfound;
  if (t == 0) { s_rfound = 0; s_rdeg = 0; }
  __syncthreads();
  for (u32 i = t; i < db; i += nt)
    if (b[i] != 0) { atomicMax(&s_rdeg, i); s_rfound = 1; }
  __syncthreads();
  const u32 rhs_degree = s_rdeg;
  const bool rhs_nonzero = s_rfound != 0;
  u64 cinv = 0;
  if (rhs_nonzero) cinv = field_pow(f, b[rhs_degree], f.modulus() - 2);
  u32 plen = da;  // p_coeffs.len() after trim_zeros
  while (true) {
    // find degree of the (trimmed) dividend: highest nonzero below plen
    if (t == 0) { s_deg = 0; s_ok = 0; }
    __syncthreads();
    for (u32 i = t; i < plen; i += nt)
      if (r[i] != 0) { atomicMax(&s_deg, i); s_ok = 1; }
    __syncthreads();
    const bool any = s_ok != 0;
    const u32 p_degree = s_deg;
    if (!(any && plen >= db)) break;                       // :183-184
    if (!rhs_nonzero) { if (t == 0) atomicExch(flag, 1); break; }  // rposition().unwrap()
    if (p_degree < rhs_degree) break;                      // :190-192
    const u32 diff = p_degree - rhs_degree;
    if (diff + db > plen) { if (t == 0) atomicExch(flag, 2); break; }  // p_coeffs[diff + i] out of range
    __syncthreads();
    if (t == 0) { s_s = f.mul(r[p_degree], cinv); q[diff] = s_s; }
    __syncthreads();
    const u64 s = s_s;
    for (u32 i = t; i < db; i += nt) r[diff + i] = f.sub(r[diff + i], f.mul(b[i], s));
    __syncthreads();
    plen = p_degree;  // coefficient p_degree is now 0; trim_zeros continues below via the next scan
    // trim_zeros pops every trailing zero: the next iteration's scan finds the new top, and
    // plen must equal (new top + 1) for the `plen >= db` test.
    if (t == 0) { s_deg = 0; s_ok = 0; }
    __syncthreads();
    for (u32 i = t; i < plen; i += nt)
      if (r[i] != 0) { atomicMax(&s_deg, i); s_ok = 1; }
    __syncthreads();
    plen = s_ok ? s_deg + 1 : 0;
    __syncthreads();
  }
}

// Single CTA, one row.
template <class F>
__global__ void poly_divrem_kernel(const F f, const u64* a, u32 da, const u64* b, u32 db, u64* q, u64* r, int* flag) {
  divrem_row(f, a, da, b, db, q, r, flag);
}

// `batch` rows (a, q, r: batch × da; b: rows b_stride apart, 0 for one shared divisor), one CTA per row, stepping by
// gridDim.y.  The barrier keeps a fast thread's next row from resetting the shared scalars a slow one still reads.
template <class F>
__global__ void poly_divrem_rows_kernel(const F f, const u64* a, u32 da, const u64* b, u32 db, u64 b_stride, u32 batch, u64* q,
                                        u64* r, int* flag) {
  for (u64 row = blockIdx.y; row < batch; row += gridDim.y) {
    divrem_row(f, a + row * da, da, b + row * b_stride, db, q + row * da, r + row * da, flag);
    __syncthreads();
  }
}


// ---- division by a linear factor (b0 + b1·x), §8f row 1 ------------------------------------------
// quotient_and_remainder (mod.rs:170-225) specialised to the divisor kzg::open builds
// (kzg/setup.rs:72-75: [-z, 1]).  With z = -b0/b1 the long division is the suffix recurrence
//   h_j = a_j + z·h_{j+1}  (h_d = 0),   q_j = h_{j+1} / b1,   r = h_0 = a(z),
// a first-order linear recurrence, i.e. a scan: (1) every chunk of 4096 coefficients is folded to
// its Horner value S_c = Σ a_{c0+i} z^i, (2) one CTA turns the S_c into the carry-in of every chunk,
// (3) every chunk redoes its local scan seeded with the carry and writes q.  2 reads + 1 write per
// coefficient; the general single-CTA kernel above needs O(D) sequential steps for the same result.
constexpr int DL_THR = 256, DL_PER = 16, DL_CHUNK = DL_THR * DL_PER;
RONK_DEV u32 dl_pad(u32 i) { return i + (i >> 4); }  // 16-word rows padded to 17: conflict-free both ways

template <class F>
RONK_DEV u64 pow2k_tw(const F& f, u64 x_tw, int k) {  // x^(2^k), twiddle form in and out
  for (int i = 0; i < k; i++) x_tw = f.mul_tw(x_tw, x_tw);
  return x_tw;
}

template <class F, bool APPLY>
__device__ __forceinline__ void div_linear_chunk(const F& f, const u64* __restrict__ a, u64 d, u64 z, const u64* __restrict__ carry,
                                                 u64* __restrict__ S, u64 scale, u64* __restrict__ q, u64* __restrict__ rem) {
  __shared__ u64 tile[DL_CHUNK + DL_CHUNK / 16];
  __shared__ u64 v[DL_THR + 1];
  const u32 tid = threadIdx.x;
  const u64 c0 = (u64)blockIdx.x * DL_CHUNK;
  const u64 z_tw = f.to_tw(z);
  for (u32 i = tid; i < (u32)DL_CHUNK; i += DL_THR) tile[dl_pad(i)] = (c0 + i < d) ? a[c0 + i] : 0ULL;  // coalesced
  __syncthreads();
  u64 x[DL_PER];
#pragma unroll
  for (int k = 0; k < DL_PER; k++) x[k] = tile[dl_pad(tid * DL_PER + k)];
  u64 t = 0;  // Σ_k x[k] z^k
#pragma unroll
  for (int k = DL_PER - 1; k >= 0; k--) t = f.add(x[k], f.mul_tw(t, z_tw));
  v[tid] = t;
  if (tid == 0) v[DL_THR] = APPLY ? carry[blockIdx.x] : 0ULL;  // element 256 = carry into this chunk
  u64 M = pow2k_tw(f, z_tw, 4);                                  // z^16
  for (u32 off = 1; off <= (u32)DL_THR; off <<= 1) {             // suffix scan, uniform multiplier per level
    __syncthreads();
    const bool on = tid + off <= (u32)DL_THR;
    const u64 other = on ? v[tid + off] : 0ULL;
    __syncthreads();
    if (on) v[tid] = f.add(v[tid], f.mul_tw(other, M));
    M = f.mul_tw(M, M);
  }
  __syncthreads();
  if (!APPLY) {
    if (tid == 0) S[blockIdx.x] = v[0];
    return;
  }
  const u64 s_tw = f.to_tw(scale);
  u64 run = v[tid + 1];  // h at the first index above this thread's range
#pragma unroll
  for (int k = DL_PER - 1; k >= 0; k--) {
    run = f.add(x[k], f.mul_tw(run, z_tw));  // h_{base+k}
    x[k] = run;
  }
  if (blockIdx.x == 0 && tid == 0) rem[0] = x[0];  // r = h_0 (not scaled: a = q·(b1·x + b0) + r)
#pragma unroll
  for (int k = 0; k < DL_PER; k++) tile[dl_pad(tid * DL_PER + k)] = f.mul_tw(x[k], s_tw);
  __syncthreads();
  // q_j = h_{j+1}/b1: h at chunk position i goes to q[c0 + i - 1]; the top coefficient q_{d-1} is 0
  for (u32 i = tid; i < (u32)DL_CHUNK; i += DL_THR) {
    const u64 j = c0 + i;
    if (j >= 1 && j < d) q[j - 1] = tile[dl_pad(i)];
  }
  if (c0 + DL_CHUNK >= d && c0 < d && tid == 0) q[d - 1] = 0ULL;
}

template <class F, bool APPLY>
__global__ void __launch_bounds__(DL_THR)
div_linear_kernel(const F f, const u64* __restrict__ a, u64 d, u64 z, const u64* __restrict__ carry, u64* __restrict__ S,
                  u64 scale, u64* __restrict__ q, u64* __restrict__ rem) {
  div_linear_chunk<F, APPLY>(f, a, d, z, carry, S, scale, q, rem);
}

// carry[c] = Σ_{c' > c} S_{c'} Z^{c'-c-1}, Z = z^4096.  One CTA: every thread owns a contiguous block of
// chunks (local Horner), thread 0 chains the ≤ 1024 block values, then every thread replays its block.
template <class F>
__device__ __forceinline__ void div_linear_carries(const F& f, const u64* __restrict__ S, u32 nchunks, u64 z, u64* __restrict__ carry) {
  __shared__ u64 L[1024];
  __shared__ u64 G[1025];
  const u32 t = threadIdx.x;
  const u64 Z = pow2k_tw(f, f.to_tw(z), 12);
  const u32 B = (nchunks + 1023) / 1024;
  const u32 lo = (u32)min((u64)t * B, (u64)nchunks), hi = (u32)min((u64)lo + B, (u64)nchunks);
  u64 acc = 0;
  for (u32 c = hi; c-- > lo;) acc = f.add(S[c], f.mul_tw(acc, Z));
  L[t] = acc;
  __syncthreads();
  if (t == 0) {
    u64 ZB = f.to_tw(1 % f.modulus());  // Z^B
    {
      u64 base = Z;
      for (u32 e = B; e; e >>= 1) {
        if (e & 1) ZB = f.mul_tw(ZB, base);
        base = f.mul_tw(base, base);
      }
    }
    u64 g = 0;
    G[1024] = 0;
    for (u32 i = 1024; i-- > 0;) {
      g = f.add(L[i], f.mul_tw(g, ZB));
      G[i] = g;  // Horner value of all chunks from block i upwards
    }
  }
  __syncthreads();
  u64 run = G[t + 1];
  for (u32 c = hi; c-- > lo;) {
    carry[c] = run;
    run = f.add(S[c], f.mul_tw(run, Z));
  }
}

template <class F>
__global__ void __launch_bounds__(1024)
div_linear_carry_kernel(const F f, const u64* __restrict__ S, u32 nchunks, u64 z, u64* __restrict__ carry) {
  div_linear_carries(f, S, nchunks, z, carry);
}

// The three kernels above over `batch` rows of d words (a, q, rem: rows d apart; S, carry: rows nchunks apart), row y
// stepping by gridDim.y, dividing by its own linear factor: zs[y·zstride] = b1^-1 and zs[y·zstride + 1] = z (zstride 0
// for one shared divisor).  rem[y·d] = a_y(z).  The barrier keeps one row's shared-memory reads ahead of the next row's
// writes.
template <class F, bool APPLY>
__global__ void __launch_bounds__(DL_THR)
div_linear_rows_kernel(const F f, const u64* __restrict__ a, u64 d, const u64* __restrict__ zs, u32 zstride, u32 batch,
                       const u64* __restrict__ carry, u64* __restrict__ S, u64 nchunks, u64* __restrict__ q, u64* __restrict__ rem) {
  for (u64 y = blockIdx.y; y < batch; y += gridDim.y) {
    const u64 scale = zs[y * zstride], z = zs[y * zstride + 1];
    div_linear_chunk<F, APPLY>(f, a + y * d, d, z, APPLY ? carry + y * nchunks : nullptr, APPLY ? nullptr : S + y * nchunks,
                               scale, APPLY ? q + y * d : nullptr, APPLY ? rem + y * d : nullptr);
    __syncthreads();
  }
}

template <class F>
__global__ void __launch_bounds__(1024)
div_linear_rows_carry_kernel(const F f, const u64* __restrict__ S, u32 nchunks, const u64* __restrict__ zs, u32 zstride, u32 batch,
                             u64* __restrict__ carry) {
  for (u64 y = blockIdx.y; y < batch; y += gridDim.y) {
    div_linear_carries(f, S + y * nchunks, nchunks, zs[y * zstride + 1], carry + y * nchunks);
    __syncthreads();
  }
}

template <class F>
static int div_linear_with_field(ronk_ctx* ctx, const F& f, const u64* a, size_t d, u64 z, u64 scale, u64* q, u64* rem) {
  const size_t nchunks = (d + DL_CHUNK - 1) / DL_CHUNK;
  if (nchunks > 0x7FFFFFFFULL) return set_err(ctx, RONK_EUNSUPPORTED, "polynomial too long");
  Frame fr(ctx);
  u64* S = nullptr;
  RONK_TRY(fr.take(&S, 2 * nchunks));
  u64* carry = S + nchunks;
  RONK_TRY(launch(ctx, "div_linear_fold", div_linear_kernel<F, false>, (u32)nchunks, DL_THR, 0, false, f, a, d, z, nullptr, S,
                  scale, nullptr, nullptr));
  RONK_TRY(launch(ctx, "div_linear_carry", div_linear_carry_kernel<F>, 1, 1024, 0, false, f, S, (u32)nchunks, z, carry));
  return launch(ctx, "div_linear_apply", div_linear_kernel<F, true>, (u32)nchunks, DL_THR, 0, false, f, a, d, z, carry, nullptr,
                scale, q, rem);
}

// a / (b0 + b1·x): q (d terms, top one 0) and the scalar remainder, all device pointers; q may not alias a.
static int div_linear_device(ronk_ctx* ctx, u64 p, const u64* a, size_t d, u64 b0, u64 b1, u64* q, u64* rem) {
  if (!ctx || !a || !q || !rem) return set_err(ctx, RONK_EINVAL, "null argument");
  if (q == a) return set_err(ctx, RONK_EINVAL, "the quotient may not alias the dividend");
  RONK_TRY(validate_modulus(ctx, p));
  if (d == 0) return set_err(ctx, RONK_EINVAL, "empty dividend");
  if (b0 >= p || b1 >= p) return set_err(ctx, RONK_EINVAL, "non-canonical divisor coefficient");
  if (b1 == 0) return set_err(ctx, RONK_EINVAL, "divisor is not linear (leading coefficient 0)");
  const u64 b1inv = h_powmod(b1, p - 2, p);
  const u64 z = h_mulmod(b0 ? p - b0 : 0, b1inv, p);
  return with_field(ctx, p, 0, false, [&](const auto& f) { return div_linear_with_field(ctx, f, a, d, z, b1inv, q, rem); });
}

// quotient_and_remainder (mod.rs:170-225) on device pointers, q and r of da words.  The host reads b[db-1] to choose:
// a zero top word keeps the reference's quirks (literal kernel); otherwise the division is Euclidean and goes to the
// cheapest exact path — nothing to do for da < db, the scan for a linear divisor, Newton iteration on the transforms
// when every transform size divides p - 1, else the literal kernel.
static int divrem_device(ronk_ctx* ctx, u64 p, u64 g, const u64* a, size_t da, const u64* b, size_t db, u64* q, u64* r) {
  if (!ctx || (da && (!a || !q || !r)) || (db && !b)) return set_err(ctx, RONK_EINVAL, "null argument");
  RONK_TRY(validate_modulus(ctx, p));
  if (g >= p) return set_err(ctx, RONK_EINVAL, "generator out of range");
  if (da > 0x7FFFFFF0ULL || db > 0x7FFFFFF0ULL) return set_err(ctx, RONK_EUNSUPPORTED, "polynomial too long");
  if (da == 0) return RONK_OK;
  if (overlaps(q, da, a, da) || overlaps(q, da, b, db) || overlaps(r, da, a, da) || overlaps(r, da, b, db) ||
      overlaps(q, da, r, da))
    return set_err(ctx, RONK_EINVAL, "q and r may not alias a, b or each other");
  u64 lo = 0, top = 0;  // b[0] (linear divisors only) and b[db-1]; an empty divisor counts as zero
  if (db) {
    RONK_CUDA(ctx, cudaMemcpyAsync(&top, b + db - 1, sizeof(u64), cudaMemcpyDeviceToHost, ctx->stream));
    if (db == 2) RONK_CUDA(ctx, cudaMemcpyAsync(&lo, b, sizeof(u64), cudaMemcpyDeviceToHost, ctx->stream));
    RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  }
  if (top != 0 && da < db) {  // the reference's loop never runs
    RONK_CUDA(ctx, cudaMemsetAsync(q, 0, da * sizeof(u64), ctx->stream));
    RONK_CUDA(ctx, cudaMemcpyAsync(r, a, da * sizeof(u64), cudaMemcpyDeviceToDevice, ctx->stream));
  } else if (top != 0 && db == 2 && top < p && lo < p) {
    RONK_CUDA(ctx, cudaMemsetAsync(r, 0, da * sizeof(u64), ctx->stream));
    RONK_TRY(div_linear_device(ctx, p, a, da, lo, top, q, r));
  } else if (top != 0 && divrem_newton_fits(p, g, da, db)) {
    RONK_TRY(divrem_newton_device(ctx, p, g, a, da, b, db, top, q, r));
  } else {  // the literal long division
    RONK_TRY(reset_flag(ctx));
    RONK_TRY(with_field(ctx, p, 0, false, [&](const auto& f) {
      return launch(ctx, "poly_divrem", poly_divrem_kernel<std::decay_t<decltype(f)>>, 1, 256, 0, false, f, a, (u32)da, b,
                    (u32)db, q, r, ctx->d_flag.get());
    }));
    int v = 0;
    RONK_TRY(read_flag(ctx, &v));  // synchronises the stream
    if (v) return set_err(ctx, RONK_EINVAL, "polynomial division: the reference would panic on this divisor");
    return RONK_OK;
  }
  RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return RONK_OK;
}

// The single-row entries are batch = 1 without `reserve`; the batched ones take all the call's scratch before the first
// launch (reserve), so that what follows fits the blocks that take leaves.
static int reserve_scratch(ronk_ctx* ctx, size_t words) {
  Frame fr(ctx);
  u64* all = nullptr;
  return fr.take(&all, words);
}

// ---- batches of divisions (ronk_poly_divrem_batch_u64) -------------------------------------------------------------
// flag = 1 when any of the batch rows of b (db words each, db ≥ 1) has a zero top word
__global__ void divrem_top_scan_kernel(const u64* __restrict__ b, size_t db, u32 batch, int* flag) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t y = (size_t)blockIdx.x * blockDim.x + threadIdx.x; y < batch; y += stride)
    if (b[y * db + db - 1] == 0) atomicExch(flag, 1);
}

enum DivremBatchPath { DB_COPY, DB_LINEAR, DB_NEWTON, DB_LITERAL };

constexpr u64 kDivremBatchMaxWords = (u64)1 << 40, kDivremBatchMaxTransformWords = (u64)1 << 32;

// Newton iteration or the literal kernel, from batch 2, for rows whose top words are nonzero (da ≥ db, db != 2).  The
// literal kernel runs one CTA per row, sm_count·8 rows at a time, each about L sequential steps over the dividend's
// shrinking top; Newton costs at least about 0.3 ms (its launches and transforms) and won wherever the literal estimate
// passed that.  tools/divrem_batch_timing.py on an H100 80GB HBM3 at 700 W (DESIGN.md §5), Goldilocks: the literal
// kernel took about 0.09 ms per wave of rows plus 1 µs per 2000 words of L·(da + db) (64 × 17: 0.10 ms, 256 × 17:
// 0.21, 1024 × 17: 1.02, 4096 × 2049: 8.5), Newton 0.22 … 0.47 ms up to da = 1024 at up to 4096 rows.  On BabyBear
// (the Montgomery policy) both cost 10–40 % more and cross at the same shapes, so one rule serves both policies.
static bool divrem_batch_newton(const ronk_ctx* ctx, u64 p, u64 g, size_t da, size_t db, u32 batch) {
  if (!divrem_newton_fits(p, g, da, db)) return false;
  if (ctx->tune.divrem_batch_path) return ctx->tune.divrem_batch_path == 2;
  const u64 L = da - db + 1, slots = (u64)ctx->sm_count * 8, waves = (batch + slots - 1) / slots;
  return waves * (90 + L * (da + db) / 2000) >= 300;  // µs; da, db ≤ 2^26 where Newton fits
}

// The checks that read no pointer, in the header's order, and the path of rows whose top words are nonzero.
static int divrem_batch_args(ronk_ctx* ctx, u64 p, u64 g, bool null_arg, size_t da, size_t db, bool b_shared, u32 batch,
                             DivremBatchPath* path) {
  if (!ctx || null_arg) return set_err(ctx, RONK_EINVAL, "null argument");
  RONK_TRY(validate_modulus(ctx, p));
  if (g >= p) return set_err(ctx, RONK_EINVAL, "generator out of range");
  if (da > 0x7FFFFFF0ULL || db > 0x7FFFFFF0ULL) return set_err(ctx, RONK_EUNSUPPORTED, "polynomial too long");
  if ((u64)batch * da > kDivremBatchMaxWords || (b_shared ? db : (u64)batch * db) > kDivremBatchMaxWords)
    return set_err(ctx, RONK_EUNSUPPORTED, "more than 2^40 words in a, b, q or r");
  *path = db == 0 ? DB_LITERAL : da < db ? DB_COPY : db == 2 ? DB_LINEAR
          : batch > 1 && divrem_batch_newton(ctx, p, g, da, db, batch) ? DB_NEWTON : DB_LITERAL;
  if (*path == DB_NEWTON && divrem_newton_rows_transform_words(da, db, batch) > kDivremBatchMaxTransformWords)
    return set_err(ctx, RONK_EUNSUPPORTED, "more than 2^32 words of batched transforms");
  return RONK_OK;
}

static int divrem_batch_device(ronk_ctx* ctx, u64 p, u64 g, const u64* a, size_t da, const u64* b, size_t db, bool b_shared,
                               u32 batch, u64* q, u64* r) {
  const bool empty = batch == 0 || da == 0;
  DivremBatchPath path;
  RONK_TRY(divrem_batch_args(ctx, p, g, !empty && (!a || !q || !r || (db && !b)), da, db, b_shared, batch, &path));
  if (empty) return RONK_OK;
  const size_t na = (size_t)batch * da, nb = b_shared ? db : (size_t)batch * db;
  if (overlaps(q, na, a, na) || overlaps(q, na, b, nb) || overlaps(r, na, a, na) || overlaps(r, na, b, nb) || overlaps(q, na, r, na))
    return set_err(ctx, RONK_EINVAL, "q and r may not alias a, b or each other");
  if (batch == 1) return divrem_device(ctx, p, g, a, da, b, db, q, r);
  // the divisors' top words (and a shared linear divisor's b[0]), once for all rows
  u64 lo_top[2] = {0, 0};
  if (db && b_shared) {
    const size_t w = db == 2 ? 2 : 1;
    RONK_CUDA(ctx, cudaMemcpyAsync(lo_top + 2 - w, b + db - w, w * sizeof(u64), cudaMemcpyDeviceToHost, ctx->stream));
    RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (lo_top[1] == 0) path = DB_LITERAL;
  } else if (db) {
    RONK_TRY(reset_flag(ctx));
    RONK_TRY(launch(ctx, "divrem_top_scan", divrem_top_scan_kernel, grid_for(ctx, batch, 256), 256, 0, false, b, db, batch,
                    ctx->d_flag.get()));
    int zero = 0;
    RONK_TRY(read_flag(ctx, &zero));
    if (zero) path = DB_LITERAL;
  }
  const size_t bs = b_shared ? 0 : db;
  if (path == DB_COPY) {  // the reference's loop never runs
    RONK_CUDA(ctx, cudaMemsetAsync(q, 0, na * sizeof(u64), ctx->stream));
    RONK_CUDA(ctx, cudaMemcpyAsync(r, a, na * sizeof(u64), cudaMemcpyDeviceToDevice, ctx->stream));
  } else if (path == DB_LINEAR) {
    const size_t nchunks = (da + DL_CHUNK - 1) / DL_CHUNK;
    Frame fr(ctx);
    u64* S = nullptr;
    RONK_TRY(fr.take(&S, 2 * (size_t)batch * nchunks + (b_shared ? 2 : 2 * (size_t)batch)));
    u64* carry = S + (size_t)batch * nchunks;
    u64* zs = carry + (size_t)batch * nchunks;  // [b1^-1, z] per row, or once
    if (b_shared) {  // pageable source: staged before cudaMemcpyAsync returns
      const u64 inv = h_powmod(lo_top[1], p - 2, p), z_inv[2] = {inv, h_mulmod(lo_top[0] ? p - lo_top[0] : 0, inv, p)};
      RONK_CUDA(ctx, cudaMemcpyAsync(zs, z_inv, sizeof(z_inv), cudaMemcpyHostToDevice, ctx->stream));
    } else {
      RONK_TRY(divrem_top_inverses(ctx, p, b, db, batch, zs));
    }
    RONK_CUDA(ctx, cudaMemsetAsync(r, 0, na * sizeof(u64), ctx->stream));
    const u32 zstride = b_shared ? 0 : 2;
    RONK_TRY(with_field(ctx, p, 0, false, [&](const auto& f) {
      using F = std::decay_t<decltype(f)>;
      const dim3 grid((u32)nchunks, grid_rows(ctx, batch, nchunks));
      RONK_TRY(launch(ctx, "div_linear_fold", div_linear_rows_kernel<F, false>, grid, DL_THR, 0, false, f, a, (u64)da,
                      (const u64*)zs, zstride, batch, (const u64*)nullptr, S, (u64)nchunks, (u64*)nullptr, (u64*)nullptr));
      RONK_TRY(launch(ctx, "div_linear_carry", div_linear_rows_carry_kernel<F>, dim3(1, grid_rows(ctx, batch, 1)), 1024, 0, false, f,
                      (const u64*)S, (u32)nchunks, (const u64*)zs, zstride, batch, carry));
      return launch(ctx, "div_linear_apply", div_linear_rows_kernel<F, true>, grid, DL_THR, 0, false, f, a, (u64)da, (const u64*)zs,
                    zstride, batch, (const u64*)carry, (u64*)nullptr, (u64)nchunks, q, r);
    }));
  } else if (path == DB_NEWTON) {
    RONK_TRY(reserve_scratch(ctx, divrem_newton_rows_scratch(da, db, b_shared, batch)));
    RONK_TRY(divrem_newton_rows(ctx, p, g, a, da, b, db, b_shared, batch, lo_top[1], q, r));
  } else {  // the literal long division, also for every row when any top word is zero
    RONK_TRY(reset_flag(ctx));
    RONK_TRY(with_field(ctx, p, 0, false, [&](const auto& f) {
      return launch(ctx, "poly_divrem_rows", poly_divrem_rows_kernel<std::decay_t<decltype(f)>>, dim3(1, grid_rows(ctx, batch, 1)),
                    256, 0, false, f, a, (u32)da, b, (u32)db, (u64)bs, batch, q, r, ctx->d_flag.get());
    }));
    int v = 0;
    RONK_TRY(read_flag(ctx, &v));  // synchronises the stream
    if (v) return set_err(ctx, RONK_EINVAL, "polynomial division: the reference would panic on a divisor of this batch");
    return RONK_OK;
  }
  RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return RONK_OK;
}

// ---- Lagrange interpolation (Reed–Solomon decode, §8f row 2) ------------------------------------
// Message::decode (codes/reed_solomon.rs:55-107) interpolates the first K coordinates:
//   data[i] = Σ_j y_j · (-1)^i e_{K-1-i}(x \ x_j) / Π_{k≠j}(x_k - x_j)
// which is coefficient i of Σ_j y_j · M(X)/(X - x_j) / M'(x_j), M = Π (X - x_k).  The reference
// enumerates combinations (exponential in K); the value is the unique interpolant, computed here as
// (1) M by K in-place products, (2) per node j a synthetic division M/(X - x_j) giving q_j and
// d_j = q_j(x_j) = Π_{k≠j}(x_j - x_k), c_j = y_j/d_j, (3) out = Σ_j c_j q_j with a warp-shuffle
// reduction per coefficient.  A repeated node gives d_j = 0: the reference's `/` panics → flag.  Over rows of ys (k
// words each), blockIdx.y stepping by gridDim.y: d_j^-1 is taken once per node for all the CTA's rows.
template <class F>
__global__ void __launch_bounds__(1024)
interp_master_kernel(const F f, const u64* __restrict__ xs, u32 k, u64* __restrict__ m0, u64* __restrict__ m1) {
  // m0/m1: k+1 words each, ping-pong; the result ends in (k odd ? m1 : m0)
  const u32 t = threadIdx.x;
  for (u32 i = t; i <= k; i += blockDim.x) m0[i] = (i == 0) ? 1 % f.modulus() : 0ULL;
  __syncthreads();
  u64* cur = m0;
  u64* nxt = m1;
  for (u32 s = 0; s < k; s++) {  // cur has degree s; nxt = cur · (X - x_s)
    const u64 x = xs[s];
    for (u32 i = t; i <= s + 1; i += blockDim.x) {
      const u64 lo = (i >= 1) ? cur[i - 1] : 0ULL;
      const u64 hi = (i <= s) ? f.mul(cur[i], x) : 0ULL;
      nxt[i] = f.sub(lo, hi);
    }
    __syncthreads();
    u64* tmp = cur; cur = nxt; nxt = tmp;
  }
}

template <class F>
__global__ void __launch_bounds__(256)
interp_nodes_kernel(const F f, const u64* __restrict__ M, const u64* __restrict__ xs, const u64* __restrict__ ys, u32 k,
                    u32 rows, u64* __restrict__ partial /* [rows][ceil(k/32)][k] */, int* flag) {
  const u32 j = blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = j < k;
  const u64 x = live ? xs[j] : 0ULL;
  // pass 1: d_j = q_j(x_j), with q_j[i-1] = M[i] + x_j·q_j[i], q_j[k-1] = M[k] = 1, Horner from the top
  u64 qv = 0, d = 0;
  for (u32 i = k; i >= 1; i--) {
    qv = f.add(M[i], f.mul(qv, x));  // q_j[i-1]
    d = f.add(f.mul(d, x), qv);
  }
  u64 dinv = 0;
  if (live) {
    if (d == 0) atomicExch(flag, 1);
    else dinv = field_pow(f, d, f.modulus() - 2);
  }
  // pass 2: Σ over the warp's nodes of c_j · q_j[i-1], c_j = y_j / d_j
  const u32 warp = j >> 5, lane = threadIdx.x & 31;
  const size_t nwarps = (size_t)gridDim.x * (blockDim.x / 32);
  for (u64 b = blockIdx.y; b < rows; b += gridDim.y) {
    const u64 c = live ? f.mul(ys[b * k + j], dinv) : 0ULL;
    u64* pb = partial + b * nwarps * k;
    qv = 0;
    for (u32 i = k; i >= 1; i--) {
      qv = f.add(M[i], f.mul(qv, x));
      u64 term = f.mul(c, qv);
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) term = f.add(term, __shfl_down_sync(0xFFFFFFFFu, term, off));
      if (lane == 0) pb[(size_t)warp * k + (i - 1)] = term;
    }
  }
}

template <class F>
__global__ void interp_sum_kernel(const F f, const u64* __restrict__ partial, u32 k, u32 nwarps, u32 rows, u64* __restrict__ out) {
  const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= k) return;
  for (u64 b = blockIdx.y; b < rows; b += gridDim.y) {
    const u64* pb = partial + b * nwarps * k;
    u64 acc = 0;
    for (u32 w = 0; w < nwarps; w++) acc = f.add(acc, pb[(size_t)w * k + i]);
    out[b * k + i] = acc;
  }
}

int poly_mul_schoolbook_rows(ronk_ctx* ctx, u64 p, const u64* a, size_t da, const u64* b, size_t db, size_t b_stride,
                             u64 batch, u64* c) {
  const u64 total = batch * (u64)(da + db - 1);
  return with_field(ctx, p, 0, false, [&](const auto& f) {
    return launch(ctx, "poly_mul_schoolbook", poly_mul_schoolbook_kernel<std::decay_t<decltype(f)>>, grid_for(ctx, total, 128),
                  128, 0, false, f, a, da, b, db, b_stride, c, total);
  });
}

static int poly_mul_device(ronk_ctx* ctx, u64 p, u64 g, const u64* a, size_t da, const u64* b, size_t db, u64* c) {
  if (!ctx || !a || !b || !c) return set_err(ctx, RONK_EINVAL, "null argument");
  if (da == 0 || db == 0) return set_err(ctx, RONK_EINVAL, "empty polynomial (D + D2 - 1 underflows)");
  RONK_TRY(validate_modulus(ctx, p));
  const size_t L = da + db - 1;
  const u32 log_n = log2_ceil(L);
  const bool ntt_ok = g != 0 && log_n >= 1 && pow2_fits(p, log_n);
  // NTT cost ~ 3·n·log n / 2 multiplies vs da·db for schoolbook
  const double school = (double)da * (double)db;
  const double viantt = 1.5 * (double)((size_t)1 << log_n) * (double)log_n + 4096.0;
  if (!ntt_ok || school <= viantt) {
    if (crt_mul_fits(ctx, p, g, da, db)) return crt_mul_device(ctx, p, a, da, b, db, c);  // poly_crt.cu
    return poly_mul_schoolbook_rows(ctx, p, a, da, b, db, db, 1, c);
  }
  const size_t n = (size_t)1 << log_n;
  Frame fr(ctx);
  u64* X = nullptr;
  RONK_TRY(fr.take(&X, 2 * n));
  // the zero padding of a and b and the clipping of the product to L coefficients happen inside the
  // transforms' load / store phases (no pad-copy kernels, no final device copy)
  return product_bounded(ctx, p, g, a, da, b, db, log_n, X, X + n, c, L);
}

template <bool SUB>
static int poly_addsub(ronk_ctx* ctx, u64 p, const u64* a, size_t da, const u64* b, size_t db, u64* out) {
  if (!ctx || (da && (!a || !out)) || (db && !b)) return set_err(ctx, RONK_EINVAL, "null argument");
  RONK_TRY(validate_modulus(ctx, p));
  if (da == 0) return RONK_OK;
  return with_field(ctx, p, 0, false, [&](const auto& f) {
    return launch(ctx, SUB ? "poly_sub" : "poly_add", poly_addsub_kernel<std::decay_t<decltype(f)>, SUB>, grid_for(ctx, da, 256),
                  256, 0, false, f, a, da, b, db, out);
  });
}

// poly_eval_kernel over `rows` rows of d coefficients (row b to out + b·m); 1 ≤ m ≤ 2^31 - 1.
static int poly_eval_rows(ronk_ctx* ctx, u64 p, const u64* c, size_t d, u32 rows, const u64* xs, size_t m, u64* out) {
  return with_field(ctx, p, 0, false, [&](const auto& f) {
    return launch(ctx, "poly_eval", poly_eval_kernel<std::decay_t<decltype(f)>>, dim3((u32)m, grid_rows(ctx, rows, m)), 256, 0, false, f,
                  c, d, xs, rows, out);
  });
}

int poly_eval_device(ronk_ctx* ctx, u64 p, const u64* c, size_t d, const u64* xs, size_t m, u64* out) {
  if (!ctx || (m && (!xs || !out)) || (d && !c)) return set_err(ctx, RONK_EINVAL, "null argument");
  RONK_TRY(validate_modulus(ctx, p));
  if (m == 0) return RONK_OK;
  if (m > 0x7FFFFFFFULL) return set_err(ctx, RONK_EUNSUPPORTED, "too many points");
  return poly_eval_rows(ctx, p, c, d, 1, xs, m, out);
}

// nodes[i] = ω_n^i (plain residues)
int roots_table(ronk_ctx* ctx, u64 p, u64 g, u64 n, u64* nodes) {
  u64 w;
  if (ronk_root_of_unity(p, g, n, (uint64_t*)&w) != RONK_OK)
    return set_err(ctx, RONK_EINVAL, "n must divide p - 1 (no primitive n-th root of unity)");
  if (n > 0x7FFFFFFFULL) return set_err(ctx, RONK_EUNSUPPORTED, "n too large");
  return with_field(ctx, p, 0, false, [&](const auto& f) {
    // pow_table_kernel stores to_tw(s·w^i); s = to_tw(1)^-1 (1 for Goldilocks, R^-1 for Montgomery) leaves plain residues
    const u64 s = h_powmod(f.to_tw(1), p - 2, p);
    return launch(ctx, "pow_table", pow_table_kernel<std::decay_t<decltype(f)>>, ((u32)n + 255) / 256, 256, 0, false, f, w, s,
                  nodes, (u32)n);
  });
}

// The literal interpolation (interp_* kernels above) of `rows` rows of Y (k words each) through k ≤ 8192 nodes into out;
// scratch m0 and m1 of k + 1 words, partial of rows·⌈k/256⌉·8·k words.  Synchronous; RONK_EINVAL for a repeated x, with
// out written.
static int interp_literal(ronk_ctx* ctx, u64 p, const u64* X, const u64* Y, size_t k, u32 rows, u64* out, u64* m0, u64* m1,
                          u64* partial) {
  const u32 blocks = ((u32)k + 255) / 256, nwarps = blocks * 8;
  RONK_TRY(reset_flag(ctx));
  RONK_TRY(with_field(ctx, p, 0, false, [&](const auto& f) {
    using F = std::decay_t<decltype(f)>;
    RONK_TRY(launch(ctx, "interp_master", interp_master_kernel<F>, 1, 1024, 0, false, f, X, (u32)k, m0, m1));
    const u64* M = (k & 1) ? m1 : m0;
    RONK_TRY(launch(ctx, "interp_nodes", interp_nodes_kernel<F>, dim3(blocks, grid_rows(ctx, rows, blocks)), 256, 0, false, f, M, X, Y,
                    (u32)k, rows, partial, ctx->d_flag.get()));
    return launch(ctx, "interp_sum", interp_sum_kernel<F>, dim3(blocks, grid_rows(ctx, rows, blocks)), 256, 0, false, f, partial, (u32)k,
                  nwarps, rows, out);
  }));
  int v = 0;
  RONK_TRY(read_flag(ctx, &v));
  if (v) return set_err(ctx, RONK_EINVAL, "interpolation: repeated x coordinate (the reference divides by zero)");
  return RONK_OK;
}
constexpr size_t kInterpLiteralMax = 8192;

// ---- subproduct-tree entry points (poly_tree.cu), SURVEY §8f rows 2 and 3 --------------------------------------------
// The tree runs when g != 0, every transform of its plan divides p - 1 (tree_fits) and the size reaches the crossover,
// else the existing kernels do.  The crossovers are tools/multipoint_timing.py's on an H100 80GB HBM3 at 400 W (DESIGN.md
// §5): the smallest power of two from which the tree won at every larger size measured.  RONK_TREE_MIN overrides all three.
constexpr size_t kFromRootsTreeMin = 128;     // k (0.049 vs 0.050 ms); k ≤ kTreeLeaves is the tree's shared-memory kernel alone
constexpr size_t kMultievalTreeMin = 32768;   // min(d, m), timed at d = m (1.84 vs 1.96 ms; 2^14: 1.66 vs 0.58)
constexpr size_t kInterpTreeMin = 2048;       // k (1.13 vs 1.89 ms; 1024: 1.25 vs 0.89); above kInterpLiteralMax always the tree

static size_t tree_min(const ronk_ctx* ctx, size_t measured) {
  return ctx->tune.tree_min >= 0 ? (size_t)ctx->tune.tree_min : measured;
}

// Batches of rows over one point set (tools/multipoint_batch_timing.py on an H100 80GB HBM3 at 700 W, DESIGN.md §5, at
// batch 1, 2, 16 and 256): the literal kernels cost about batch·n² (n = min(d, m) or k) and, at small n, a fixed amount per
// row and point, while the tree's cost barely grows with the batch.  Multieval takes the tree from batch·n² ≥ 2^30 (at
// batch 1 the single-row n ≥ 2^15; 16 rows from n = 8192: 1.41 vs 1.92 ms, 4096: 1.17 vs 0.56) or batch·n ≥ 2^18 (256
// rows from n = 1024: 0.82 vs 0.83 ms, 2048: 0.99 vs 2.52); interpolation from k ≥ 2048 as for one row, or batch·k² ≥
// 2^28 (256 rows from k = 1024: 1.19 vs 2.60 ms; 512: 0.79 vs 0.79).  RONK_TREE_MIN overrides both, whatever the batch.
static bool multieval_takes_tree(const ronk_ctx* ctx, size_t n, u32 batch) {
  if (ctx->tune.tree_min >= 0) return n >= (size_t)ctx->tune.tree_min;
  static_assert(kMultievalTreeMin == (size_t)1 << 15, "batch·n² ≥ 2^30 is n ≥ kMultievalTreeMin at batch 1");
  const u64 n64 = n, b = batch;
  return n64 >= kMultievalTreeMin || n64 * n64 >= (((u64)1 << 30) + b - 1) / b || b * n64 >= ((u64)1 << 18);  // n ≤ 2^24
}
static bool interp_takes_tree(const ronk_ctx* ctx, size_t k, u32 batch) {
  if (ctx->tune.tree_min >= 0) return k >= (size_t)ctx->tune.tree_min;
  const u64 k64 = k;
  return k64 >= kInterpTreeMin || k64 * k64 >= (((u64)1 << 28) + batch - 1) / batch;  // k ≤ 2^24
}

// Checks shared by the three: RONK_EINVAL for a null pointer or g out of range, RONK_EUNSUPPORTED above 2^24 points.
static int tree_args(ronk_ctx* ctx, u64 p, u64 g, size_t k, bool null_arg) {
  if (!ctx || null_arg) return set_err(ctx, RONK_EINVAL, "null argument");
  RONK_TRY(validate_modulus(ctx, p));
  if (g >= p) return set_err(ctx, RONK_EINVAL, "generator out of range");
  if (k > kTreeMaxLeaves) return set_err(ctx, RONK_EUNSUPPORTED, "more than 2^24 points");
  return RONK_OK;
}

static int from_roots_device(ronk_ctx* ctx, u64 p, u64 g, const u64* xs, size_t k, u64* out) {
  RONK_TRY(tree_args(ctx, p, g, k, !out || (k && !xs)));
  if (overlaps(out, k + 1, xs, k)) return set_err(ctx, RONK_EINVAL, "out may not overlap xs");
  if (k == 0) {  // the empty product (pageable source: staged before cudaMemcpyAsync returns)
    const u64 one = 1;
    RONK_CUDA(ctx, cudaMemcpyAsync(out, &one, sizeof(u64), cudaMemcpyHostToDevice, ctx->stream));
    return RONK_OK;
  }
  if (k <= kTreeLeaves || (tree_fits(p, g, k, 0) && k >= tree_min(ctx, kFromRootsTreeMin)))
    return tree_from_roots(ctx, p, g, xs, k, out);
  if (k > kInterpLiteralMax)
    return set_err(ctx, RONK_EUNSUPPORTED, "more than 8192 roots off the tree path (k sequential linear products)");
  // k linear products in one CTA (interp_master_kernel), ping-ponging between out and k + 1 words of scratch so that
  // the last one lands in out
  Frame fr(ctx);
  u64* tmp = nullptr;
  RONK_TRY(fr.take(&tmp, k + 1));
  return with_field(ctx, p, 0, false, [&](const auto& f) {
    return launch(ctx, "interp_master", interp_master_kernel<std::decay_t<decltype(f)>>, 1, 1024, 0, false, f, xs, (u32)k,
                  (k & 1) ? tmp : out, (k & 1) ? out : tmp);
  });
}

// The batched entries' envelope: batch·N words in each row buffer of the tree, N = 2^⌈log2 size⌉ (for multieval also
// the root's 2^⌈log2(2d - 1)⌉), as ronk_poly_mul_batch_u64's batched transforms; batch·⌈k/256⌉·8·k words of the literal
// interpolation's per-warp partial sums.
constexpr u64 kTreeBatchMaxWords = (u64)1 << 32;

// The path of a non-empty call and the checks that go with it, which read no pointer, so that the _host twins make them
// before they stage anything: *tree, or RONK_EUNSUPPORTED past the envelope.
int multieval_path(ronk_ctx* ctx, u64 p, u64 g, size_t d, u32 batch, size_t m, bool* tree) {
  *tree = d && tree_fits(p, g, m, d) && multieval_takes_tree(ctx, std::min(d, m), batch);
  if (!*tree) return RONK_OK;
  const u64 N = std::max((u64)1 << log2_ceil(m), (u64)1 << std::max<u32>(1, log2_ceil(2 * d - 1)));
  if ((u64)batch * N > kTreeBatchMaxWords) return set_err(ctx, RONK_EUNSUPPORTED, "more than 2^32 words of tree rows");
  return RONK_OK;
}

int interpolate_path(ronk_ctx* ctx, u64 p, u64 g, size_t k, u32 batch, bool* tree) {
  *tree = tree_fits(p, g, k, k) && (interp_takes_tree(ctx, k, batch) || k > kInterpLiteralMax);
  if (*tree) {
    if ((u64)batch << log2_ceil(k) > kTreeBatchMaxWords)
      return set_err(ctx, RONK_EUNSUPPORTED, "more than 2^32 words of tree rows");
    return RONK_OK;
  }
  if (k > kInterpLiteralMax)
    return set_err(ctx, RONK_EUNSUPPORTED, "more than 8192 nodes off the tree path (O(K²) interpolation)");
  if ((u64)batch * ((k + 255) / 256 * 8) * k > kTreeBatchMaxWords)
    return set_err(ctx, RONK_EUNSUPPORTED, "more than 2^32 words of per-warp partial sums");
  return RONK_OK;
}

static int multieval_device(ronk_ctx* ctx, u64 p, u64 g, const u64* c, size_t d, u32 batch, const u64* xs, size_t m, u64* out,
                            bool reserve) {
  RONK_TRY(tree_args(ctx, p, g, m, (m && (!xs || !out)) || (d && !c)));
  if (m == 0 || batch == 0) return RONK_OK;
  if (d > ~(u64)0 / batch) return set_err(ctx, RONK_EUNSUPPORTED, "batch·d words overflow");
  const size_t nc = (size_t)batch * d, no = (size_t)batch * m;
  if (overlaps(out, no, xs, m) || overlaps(out, no, c, nc)) return set_err(ctx, RONK_EINVAL, "out may not overlap coeffs or xs");
  bool tree = false;
  RONK_TRY(multieval_path(ctx, p, g, d, batch, m, &tree));
  if (!tree) return poly_eval_rows(ctx, p, c, d, batch, xs, m, out);
  if (reserve) RONK_TRY(reserve_scratch(ctx, tree_scratch_words(ctx, m, d, batch, false)));
  return tree_multieval(ctx, p, g, c, d, batch, xs, m, out);
}

static int interpolate_device(ronk_ctx* ctx, u64 p, u64 g, const u64* xs, const u64* ys, size_t k, u32 batch, u64* out,
                              bool reserve) {
  RONK_TRY(tree_args(ctx, p, g, k, k && (!xs || !ys || !out)));
  if (k == 0 || batch == 0) return RONK_OK;
  const size_t ny = (size_t)batch * k;
  if (overlaps(out, ny, xs, k) || overlaps(out, ny, ys, ny)) return set_err(ctx, RONK_EINVAL, "out may not overlap xs or ys");
  bool tree = false;
  RONK_TRY(interpolate_path(ctx, p, g, k, batch, &tree));
  if (tree) {
    if (reserve) RONK_TRY(reserve_scratch(ctx, tree_scratch_words(ctx, k, k, batch, true)));
    return tree_interpolate(ctx, p, g, xs, ys, k, batch, out);
  }
  // the literal kernels into scratch, so that a repeated x leaves out unwritten
  const size_t nwarps = (k + 255) / 256 * 8;
  Frame fr(ctx);
  u64* res = nullptr;
  RONK_TRY(fr.take(&res, ny + 2 * (k + 1) + batch * nwarps * k));
  u64* m0 = res + ny;
  u64* m1 = m0 + k + 1;
  RONK_TRY(interp_literal(ctx, p, xs, ys, k, batch, res, m0, m1, m1 + k + 1));
  RONK_CUDA(ctx, cudaMemcpyAsync(out, res, ny * sizeof(u64), cudaMemcpyDeviceToDevice, ctx->stream));
  RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return RONK_OK;
}

static int dft_device(ronk_ctx* ctx, u64 p, u64 g, const u64* in, u64 n, u64* out) {
  if (!ctx || !in || !out) return set_err(ctx, RONK_EINVAL, "null argument");
  RONK_TRY(validate_modulus(ctx, p));
  if (g == 0 || g >= p) return set_err(ctx, RONK_EINVAL, "generator out of range");
  if (n == 0 || (p - 1) % n != 0)
    return set_err(ctx, RONK_EINVAL, "n must divide p - 1 (no primitive n-th root of unity)");
  Frame fr(ctx);
  u64* nodes = nullptr;
  RONK_TRY(fr.take(&nodes, n));
  RONK_TRY(roots_table(ctx, p, g, n, nodes));
  return poly_eval_device(ctx, p, in, n, nodes, n, out);  // X[i] = a(ω^i)
}

}  // namespace ronk

using namespace ronk;

extern "C" {

int ronk_poly_mul_u64(ronk_ctx* ctx, uint64_t p, uint64_t g, const uint64_t* a, size_t da, const uint64_t* b,
                      size_t db, uint64_t* c) {
  ronk::DeviceGuard _dg(ctx);
  return poly_mul_device(ctx, p, g, (const u64*)a, da, (const u64*)b, db, (u64*)c);
}

int ronk_poly_add_u64(ronk_ctx* ctx, uint64_t p, const uint64_t* a, size_t da, const uint64_t* b, size_t db,
                      uint64_t* out) {
  ronk::DeviceGuard _dg(ctx);
  return poly_addsub<false>(ctx, p, (const u64*)a, da, (const u64*)b, db, (u64*)out);
}
int ronk_poly_sub_u64(ronk_ctx* ctx, uint64_t p, const uint64_t* a, size_t da, const uint64_t* b, size_t db,
                      uint64_t* out) {
  ronk::DeviceGuard _dg(ctx);
  return poly_addsub<true>(ctx, p, (const u64*)a, da, (const u64*)b, db, (u64*)out);
}

int ronk_poly_eval_u64(ronk_ctx* ctx, uint64_t p, const uint64_t* coeffs, size_t d, const uint64_t* xs, size_t m,
                       uint64_t* out) {
  ronk::DeviceGuard _dg(ctx);
  return poly_eval_device(ctx, p, (const u64*)coeffs, d, (const u64*)xs, m, (u64*)out);
}

int ronk_dft_u64(ronk_ctx* ctx, uint64_t p, uint64_t g, const uint64_t* in, uint64_t n, uint64_t* out) {
  ronk::DeviceGuard _dg(ctx);
  return dft_device(ctx, p, g, (const u64*)in, n, (u64*)out);
}

int ronk_poly_div_linear_u64(ronk_ctx* ctx, uint64_t p, const uint64_t* a, size_t d, uint64_t b0, uint64_t b1,
                             uint64_t* q, uint64_t* rem) {
  ronk::DeviceGuard _dg(ctx);
  return div_linear_device(ctx, p, (const u64*)a, d, b0, b1, (u64*)q, (u64*)rem);
}

int ronk_poly_divrem_u64(ronk_ctx* ctx, uint64_t p, uint64_t g, const uint64_t* a, size_t da, const uint64_t* b, size_t db,
                         uint64_t* q, uint64_t* r) {
  ronk::DeviceGuard _dg(ctx);
  return divrem_device(ctx, p, g, (const u64*)a, da, (const u64*)b, db, (u64*)q, (u64*)r);
}

// ---- host-pointer variants ---------------------------------------------------------------------
// Each stages its arguments, runs the device-pointer function on them and copies the results back.  The device
// function's checks repeated here are those staging needs first: a null argument cannot be uploaded.
int ronk_poly_mul_u64_host(ronk_ctx* ctx, uint64_t p, uint64_t g, const uint64_t* a, size_t da, const uint64_t* b,
                           size_t db, uint64_t* c) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx || !a || !b || !c) return set_err(ctx, RONK_EINVAL, "null argument");
  if (da == 0 || db == 0) return set_err(ctx, RONK_EINVAL, "empty polynomial (D + D2 - 1 underflows)");
  Staged s[] = {{da * 8, a}, {db * 8, b}, {(da + db - 1) * 8, nullptr, c}};
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  return stage_out(ctx, poly_mul_device(ctx, p, g, s[0].dev, da, s[1].dev, db, s[2].dev), s);
}

int ronk_poly_eval_u64_host(ronk_ctx* ctx, uint64_t p, const uint64_t* coeffs, size_t d, const uint64_t* xs, size_t m,
                            uint64_t* out) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx || (m && (!xs || !out)) || (d && !coeffs)) return set_err(ctx, RONK_EINVAL, "null argument");
  Staged s[] = {{d * 8, coeffs}, {m * 8, xs}, {m * 8, nullptr, out}};
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  return stage_out(ctx, poly_eval_device(ctx, p, s[0].dev, d, s[1].dev, m, s[2].dev), s);
}

int ronk_dft_u64_host(ronk_ctx* ctx, uint64_t p, uint64_t g, const uint64_t* in, uint64_t n, uint64_t* out) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx || !in || !out) return set_err(ctx, RONK_EINVAL, "null argument");
  Staged s[] = {{n * 8, in}, {n * 8, nullptr, out}};
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  return stage_out(ctx, dft_device(ctx, p, g, s[0].dev, n, s[1].dev), s);
}

int ronk_poly_lagrange_eval_u64_host(ronk_ctx* ctx, uint64_t p, uint64_t g, const uint64_t* coeffs, size_t n,
                                     uint64_t x, uint64_t* out) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx || !coeffs || !out) return set_err(ctx, RONK_EINVAL, "null argument");
  RONK_TRY(validate_modulus(ctx, p));
  if (g == 0 || g >= p || x >= p) return set_err(ctx, RONK_EINVAL, "argument out of range");
  if (n == 0 || (p - 1) % n != 0)
    return set_err(ctx, RONK_EINVAL, "n must divide p - 1 (Lagrange::new asserts)");  // mod.rs:361
  if (n > (1u << 20)) return set_err(ctx, RONK_EUNSUPPORTED, "n too large for the O(n²) barycentric form");
  Staged s[] = {{n * 8, coeffs}, {n * 8}, {8, nullptr, out}};  // coefficients, nodes, result
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  RONK_TRY(roots_table(ctx, p, g, n, s[1].dev));
  RONK_TRY(reset_flag(ctx));
  RONK_TRY(with_field(ctx, p, 0, false, [&](const auto& f) {
    return launch(ctx, "lagrange_eval", lagrange_eval_kernel<std::decay_t<decltype(f)>>, 1, 256, 0, false, f, s[0].dev,
                  s[1].dev, (u32)n, x, s[2].dev, ctx->d_flag.get());
  }));
  int v = 0;
  RONK_TRY(read_flag(ctx, &v));
  if (v)  // mod.rs:386-393: F::ONE.div(x_j - x_m) panics when two nodes coincide (g not of order n)
    return set_err(ctx, RONK_EINVAL, "Lagrange evaluate: repeated node (the reference divides by zero)");
  return stage_out(ctx, RONK_OK, s);
}

int ronk_poly_interpolate_u64_host(ronk_ctx* ctx, uint64_t p, const uint64_t* xs, const uint64_t* ys, size_t k,
                                   uint64_t* out) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx || (k && (!xs || !ys || !out))) return set_err(ctx, RONK_EINVAL, "null argument");
  RONK_TRY(validate_modulus(ctx, p));
  if (k == 0) return RONK_OK;
  if (k > 8192) return set_err(ctx, RONK_EUNSUPPORTED, "more than 8192 nodes (O(K²) interpolation)");
  for (size_t i = 0; i < k; i++)
    if (xs[i] >= p || ys[i] >= p) return set_err(ctx, RONK_EINVAL, "non-canonical residue");
  const size_t nwarps = (k + 255) / 256 * 8;
  // xs, ys, out, then the scratch: the master polynomial's two ping-pong buffers and the per-warp partial sums
  Staged s[] = {{k * 8, xs}, {k * 8, ys}, {k * 8, nullptr, out}, {(k + 1) * 8}, {(k + 1) * 8}, {nwarps * k * 8}};
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  RONK_TRY(interp_literal(ctx, p, s[0].dev, s[1].dev, k, 1, s[2].dev, s[3].dev, s[4].dev, s[5].dev));
  return stage_out(ctx, RONK_OK, s);
}

int ronk_poly_from_roots_u64(ronk_ctx* ctx, uint64_t p, uint64_t g, const uint64_t* xs, size_t k, uint64_t* out) {
  ronk::DeviceGuard _dg(ctx);
  return from_roots_device(ctx, p, g, (const u64*)xs, k, (u64*)out);
}

int ronk_poly_multieval_u64(ronk_ctx* ctx, uint64_t p, uint64_t g, const uint64_t* coeffs, size_t d, const uint64_t* xs,
                            size_t m, uint64_t* out) {
  ronk::DeviceGuard _dg(ctx);
  return multieval_device(ctx, p, g, (const u64*)coeffs, d, 1, (const u64*)xs, m, (u64*)out, false);
}

int ronk_poly_interpolate_u64(ronk_ctx* ctx, uint64_t p, uint64_t g, const uint64_t* xs, const uint64_t* ys, size_t k,
                              uint64_t* out) {
  ronk::DeviceGuard _dg(ctx);
  return interpolate_device(ctx, p, g, (const u64*)xs, (const u64*)ys, k, 1, (u64*)out, false);
}

int ronk_poly_multieval_batch_u64(ronk_ctx* ctx, uint64_t p, uint64_t g, const uint64_t* coeffs, size_t d, uint32_t batch,
                                  const uint64_t* xs, size_t m, uint64_t* out) {
  ronk::DeviceGuard _dg(ctx);
  return multieval_device(ctx, p, g, (const u64*)coeffs, d, batch, (const u64*)xs, m, (u64*)out, true);
}

int ronk_poly_interpolate_batch_u64(ronk_ctx* ctx, uint64_t p, uint64_t g, const uint64_t* xs, const uint64_t* ys, size_t k,
                                    uint32_t batch, uint64_t* out) {
  ronk::DeviceGuard _dg(ctx);
  return interpolate_device(ctx, p, g, (const u64*)xs, (const u64*)ys, k, batch, (u64*)out, true);
}

// Host pointers: the device function's checks that read no pointer, and its size checks, come first, so that nothing is
// staged for an empty call or one refused for its arguments or its size.
int ronk_poly_multieval_batch_u64_host(ronk_ctx* ctx, uint64_t p, uint64_t g, const uint64_t* coeffs, size_t d, uint32_t batch,
                                       const uint64_t* xs, size_t m, uint64_t* out) {
  ronk::DeviceGuard _dg(ctx);
  RONK_TRY(tree_args(ctx, p, g, m, (m && (!xs || !out)) || (d && !coeffs)));
  if (m == 0 || batch == 0) return RONK_OK;
  if (d > ~(u64)0 / 8 / batch) return set_err(ctx, RONK_EUNSUPPORTED, "batch·d words overflow");
  bool tree = false;
  RONK_TRY(multieval_path(ctx, p, g, d, batch, m, &tree));
  Staged s[] = {{(size_t)batch * d * 8, coeffs}, {m * 8, xs}, {(size_t)batch * m * 8, nullptr, out}};
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  return stage_out(ctx, multieval_device(ctx, p, g, s[0].dev, d, batch, s[1].dev, m, s[2].dev, true), s);
}

int ronk_poly_interpolate_batch_u64_host(ronk_ctx* ctx, uint64_t p, uint64_t g, const uint64_t* xs, const uint64_t* ys,
                                         size_t k, uint32_t batch, uint64_t* out) {
  ronk::DeviceGuard _dg(ctx);
  RONK_TRY(tree_args(ctx, p, g, k, k && (!xs || !ys || !out)));
  if (k == 0 || batch == 0) return RONK_OK;
  bool tree = false;
  RONK_TRY(interpolate_path(ctx, p, g, k, batch, &tree));
  Staged s[] = {{k * 8, xs}, {(size_t)batch * k * 8, ys}, {(size_t)batch * k * 8, nullptr, out}};
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  return stage_out(ctx, interpolate_device(ctx, p, g, s[0].dev, s[1].dev, k, batch, s[2].dev, true), s);
}

int ronk_poly_divrem_batch_u64(ronk_ctx* ctx, uint64_t p, uint64_t g, const uint64_t* a, size_t da, const uint64_t* b, size_t db,
                               int b_shared, uint32_t batch, uint64_t* q, uint64_t* r) {
  ronk::DeviceGuard _dg(ctx);
  return divrem_batch_device(ctx, p, g, (const u64*)a, da, (const u64*)b, db, b_shared != 0, batch, (u64*)q, (u64*)r);
}

// Host pointers: every check that reads no pointer comes first, so that nothing is staged for an empty or refused call.
int ronk_poly_divrem_batch_u64_host(ronk_ctx* ctx, uint64_t p, uint64_t g, const uint64_t* a, size_t da, const uint64_t* b,
                                    size_t db, int b_shared, uint32_t batch, uint64_t* q, uint64_t* r) {
  ronk::DeviceGuard _dg(ctx);
  const bool empty = batch == 0 || da == 0;
  DivremBatchPath path;
  RONK_TRY(divrem_batch_args(ctx, p, g, !empty && (!a || !q || !r || (db && !b)), da, db, b_shared != 0, batch, &path));
  if (empty) return RONK_OK;
  const size_t na = (size_t)batch * da, nb = b_shared ? db : (size_t)batch * db;
  Staged s[] = {{na * 8, a}, {nb * 8, b}, {na * 8, nullptr, q}, {na * 8, nullptr, r}};
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  return stage_out(ctx, divrem_batch_device(ctx, p, g, s[0].dev, da, s[1].dev, db, b_shared != 0, batch, s[2].dev, s[3].dev), s);
}

// ronk_poly_divrem_u64 with g = 0 (no Newton path) on staged copies of a and b.  Its checks up to da == 0 run before
// staging, in the device function's order, so that an overlong operand is refused before it is copied.
int ronk_poly_divrem_u64_host(ronk_ctx* ctx, uint64_t p, const uint64_t* a, size_t da, const uint64_t* b, size_t db,
                              uint64_t* q, uint64_t* r) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx || (da && (!a || !q || !r)) || (db && !b)) return set_err(ctx, RONK_EINVAL, "null argument");
  RONK_TRY(validate_modulus(ctx, p));
  if (da > 0x7FFFFFF0ULL || db > 0x7FFFFFF0ULL) return set_err(ctx, RONK_EUNSUPPORTED, "polynomial too long");
  if (da == 0) return RONK_OK;
  Staged s[] = {{da * 8, a}, {db * 8, b}, {da * 8, nullptr, q}, {da * 8, nullptr, r}};
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  return stage_out(ctx, divrem_device(ctx, p, /*g=*/0, s[0].dev, da, s[1].dev, db, s[2].dev, s[3].dev), s);
}

}  // extern "C"
