// field_ops.cu — PrimeField<P> element-wise kernels and FiniteField metadata.
// Mirrors src/algebra/field/prime/arithmetic.rs:3-71 and src/algebra/field/prime/mod.rs:58-123.
#include "ronk_internal.h"

namespace ronk {

enum { OP_ADD = 0, OP_SUB = 1, OP_MUL = 2, OP_DIV = 3 };
enum { UOP_NEG = 0, UOP_INV = 1 };

template <class F, int OP>
__global__ void binop_kernel(const F f, const u64* a, const u64* b, u64* out,
                             size_t n, int* flag) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const u64 x = a[i], y = b[i];
    u64 r;
    if (OP == OP_ADD) r = f.add(x, y);
    else if (OP == OP_SUB) r = f.sub(x, y);
    else if (OP == OP_MUL) r = f.mul(x, y);
    else {
      if (y == 0) { atomicExch(flag, 1); r = 0; }                 // rhs.inverse().unwrap() panics
      else r = f.mul(x, field_pow(f, y, f.modulus() - 2));        // prime/arithmetic.rs:54
    }
    out[i] = r;
  }
}

template <class F, int OP>
__global__ void unop_kernel(const F f, const u64* a, u64* out, size_t n, u64 e, int* flag) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const u64 x = a[i];
    u64 r;
    if (OP == UOP_NEG) r = f.neg(x);
    else if (OP == UOP_INV) {
      if (x == 0) { atomicExch(flag, 1); r = 0; }                 // inverse() == None
      else r = field_pow(f, x, f.modulus() - 2);                  // prime/mod.rs:62-72
    } else r = field_pow(f, x, e);                                // prime/mod.rs:74-84
    out[i] = r;
  }
}

// out[i] = scale·base^i
template <class F>
__global__ void powers_kernel(const F f, u64 base, u64 scale, u64* out, size_t n) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i0 >= n) return;
  u64 cur = f.mul(scale, field_pow(f, base, (u64)i0));
  const u64 step = field_pow(f, base, (u64)stride);
  for (size_t i = i0; i < n; i += stride) {
    out[i] = cur;
    cur = f.mul(cur, step);
  }
}

// In-place G-point DFT (G = 2^log_g ≤ 16) over data[k + j·stride]; wt[j] = ω_G^(±j) plain residues,
// sc = 1 or G^-1.  O(G²) per k — the cross-rank stage is a sliver of the whole transform.
template <class F>
__global__ void strided_dft_kernel(const F f, u64* data, u32 G, size_t stride, size_t count, const u64* wt, u64 sc) {
  const size_t step = (size_t)gridDim.x * blockDim.x;
  for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < count; k += step) {
    u64 x[16], y[16];
    for (u32 j = 0; j < G; j++) x[j] = data[k + (size_t)j * stride];
    for (u32 q = 0; q < G; q++) {
      u64 acc = 0;
      for (u32 j = 0; j < G; j++) acc = f.add(acc, f.mul(x[j], wt[(j * q) & (G - 1)]));
      y[q] = f.mul(acc, sc);
    }
    for (u32 q = 0; q < G; q++) data[k + (size_t)q * stride] = y[q];
  }
}

// Fused cross-rank stage of the distributed transform.  Thread k'' of rank s handles
// k' = s·blk + k'': it loads Y_r'[k'] from every peer r' (plain ld.global on peer-mapped addresses —
// NVLink P2P), multiplies by ω_n^(r'·k') = base^r' (base = ω_n^k' from `twbase`), runs the G-point
// transform and writes X[k' + m·q] to out[q·blk + k''].  O(G²) per k', G ≤ 16.
struct PeerPtrs {
  const u64* p[16];
};
template <class F>
__global__ void cross_rank_fused_kernel(const F f, const PeerPtrs peers, const u64* __restrict__ twbase, const u64* wt,
                                        u64* __restrict__ out, u32 G, size_t blk, u32 rank) {
  const size_t step = (size_t)gridDim.x * blockDim.x;
  for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < blk; k += step) {
    const size_t kp = (size_t)rank * blk + k;
    u64 x[16], y[16];
    for (u32 r = 0; r < G; r++) x[r] = peers.p[r][kp];   // P2P loads first: all in flight together
    const u64 base = twbase[k];
    u64 tw = base;
    for (u32 r = 1; r < G; r++) {
      x[r] = f.mul(x[r], tw);
      tw = f.mul(tw, base);
    }
    for (u32 q = 0; q < G; q++) {
      u64 acc = 0;
      for (u32 j = 0; j < G; j++) acc = f.add(acc, f.mul(x[j], wt[(j * q) & (G - 1)]));
      y[q] = acc;
    }
    for (u32 q = 0; q < G; q++) out[(size_t)q * blk + k] = y[q];
  }
}

__global__ void splitmix_kernel(u64 p, u64 seed, u64* out, size_t n) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    u64 z = seed + (u64)(i + 1) * 0x9E3779B97F4A7C15ULL;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    z ^= z >> 31;
    out[i] = z % p;
  }
}

static bool h_is_prime(u64 n) {  // deterministic Miller–Rabin for 64-bit n
  if (n < 2) return false;
  for (u64 q : {2ULL, 3ULL, 5ULL, 7ULL, 11ULL, 13ULL, 17ULL, 19ULL, 23ULL, 29ULL, 31ULL, 37ULL}) {
    if (n % q == 0) return n == q;
  }
  u64 d = n - 1;
  int s = 0;
  while ((d & 1) == 0) { d >>= 1; s++; }
  for (u64 a : {2ULL, 3ULL, 5ULL, 7ULL, 11ULL, 13ULL, 17ULL, 19ULL, 23ULL, 29ULL, 31ULL, 37ULL}) {
    u64 x = h_powmod(a, d, n);
    if (x == 1 || x == n - 1) continue;
    bool comp = true;
    for (int r = 1; r < s; r++) {
      x = h_mulmod(x, x, n);
      if (x == n - 1) { comp = false; break; }
    }
    if (comp) return false;
  }
  return true;
}

// PrimeField::new's const is_prime(P) (prime/mod.rs:48-50, :92-100) panics for composite P.
int validate_modulus(ronk_ctx* ctx, u64 p) {
  if (p == GL_P) return RONK_OK;
  if (p == 2) return set_err(ctx, RONK_EUNSUPPORTED, "p = 2 (AESField) is outside this library's scope");
  if (!h_is_prime(p)) return set_err(ctx, RONK_EINVAL, "input is not a prime number");
  return RONK_OK;
}

template <int OP>
static int binop(ronk_ctx* ctx, u64 p, const u64* a, const u64* b, u64* out, size_t n, const char* name) {
  if (!ctx || (n && (!a || !b || !out))) return set_err(ctx, RONK_EINVAL, "null argument");
  RONK_TRY(validate_modulus(ctx, p));
  if (n == 0) return RONK_OK;
  if (OP == OP_DIV) RONK_TRY(reset_flag(ctx));
  RONK_TRY(with_field(ctx, p, 0, false, [&](const auto& f) {
    return launch(ctx, name, binop_kernel<std::decay_t<decltype(f)>, OP>, grid_for(ctx, n, 256), 256, 0, false, f, a, b,
                  out, n, ctx->d_flag.get());
  }));
  if (OP == OP_DIV) {
    int v = 0;
    RONK_TRY(read_flag(ctx, &v));
    if (v) return set_err(ctx, RONK_EINVAL, "division by zero (inverse of 0 is None)");
  }
  return RONK_OK;
}

template <int OP>
static int unop(ronk_ctx* ctx, u64 p, const u64* a, u64* out, size_t n, u64 e, const char* name) {
  if (!ctx || (n && (!a || !out))) return set_err(ctx, RONK_EINVAL, "null argument");
  RONK_TRY(validate_modulus(ctx, p));
  if (n == 0) return RONK_OK;
  if (OP == UOP_INV) RONK_TRY(reset_flag(ctx));
  RONK_TRY(with_field(ctx, p, 0, false, [&](const auto& f) {
    return launch(ctx, name, unop_kernel<std::decay_t<decltype(f)>, OP>, grid_for(ctx, n, 256), 256, 0, false, f, a, out,
                  n, e, ctx->d_flag.get());
  }));
  if (OP == UOP_INV) {
    int v = 0;
    RONK_TRY(read_flag(ctx, &v));
    if (v) return set_err(ctx, RONK_EINVAL, "inverse of 0 is None");
  }
  return RONK_OK;
}

}  // namespace ronk

using namespace ronk;

extern "C" {

int ronk_field_generator(uint64_t p, uint64_t* g) {
  if (!g) return RONK_EINVAL;
  switch (p) {  // results of find_primitive_element (prime/mod.rs:110-123) for the reference's moduli
    case 101: *g = 2; return RONK_OK;
    case 17: *g = 14; return RONK_OK;
    case 127: *g = 3; return RONK_OK;
    case 59: *g = 2; return RONK_OK;
    case RONK_GOLDILOCKS: *g = 7; return RONK_OK;  // pinned (SURVEY §8a D4)
    default: break;
  }
  if (p < 3 || !h_is_prime(p)) return RONK_EINVAL;
  if (p > (1ULL << 32)) return RONK_EUNSUPPORTED;  // pass g explicitly for other large moduli
  // the reference's literal search, for other small primes
  for (u64 i = 2; i * i <= p; i++) {
    if ((p - 1) % i == 0) {
      if (h_powmod(i, (p - 1) / i, p) != 1) { *g = i; return RONK_OK; }
      else if (h_powmod(p + 1 - i, i, p) != 1) { *g = p + 1 - i; return RONK_OK; }
    }
  }
  return RONK_EINVAL;  // panic!("generator not found")
}

int ronk_root_of_unity(uint64_t p, uint64_t g, uint64_t n, uint64_t* out) {
  if (!out || p < 3 || g == 0 || g >= p) return RONK_EINVAL;
  if (n == 0 || (p - 1) % n != 0) return RONK_EINVAL;  // assert!(p_minus_one % n == 0)
  *out = h_powmod(g, (p - 1) / n, p);
  return RONK_OK;
}

int ronk_field_add_u64(ronk_ctx* ctx, uint64_t p, const uint64_t* a, const uint64_t* b, uint64_t* out, size_t n) {
  ronk::DeviceGuard _dg(ctx);
  return binop<OP_ADD>(ctx, p, (const u64*)a, (const u64*)b, (u64*)out, n, "field_add");
}
int ronk_field_sub_u64(ronk_ctx* ctx, uint64_t p, const uint64_t* a, const uint64_t* b, uint64_t* out, size_t n) {
  ronk::DeviceGuard _dg(ctx);
  return binop<OP_SUB>(ctx, p, (const u64*)a, (const u64*)b, (u64*)out, n, "field_sub");
}
int ronk_field_mul_u64(ronk_ctx* ctx, uint64_t p, const uint64_t* a, const uint64_t* b, uint64_t* out, size_t n) {
  ronk::DeviceGuard _dg(ctx);
  return binop<OP_MUL>(ctx, p, (const u64*)a, (const u64*)b, (u64*)out, n, "field_mul");
}
int ronk_field_div_u64(ronk_ctx* ctx, uint64_t p, const uint64_t* a, const uint64_t* b, uint64_t* out, size_t n) {
  ronk::DeviceGuard _dg(ctx);
  return binop<OP_DIV>(ctx, p, (const u64*)a, (const u64*)b, (u64*)out, n, "field_div");
}
int ronk_field_neg_u64(ronk_ctx* ctx, uint64_t p, const uint64_t* a, uint64_t* out, size_t n) {
  ronk::DeviceGuard _dg(ctx);
  return unop<UOP_NEG>(ctx, p, (const u64*)a, (u64*)out, n, 0, "field_neg");
}
int ronk_field_inv_u64(ronk_ctx* ctx, uint64_t p, const uint64_t* a, uint64_t* out, size_t n) {
  ronk::DeviceGuard _dg(ctx);
  return unop<UOP_INV>(ctx, p, (const u64*)a, (u64*)out, n, 0, "field_inv");
}
int ronk_field_pow_u64(ronk_ctx* ctx, uint64_t p, const uint64_t* a, uint64_t e, uint64_t* out, size_t n) {
  ronk::DeviceGuard _dg(ctx);
  return unop<2>(ctx, p, (const u64*)a, (u64*)out, n, e, "field_pow");
}

int ronk_field_powers_u64(ronk_ctx* ctx, uint64_t p, uint64_t base, uint64_t scale, uint64_t* out, size_t n) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx || (n && !out)) return set_err(ctx, RONK_EINVAL, "null argument");
  RONK_TRY(validate_modulus(ctx, p));
  if (base >= p || scale >= p) return set_err(ctx, RONK_EINVAL, "non-canonical argument");
  if (n == 0) return RONK_OK;
  return with_field(ctx, p, 0, false, [&](const auto& f) {
    return launch(ctx, "field_powers", powers_kernel<std::decay_t<decltype(f)>>, grid_for(ctx, (n + 7) / 8, 256), 256, 0,
                  false, f, base, scale, (u64*)out, n);
  });
}

int ronk_ntt_strided_small_u64(ronk_ctx* ctx, uint64_t p, uint64_t g, uint64_t* data, uint32_t log_g, size_t stride,
                               size_t count, int inverse) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx || (count && !data)) return set_err(ctx, RONK_EINVAL, "null argument");
  RONK_TRY(validate_modulus(ctx, p));
  if (g == 0 || g >= p) return set_err(ctx, RONK_EINVAL, "generator out of range");
  if (log_g > 4) return set_err(ctx, RONK_EUNSUPPORTED, "log_g > 4 not supported");
  const u64 G = (u64)1 << log_g;
  if ((p - 1) % G != 0) return set_err(ctx, RONK_EINVAL, "n must divide p - 1 (no primitive n-th root of unity)");
  if (count == 0 || log_g == 0) return RONK_OK;
  u64 w = h_powmod(g, (p - 1) / G, p);
  if (inverse) w = h_powmod(w, p - 2, p);
  u64 h_wt[16];
  for (u64 j = 0; j < G; j++) h_wt[j] = h_powmod(w, j, p);
  const u64 sc = inverse ? h_powmod(G % p, p - 2, p) : 1 % p;
  Frame fr(ctx);
  u64* d_wt = nullptr;
  RONK_TRY(fr.take(&d_wt, 16));
  RONK_CUDA(ctx, cudaMemcpyAsync(d_wt, h_wt, G * sizeof(u64), cudaMemcpyHostToDevice, ctx->stream));
  RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // h_wt is a stack buffer
  return with_field(ctx, p, 0, false, [&](const auto& f) {  // the transform's roots come from the wt table, not the policy
    return launch(ctx, "ntt_cross_rank", strided_dft_kernel<std::decay_t<decltype(f)>>, grid_for(ctx, count, 128), 128, 0,
                  false, f, (u64*)data, (u32)G, stride, count, (const u64*)d_wt, sc);
  });
}

int ronk_ntt_cross_rank_fused_u64(ronk_ctx* ctx, uint64_t p, uint64_t g, const uint64_t* const* peer_bufs,
                                  uint32_t log_g, uint32_t rank, uint32_t log_n, uint64_t* out) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx || !peer_bufs || !out) return set_err(ctx, RONK_EINVAL, "null argument");
  RONK_TRY(validate_modulus(ctx, p));
  if (g == 0 || g >= p) return set_err(ctx, RONK_EINVAL, "generator out of range");
  if (log_g > 4 || log_g == 0) return set_err(ctx, RONK_EUNSUPPORTED, "group size must be 2..16");
  if (log_n >= 64 || (p - 1) % ((u64)1 << log_n) != 0)
    return set_err(ctx, RONK_EINVAL, "n must divide p - 1 (no primitive n-th root of unity)");
  if (log_n < 2 * log_g) return set_err(ctx, RONK_EINVAL, "transform too small for this group");
  const u32 G = 1u << log_g;
  if (rank >= G) return set_err(ctx, RONK_EINVAL, "rank out of range");
  const size_t m = (size_t)1 << (log_n - log_g), blk = m >> log_g;
  const u64 wn = h_powmod(g, (p - 1) >> log_n, p);
  const u64 wg = h_powmod(g, (p - 1) >> log_g, p);
  // [ wt: 16 words | twbase: blk words ]
  Frame fr(ctx);
  u64* d_wt = nullptr;
  RONK_TRY(fr.take(&d_wt, 16 + blk));
  u64* d_tw = d_wt + 16;
  u64 h_wt[16];
  for (u32 j = 0; j < 16; j++) h_wt[j] = j < G ? h_powmod(wg, j, p) : 0;
  RONK_CUDA(ctx, cudaMemcpyAsync(d_wt, h_wt, sizeof(h_wt), cudaMemcpyHostToDevice, ctx->stream));
  RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // h_wt is a stack buffer
  // twbase[k''] = ω_n^(rank·blk + k'')
  RONK_TRY(ronk_field_powers_u64(ctx, p, wn, h_powmod(wn, (u64)rank * blk, p), (uint64_t*)d_tw, blk));
  PeerPtrs pp;
  for (u32 r = 0; r < 16; r++) pp.p[r] = r < G ? (const u64*)peer_bufs[r] : nullptr;
  for (u32 r = 0; r < G; r++)
    if (!pp.p[r]) return set_err(ctx, RONK_EINVAL, "null peer buffer");
  return with_field(ctx, p, 0, false, [&](const auto& f) {
    return launch(ctx, "ntt_cross_rank_fused", cross_rank_fused_kernel<std::decay_t<decltype(f)>>, grid_for(ctx, blk, 128, 16),
                  128, 0, false, f, pp, d_tw, d_wt, (u64*)out, G, blk, rank);
  });
}

int ronk_splitmix_fill_u64(ronk_ctx* ctx, uint64_t p, uint64_t seed, uint64_t* out, size_t n) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx || (n && !out) || p == 0) return set_err(ctx, RONK_EINVAL, "bad argument");
  if (n == 0) return RONK_OK;
  return launch(ctx, "splitmix_fill", splitmix_kernel, grid_for(ctx, n, 256), 256, 0, false, p, seed, (u64*)out, n);
}

// ---- host-pointer variants -------------------------------------------------------------------
// Unlike the device variants, n == 0 returns RONK_OK before the modulus or the op is looked at.
int ronk_field_binop_u64_host(ronk_ctx* ctx, int op, uint64_t p, const uint64_t* a, const uint64_t* b, uint64_t* out,
                              size_t n) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx || (n && (!a || !b || !out))) return set_err(ctx, RONK_EINVAL, "null argument");
  if (n == 0) return RONK_OK;
  Staged s[] = {{n * 8, a}, {n * 8, b}, {n * 8, nullptr, out}};
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  u64 *da = s[0].dev, *db = s[1].dev, *dout = s[2].dev;
  int rc;
  switch (op) {
    case 0: rc = ronk_field_add_u64(ctx, p, da, db, dout, n); break;
    case 1: rc = ronk_field_sub_u64(ctx, p, da, db, dout, n); break;
    case 2: rc = ronk_field_mul_u64(ctx, p, da, db, dout, n); break;
    case 3: rc = ronk_field_div_u64(ctx, p, da, db, dout, n); break;
    default: return set_err(ctx, RONK_EINVAL, "unknown op");
  }
  return stage_out(ctx, rc, s);
}

int ronk_field_unop_u64_host(ronk_ctx* ctx, int op, uint64_t p, const uint64_t* a, uint64_t* out, size_t n) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx || (n && (!a || !out))) return set_err(ctx, RONK_EINVAL, "null argument");
  if (n == 0) return RONK_OK;
  Staged s[] = {{n * 8, a}, {n * 8, nullptr, out}};
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  const int rc = (op == 0)   ? ronk_field_neg_u64(ctx, p, s[0].dev, s[1].dev, n)
                 : (op == 1) ? ronk_field_inv_u64(ctx, p, s[0].dev, s[1].dev, n)
                             : set_err(ctx, RONK_EINVAL, "unknown op");
  return stage_out(ctx, rc, s);
}

int ronk_field_pow_u64_host(ronk_ctx* ctx, uint64_t p, const uint64_t* a, uint64_t e, uint64_t* out, size_t n) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx || (n && (!a || !out))) return set_err(ctx, RONK_EINVAL, "null argument");
  if (n == 0) return RONK_OK;
  Staged s[] = {{n * 8, a}, {n * 8, nullptr, out}};
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  return stage_out(ctx, ronk_field_pow_u64(ctx, p, s[0].dev, e, s[1].dev, n), s);
}

}  // extern "C"
