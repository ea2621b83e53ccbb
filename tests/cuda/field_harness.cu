// field_harness.cu — TEST INFRASTRUCTURE: runs the device half of ronkathon_b200/csrc/field.cuh (and the
// radix-16 butterfly network of ntt_kernel.cuh) primitive by primitive, one element (or one 16-word group)
// per thread, so that tests/test_gpu_field_device.py can compare every primitive with exact integers on
// inputs chosen to reach each carry and borrow case.  The headers are included unchanged and compiled with
// the library's own flags (ronkathon_b200/csrc/flags.mk); a variant build passes one -D switch of field.cuh.
// Never linked into libronk_b200.so.
//
// Every export is synchronous and takes host pointers: allocate, copy in, launch, copy out, free; it
// returns the CUDA error code (cudaSuccess = 0), or -1 for an argument the harness has no kernel for.
#include <cuda_runtime.h>

#include <cstdint>
#include <utility>

#include "../../ronkathon_b200/csrc/field.cuh"
#include "../../ronkathon_b200/csrc/ntt_kernel.cuh"

using namespace ronk;

namespace {

// out[i] = op(a[i], b[i]) (b may be null: op(a[i], 0)).
template <class Op>
__global__ void elem_kernel(Op op, const u64* a, const u64* b, u64* out, u64 n) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = op(a[i], b ? b[i] : 0);
}

// One 16-word group per thread, held in registers across the whole network as in the transform kernels.
template <int NST, bool INV, class F>
__global__ void radix_kernel(F f, const u64* in, u64* out, u64 groups) {
  const u64 g = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= groups) return;
  u64 x[16];
#pragma unroll
  for (int i = 0; i < 16; i++) x[i] = in[16 * g + i];
  radix_network<NST, INV>(f, x);
#pragma unroll
  for (int i = 0; i < 16; i++) out[16 * g + i] = x[i];
}

struct Dev {
  u64* p = nullptr;
  cudaError_t alloc(const u64* h, u64 n) {
    cudaError_t e = cudaMalloc((void**)&p, (n ? n : 1) * sizeof(u64));
    if (e == cudaSuccess && h && n) e = cudaMemcpy(p, h, n * sizeof(u64), cudaMemcpyHostToDevice);
    return e;
  }
  ~Dev() { if (p) cudaFree(p); }
};

constexpr unsigned THREADS = 256;

template <class Op>
int run_elem(Op op, const u64* a, const u64* b, u64* out, u64 n) {
  Dev da, db, dout;
  cudaError_t e = da.alloc(a, n);
  if (e == cudaSuccess && b) e = db.alloc(b, n);
  if (e == cudaSuccess) e = dout.alloc(nullptr, n);
  if (e != cudaSuccess) return (int)e;
  if (n) {
    elem_kernel<<<(unsigned)((n + THREADS - 1) / THREADS), THREADS>>>(op, da.p, db.p, dout.p, n);
    if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
    if ((e = cudaMemcpy(out, dout.p, n * sizeof(u64), cudaMemcpyDeviceToHost)) != cudaSuccess) return (int)e;
  }
  return (int)cudaDeviceSynchronize();
}

template <int NST, bool INV, class F>
int run_radix(const F& f, const u64* in, u64* out, u64 groups) {
  Dev din, dout;
  cudaError_t e = din.alloc(in, 16 * groups);
  if (e == cudaSuccess) e = dout.alloc(nullptr, 16 * groups);
  if (e != cudaSuccess) return (int)e;
  if (groups) {
    radix_kernel<NST, INV><<<(unsigned)((groups + THREADS - 1) / THREADS), THREADS>>>(f, din.p, dout.p, groups);
    if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
    if ((e = cudaMemcpy(out, dout.p, 16 * groups * sizeof(u64), cudaMemcpyDeviceToHost)) != cudaSuccess) return (int)e;
  }
  return (int)cudaDeviceSynchronize();
}

template <class F, bool INV>
int radix_dispatch(const F& f, int nst, const u64* in, u64* out, u64 groups) {
  switch (nst) {
    case 1: return run_radix<1, INV>(f, in, out, groups);
    case 2: return run_radix<2, INV>(f, in, out, groups);
    case 3: return run_radix<3, INV>(f, in, out, groups);
    case 4: return run_radix<4, INV>(f, in, out, groups);
    default: return -1;
  }
}

// ---- the element-wise operations, as functors the kernel template takes by value --------------------------
enum { OP_ADD = 0, OP_SUB = 1, OP_NEG = 2, OP_MUL = 3, OP_MUL_TW = 4, OP_POW = 5, OP_REDC_MUL = 6, OP_TO_TW = 7 };

template <class F>
struct FieldOp {
  F f;
  int op;
  __device__ u64 operator()(u64 a, u64 b) const {
    switch (op) {
      case OP_ADD: return f.add(a, b);
      case OP_SUB: return f.sub(a, b);
      case OP_NEG: return f.neg(a);
      case OP_MUL: return f.mul(a, b);
      case OP_MUL_TW: return f.mul_tw(a, b);
      case OP_POW: return field_pow(f, a, b);
      case OP_TO_TW: return f.to_tw(a);
      default: return 0;
    }
  }
};
struct MontRedc {
  MontField f;
  __device__ u64 operator()(u64 a, u64 b) const { return f.redc_mul(a, b); }
};

template <int S>
struct Pow2 {
  __device__ u64 operator()(u64 a, u64) const { return GoldilocksField{}.mul_pow2<S>(a); }
};
template <int S>
int run_pow2(const u64* a, u64* out, u64 n) { return run_elem(Pow2<S>{}, a, nullptr, out, n); }
template <int... S>
int pow2_dispatch(int s, const u64* a, u64* out, u64 n, std::integer_sequence<int, S...>) {
  static int (*const table[])(const u64*, u64*, u64) = {&run_pow2<S>...};
  return table[s](a, out, n);
}

// w16<E, INV>(a) (sub = 0) or w16_sub<E, INV>(a, b) (sub = 1)
template <class F, int E, bool INV, bool SUB>
struct W16 {
  F f;
  __device__ u64 operator()(u64 a, u64 b) const {
    if constexpr (SUB) return f.template w16_sub<E, INV>(a, b);
    else return f.template w16<E, INV>(a);
  }
};
template <class F, int E, bool INV, bool SUB>
int run_w16(const F& f, const u64* a, const u64* b, u64* out, u64 n) {
  return run_elem(W16<F, E, INV, SUB>{f}, a, SUB ? b : nullptr, out, n);
}
template <class F, bool INV, bool SUB, int... E>
int w16_dispatch(const F& f, int e, const u64* a, const u64* b, u64* out, u64 n, std::integer_sequence<int, E...>) {
  static int (*const table[])(const F&, const u64*, const u64*, u64*, u64) = {&run_w16<F, E, INV, SUB>...};
  return table[e](f, a, b, out, n);
}
template <class F>
int w16_any(const F& f, int e, int inv, int sub, const u64* a, const u64* b, u64* out, u64 n) {
  if (e < 0 || e >= 8) return -1;
  using seq = std::make_integer_sequence<int, 8>;
  if (inv) return sub ? w16_dispatch<F, true, true>(f, e, a, b, out, n, seq{}) : w16_dispatch<F, true, false>(f, e, a, b, out, n, seq{});
  return sub ? w16_dispatch<F, false, true>(f, e, a, b, out, n, seq{}) : w16_dispatch<F, false, false>(f, e, a, b, out, n, seq{});
}

// The formula of make_mont_field() in ronkathon_b200/csrc/ntt.cu: ω16^±e in Montgomery form where the
// 2-adicity (capped at 4) allows it, R mod p elsewhere.
MontField mont_field(u64 p, u64 g, bool inverse) {
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

}  // namespace

extern "C" {

// Goldilocks (GoldilocksField, the inline-PTX path).  op: 0 add, 1 sub, 2 neg(a), 3 mul, 4 mul_tw, 5 a^b.
int fh_gl_op(int op, const uint64_t* a, const uint64_t* b, uint64_t* out, uint64_t n) {
  if (op < OP_ADD || op > OP_POW) return -1;
  return run_elem(FieldOp<GoldilocksField>{GoldilocksField{}, op}, a, op == OP_NEG ? nullptr : b, out, n);
}
// out[i] = mul_pow2<s>(a[i]), s in [0, 192)
int fh_gl_mul_pow2(int s, const uint64_t* a, uint64_t* out, uint64_t n) {
  if (s < 0 || s >= 192) return -1;
  return pow2_dispatch(s, a, out, n, std::make_integer_sequence<int, 192>{});
}
int fh_gl_w16(int e, int inv, int sub, const uint64_t* a, const uint64_t* b, uint64_t* out, uint64_t n) {
  return w16_any(GoldilocksField{}, e, inv, sub, a, b, out, n);
}
// radix_network<nst, inv> on each 16-word group of in
int fh_gl_radix(int nst, int inv, const uint64_t* in, uint64_t* out, uint64_t groups) {
  GoldilocksField f;
  return inv ? radix_dispatch<GoldilocksField, true>(f, nst, in, out, groups)
             : radix_dispatch<GoldilocksField, false>(f, nst, in, out, groups);
}

// MontField for the odd modulus p, with the ω16 table of generator g (forward, or inverse if inv).
// op: 0 add, 1 sub, 2 neg(a), 3 mul, 4 mul_tw (b in Montgomery form), 5 a^b, 6 redc_mul (a·b·2^-64), 7 to_tw(a).
int fh_mont_op(uint64_t p, int op, const uint64_t* a, const uint64_t* b, uint64_t* out, uint64_t n) {
  const MontField f = mont_field(p, 0, false);
  if (op == OP_REDC_MUL) return run_elem(MontRedc{f}, a, b, out, n);
  if (op < OP_ADD || op > OP_TO_TW) return -1;
  return run_elem(FieldOp<MontField>{f, op}, a, (op == OP_NEG || op == OP_TO_TW) ? nullptr : b, out, n);
}
int fh_mont_w16(uint64_t p, uint64_t g, int e, int inv, int sub, const uint64_t* a, const uint64_t* b, uint64_t* out,
                uint64_t n) {
  return w16_any(mont_field(p, g, inv != 0), e, inv, sub, a, b, out, n);
}
int fh_mont_radix(uint64_t p, uint64_t g, int nst, int inv, const uint64_t* in, uint64_t* out, uint64_t groups) {
  const MontField f = mont_field(p, g, inv != 0);
  return inv ? radix_dispatch<MontField, true>(f, nst, in, out, groups)
             : radix_dispatch<MontField, false>(f, nst, in, out, groups);
}

}  // extern "C"
