// ronk_b200.hpp — header-only C++17 host mirror of ronkathon's Rust surface for the hot path,
// written above the C ABI (ronk_b200.h).  The reference's host language (Rust) is not available
// in this build environment, so this is the compiled-language host layer; bindings/rust/ holds
// the equivalent `extern "C"` declarations for a Rust `-sys` crate (unbuilt here).
//
//   ronk::PrimeField<P>                 ↔ src/algebra/field/prime/mod.rs:39-90, prime/arithmetic.rs
//   ronk::Polynomial<Basis, F, D>       ↔ src/polynomial/mod.rs:35-485, polynomial/arithmetic.rs
//   ronk::AffinePoint, ronk::kzg::*     ↔ src/curve/mod.rs:67-235, src/kzg/setup.rs:10-78
//
// Same names, argument meaning and error behaviour: where the Rust code panics, these throw
// ronk::Panic (RONK_EINVAL).  Every arithmetic operation executes in libronk_b200.so's CUDA
// kernels — there is no host arithmetic and no CPU fallback.
#pragma once
#include <array>
#include <cstdint>
#include <optional>
#include <stdexcept>
#include <string>
#include <vector>

#include "ronk_b200.h"

namespace ronk {

struct Error : std::runtime_error {
  int code;
  Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};
struct Panic : Error {  // the reference would panic / assert / unwrap(None) here
  explicit Panic(const std::string& m) : Error(RONK_EINVAL, m) {}
};

class Context {
 public:
  explicit Context(int device = 0, void* stream = nullptr) {
    int rc = ronk_ctx_create(&ctx_, device, stream);
    if (rc != RONK_OK) throw Error(rc, "ronk_ctx_create failed: an H100 (sm_90) GPU is required, there is no CPU fallback");
  }
  ~Context() { ronk_ctx_destroy(ctx_); }
  Context(const Context&) = delete;
  Context& operator=(const Context&) = delete;
  ronk_ctx* get() const { return ctx_; }
  void check(int rc) const {
    if (rc == RONK_OK) return;
    if (rc == RONK_EINVAL) throw Panic(ronk_last_error(ctx_));
    throw Error(rc, ronk_last_error(ctx_));
  }
  static Context& global() {
    static Context c;
    return c;
  }

 private:
  ronk_ctx* ctx_ = nullptr;
};

// ---------------------------------------------------------------------------------------------
// PrimeField<P>
// ---------------------------------------------------------------------------------------------
template <uint64_t P>
struct PrimeField {
  uint64_t value = 0;
  static constexpr uint64_t ORDER = P;  // Finite::ORDER
  PrimeField() = default;
  explicit PrimeField(uint64_t v) : value(v % P) {}  // PrimeField::new (prime/mod.rs:48-51)
  static PrimeField ZERO() { return PrimeField(0); }
  static PrimeField ONE() { return PrimeField(1); }
  static PrimeField PRIMITIVE_ELEMENT() {  // prime/mod.rs:87-90
    uint64_t g;
    if (ronk_field_generator(P, &g) != RONK_OK) throw Panic("generator not found");
    return PrimeField(g);
  }
  static PrimeField primitive_root_of_unity(uint64_t n) {  // field/mod.rs:70-75
    uint64_t w;
    if (ronk_root_of_unity(P, PRIMITIVE_ELEMENT().value, n, &w) != RONK_OK) throw Panic("n must divide p^q - 1");
    return PrimeField(w);
  }
  friend PrimeField operator+(PrimeField a, PrimeField b) { return bin(0, a, b); }
  friend PrimeField operator-(PrimeField a, PrimeField b) { return bin(1, a, b); }
  friend PrimeField operator*(PrimeField a, PrimeField b) { return bin(2, a, b); }
  friend PrimeField operator/(PrimeField a, PrimeField b) { return bin(3, a, b); }  // panics on b == 0
  PrimeField operator-() const {
    PrimeField r;
    Context::global().check(ronk_field_unop_u64_host(Context::global().get(), 0, P, &value, &r.value, 1));
    return r;
  }
  std::optional<PrimeField> inverse() const {  // prime/mod.rs:62-72
    PrimeField r;
    int rc = ronk_field_unop_u64_host(Context::global().get(), 1, P, &value, &r.value, 1);
    if (rc == RONK_EINVAL) return std::nullopt;
    Context::global().check(rc);
    return r;
  }
  PrimeField pow(uint64_t e) const {  // prime/mod.rs:74-84
    PrimeField r;
    Context::global().check(ronk_field_pow_u64_host(Context::global().get(), P, &value, e, &r.value, 1));
    return r;
  }
  bool operator==(const PrimeField& o) const { return value == o.value; }
  bool operator!=(const PrimeField& o) const { return value != o.value; }

 private:
  static PrimeField bin(int op, PrimeField a, PrimeField b) {
    PrimeField r;
    Context::global().check(ronk_field_binop_u64_host(Context::global().get(), op, P, &a.value, &b.value, &r.value, 1));
    return r;
  }
};
using PlutoBaseField = PrimeField<101>;                     // prime/mod.rs:27
using PlutoScalarField = PrimeField<17>;                    // prime/mod.rs:31
using GoldilocksField = PrimeField<RONK_GOLDILOCKS>;        // the 64-bit instantiation

// ---------------------------------------------------------------------------------------------
// Polynomial<Basis, F, D>  (D is a run-time length: SURVEY §8a delta D5)
// ---------------------------------------------------------------------------------------------
struct Monomial {};
struct Lagrange {};

template <class B, class F>
struct Polynomial {
  std::vector<F> coefficients;
  Polynomial() = default;
  explicit Polynomial(std::vector<F> c) : coefficients(std::move(c)) {
    if constexpr (std::is_same_v<B, Lagrange>)  // Lagrange::new asserts (polynomial/mod.rs:361)
      if (coefficients.empty() || (F::ORDER - 1) % coefficients.size() != 0) throw Panic("(ORDER - 1) % n != 0");
  }
  size_t num_terms() const { return coefficients.size(); }
  bool operator==(const Polynomial& o) const { return coefficients == o.coefficients; }

  F evaluate(F x) const {
    F out;
    auto raw = to_raw();
    if constexpr (std::is_same_v<B, Monomial>) {  // polynomial/mod.rs:133-139
      ctx().check(ronk_poly_eval_u64_host(ctx().get(), F::ORDER, raw.data(), raw.size(), &x.value, 1, &out.value));
    } else {  // polynomial/mod.rs:382-415
      ctx().check(ronk_poly_lagrange_eval_u64_host(ctx().get(), F::ORDER, F::PRIMITIVE_ELEMENT().value, raw.data(),
                                                   raw.size(), x.value, &out.value));
    }
    return out;
  }
  // evaluate at many points (Lagrange: the barycentric form in O(n) per point, 0 at a node, as evaluate)
  std::vector<F> evaluate_many(const std::vector<F>& xs) const {
    auto raw = to_raw();
    std::vector<uint64_t> rx(xs.size()), out(xs.size());
    for (size_t i = 0; i < xs.size(); i++) rx[i] = xs[i].value;
    if constexpr (std::is_same_v<B, Monomial>) {
      ctx().check(ronk_poly_eval_u64_host(ctx().get(), F::ORDER, raw.data(), raw.size(), rx.data(), rx.size(), out.data()));
    } else {
      ctx().check(ronk_poly_lagrange_eval_batch_u64_host(ctx().get(), F::ORDER, F::PRIMITIVE_ELEMENT().value, raw.data(),
                                                         raw.size(), 1, 1, rx.data(), rx.size(), out.data()));
    }
    return from_raw(out);
  }
  // evaluate each of `polys` (monomial basis, equal lengths) at the same points (Shamir split of many secrets): one
  // batched call sharing one subproduct tree; row b holds polys[b] at every xs[i]
  static std::vector<std::vector<F>> evaluate_many_batch(const std::vector<Polynomial>& polys, const std::vector<F>& xs) {
    static_assert(std::is_same_v<B, Monomial>);
    const size_t d = polys.empty() ? 0 : polys[0].num_terms(), m = xs.size();
    std::vector<uint64_t> rc(polys.size() * d), rx(m), out(polys.size() * m);
    for (size_t b = 0; b < polys.size(); b++) {
      if (polys[b].num_terms() != d) throw Panic("evaluate_many_batch: polynomials of different lengths");
      for (size_t j = 0; j < d; j++) rc[b * d + j] = polys[b].coefficients[j].value;
    }
    for (size_t i = 0; i < m; i++) rx[i] = xs[i].value;
    ctx().check(ronk_poly_multieval_batch_u64_host(ctx().get(), F::ORDER, F::PRIMITIVE_ELEMENT().value, rc.data(), d,
                                                   (uint32_t)polys.size(), rx.data(), m, out.data()));
    std::vector<std::vector<F>> rows(polys.size());
    for (size_t b = 0; b < polys.size(); b++)
      rows[b] = from_raw(std::vector<uint64_t>(out.begin() + b * m, out.begin() + (b + 1) * m));
    return rows;
  }
  // kzg::open (kzg/setup.rs:63-78) in evaluation form: f(z) and the evaluations of (f - f(z)) / (X - z) on the nodes
  std::pair<F, Polynomial> open(F z) const {
    static_assert(std::is_same_v<B, Lagrange>);
    auto raw = to_raw();
    std::vector<uint64_t> q(raw.size());
    F v;
    ctx().check(ronk_poly_lagrange_open_u64_host(ctx().get(), F::ORDER, F::PRIMITIVE_ELEMENT().value, raw.data(), raw.size(),
                                                 1, 1, z.value, &v.value, q.data()));
    return {v, Polynomial(from_raw(q))};
  }
  size_t degree() const {  // polynomial/mod.rs:113-115
    for (size_t i = coefficients.size(); i-- > 0;)
      if (coefficients[i] != F::ZERO()) return i;
    return 0;
  }
  F leading_coefficient() const {  // polynomial/mod.rs:120-122
    for (size_t i = coefficients.size(); i-- > 0;)
      if (coefficients[i] != F::ZERO()) return coefficients[i];
    return F::ZERO();
  }
  Polynomial<Lagrange, F> dft() const {  // polynomial/mod.rs:240-258
    static_assert(std::is_same_v<B, Monomial>);
    auto raw = to_raw();
    std::vector<uint64_t> out(raw.size());
    ctx().check(ronk_dft_u64_host(ctx().get(), F::ORDER, F::PRIMITIVE_ELEMENT().value, raw.data(), raw.size(), out.data()));
    return Polynomial<Lagrange, F>(from_raw(out));
  }
  Polynomial<Lagrange, F> fft() const {  // polynomial/mod.rs:273-290
    static_assert(std::is_same_v<B, Monomial>);
    return Polynomial<Lagrange, F>(from_raw(ntt(false)));
  }
  Polynomial<Monomial, F> ifft() const {  // polynomial/mod.rs:430-453
    static_assert(std::is_same_v<B, Lagrange>);
    return Polynomial<Monomial, F>(from_raw(ntt(true)));
  }
  friend Polynomial operator*(const Polynomial& a, const Polynomial& b) {  // arithmetic.rs:97-119
    if (a.coefficients.empty() || b.coefficients.empty()) throw Panic("D + D2 - 1 underflows");
    auto ra = a.to_raw(), rb = b.to_raw();
    std::vector<uint64_t> out(ra.size() + rb.size() - 1);
    ctx().check(ronk_poly_mul_u64_host(ctx().get(), F::ORDER, F::PRIMITIVE_ELEMENT().value, ra.data(), ra.size(), rb.data(),
                                       rb.size(), out.data()));
    return Polynomial(from_raw(out));
  }
  friend Polynomial operator+(const Polynomial& a, const Polynomial& b) { return addsub(a, b, false); }  // :16-35
  friend Polynomial operator-(const Polynomial& a, const Polynomial& b) { return addsub(a, b, true); }   // :49-68
  std::pair<Polynomial, Polynomial> quotient_and_remainder(const Polynomial& rhs) const {  // mod.rs:170-225
    auto ra = to_raw(), rb = rhs.to_raw();
    std::vector<uint64_t> q(ra.size()), r(ra.size());
    ctx().check(ronk_poly_divrem_u64_host(ctx().get(), F::ORDER, ra.data(), ra.size(), rb.data(), rb.size(), q.data(), r.data()));
    return {Polynomial(from_raw(q)), Polynomial(from_raw(r))};
  }
  friend Polynomial operator/(const Polynomial& a, const Polynomial& b) { return a.quotient_and_remainder(b).first; }
  friend Polynomial operator%(const Polynomial& a, const Polynomial& b) { return a.quotient_and_remainder(b).second; }

  std::vector<uint64_t> to_raw() const {
    std::vector<uint64_t> r(coefficients.size());
    for (size_t i = 0; i < r.size(); i++) r[i] = coefficients[i].value;
    return r;
  }
  static std::vector<F> from_raw(const std::vector<uint64_t>& r) {
    std::vector<F> c(r.size());
    for (size_t i = 0; i < r.size(); i++) c[i].value = r[i];
    return c;
  }

 private:
  static Context& ctx() { return Context::global(); }
  std::vector<uint64_t> ntt(bool inverse) const {
    const size_t n = coefficients.size();
    if (n == 0 || (n & (n - 1))) throw Panic("D must be a power of two");  // mod.rs:274
    uint32_t lg = 0;
    while ((size_t(1) << lg) < n) lg++;
    auto raw = to_raw();
    ctx().check(ronk_ntt_u64_host(ctx().get(), F::ORDER, F::PRIMITIVE_ELEMENT().value, raw.data(), lg, 1, inverse ? 1 : 0));
    return raw;
  }
  static Polynomial addsub(const Polynomial& a, const Polynomial& b, bool sub) {
    // element-wise through the field kernels with b zero-extended / truncated to a's length
    auto ra = a.to_raw();
    std::vector<uint64_t> rb(ra.size(), 0), out(ra.size());
    for (size_t i = 0; i < ra.size() && i < b.coefficients.size(); i++) rb[i] = b.coefficients[i].value;
    if (!ra.empty())
      ctx().check(ronk_field_binop_u64_host(ctx().get(), sub ? 1 : 0, F::ORDER, ra.data(), rb.data(), out.data(), ra.size()));
    return Polynomial(from_raw(out));
  }
};

// ---------------------------------------------------------------------------------------------
// AffinePoint<PlutoExtendedCurve> and kzg
// ---------------------------------------------------------------------------------------------
struct AffinePoint {
  std::array<uint8_t, 4> raw{0xFF, 0xFF, 0xFF, 0xFF};  // x0,x1,y0,y1; 0xFF×4 = Infinity
  static AffinePoint Infinity() { return AffinePoint{}; }
  static AffinePoint make(uint8_t x0, uint8_t x1, uint8_t y0, uint8_t y1) {  // AffinePoint::new (curve/mod.rs:78-82)
    AffinePoint p;
    p.raw = {x0, x1, y0, y1};
    (void)(p + Infinity());  // the add kernel validates is_on_curve
    return p;
  }
  bool is_infinity() const { return raw == Infinity().raw; }
  friend AffinePoint operator+(const AffinePoint& a, const AffinePoint& b) {  // curve/mod.rs:178-213
    AffinePoint r;
    Context::global().check(ronk_point_add_pluto_ext_host(Context::global().get(), a.raw.data(), b.raw.data(), r.raw.data(), 1));
    return r;
  }
  AffinePoint operator-() const {  // curve/mod.rs:225-235
    AffinePoint r;
    Context::global().check(ronk_point_neg_pluto_ext_host(Context::global().get(), raw.data(), r.raw.data(), 1));
    return r;
  }
  friend AffinePoint operator*(const AffinePoint& a, PlutoScalarField s) {  // curve/mod.rs:157-172
    AffinePoint r;
    uint8_t sc = (uint8_t)s.value;
    Context::global().check(ronk_point_smul_pluto_ext_host(Context::global().get(), a.raw.data(), &sc, r.raw.data(), 1));
    return r;
  }
  bool operator==(const AffinePoint& o) const { return raw == o.raw; }
};
inline AffinePoint G1_GENERATOR() { AffinePoint p; p.raw = {1, 0, 2, 0}; return p; }    // pluto_curve.rs:36-37
inline AffinePoint G2_GENERATOR() { AffinePoint p; p.raw = {36, 0, 0, 31}; return p; }  // pluto_curve.rs:46-49

namespace kzg {
// kzg/setup.rs:10-43
inline std::pair<std::vector<AffinePoint>, std::vector<AffinePoint>> setup() {
  std::vector<AffinePoint> g1, g2;
  PlutoScalarField tau(2);
  for (int i = 0; i < 7; i++) {
    g1.push_back(G1_GENERATOR() * tau.pow(i));
    if (i < 2) g2.push_back(G2_GENERATOR() * tau.pow(i));
  }
  return {g1, g2};
}
// kzg/setup.rs:48-60 — Pippenger bucket MSM on the device
inline AffinePoint commit(const std::vector<PlutoScalarField>& coeffs, const std::vector<AffinePoint>& g1_srs) {
  std::vector<uint8_t> pts(g1_srs.size() * 4), sc(coeffs.size());
  for (size_t i = 0; i < g1_srs.size(); i++)
    for (int k = 0; k < 4; k++) pts[4 * i + k] = g1_srs[i].raw[k];
  for (size_t i = 0; i < coeffs.size(); i++) sc[i] = (uint8_t)coeffs[i].value;
  AffinePoint out;
  Context::global().check(ronk_msm_pluto_ext_host(Context::global().get(), pts.data(), g1_srs.size(), sc.data(), sc.size(), out.raw.data()));
  return out;
}
// kzg/setup.rs:63-78
inline AffinePoint open(const std::vector<PlutoScalarField>& coeffs, PlutoScalarField z, const std::vector<AffinePoint>& g1_srs) {
  Polynomial<Monomial, PlutoScalarField> poly(coeffs);
  Polynomial<Monomial, PlutoScalarField> divisor({-z, PlutoScalarField::ONE()});
  auto q = poly / divisor;
  return commit(q.coefficients, g1_srs);
}
}  // namespace kzg

// ---------------------------------------------------------------------------------------------
// codes::reed_solomon (src/codes/reed_solomon.rs) — §8f "next" row: Message / Codeword over PrimeField<P>
// ---------------------------------------------------------------------------------------------
namespace codes {

template <class F>
struct Coordinate {  // reed_solomon.rs:28-35
  F x, y;
  bool operator==(const Coordinate& o) const { return x == o.x && y == o.y; }
};

template <class F>
struct Message {  // reed_solomon.rs:13-17
  std::vector<F> data;
  explicit Message(std::vector<F> d) : data(std::move(d)) {}

  // encode::<N> (reed_solomon.rs:42-52): (ω_N^i, m(ω_N^i)) for i < N — the transform of the message
  // zero-padded to N coefficients (ronk_ntt for a power of two, ronk_dft otherwise).
  std::vector<Coordinate<F>> encode(size_t n) const {
    if (n < data.size()) throw Panic("Code size must be greater than or equal to K");  // assert_ge, :110-112
    const F w = F::primitive_root_of_unity(n);                                         // panics if n does not divide P - 1
    std::vector<F> padded(data);
    padded.resize(n, F::ZERO());
    Polynomial<Monomial, F> poly(padded);
    const auto ys = (n > 1 && (n & (n - 1)) == 0) ? poly.fft().coefficients : poly.dft().coefficients;
    std::vector<Coordinate<F>> out(n);
    F x = F::ONE();
    for (size_t i = 0; i < n; i++, x = x * w) out[i] = {x, ys[i]};
    return out;
  }
  // decode::<M> (reed_solomon.rs:55-107): interpolation through the first K coordinates.
  static Message decode(const std::vector<Coordinate<F>>& codeword, size_t k) {
    if (codeword.size() < k) throw Panic("Code size must be greater than or equal to K");
    std::vector<uint64_t> xs(k), ys(k), out(k);
    for (size_t i = 0; i < k; i++) { xs[i] = codeword[i].x.value; ys[i] = codeword[i].y.value; }
    Context::global().check(ronk_poly_interpolate_u64_host(Context::global().get(), F::ORDER, xs.data(), ys.data(), k, out.data()));
    return Message(Polynomial<Monomial, F>::from_raw(out));
  }
  // decode of many codewords whose first k coordinates share their x's: one batched interpolation over one tree
  static std::vector<Message> decode_batch(const std::vector<std::vector<Coordinate<F>>>& codewords, size_t k) {
    std::vector<uint64_t> xs(k), ys(codewords.size() * k), out(codewords.size() * k);
    for (size_t b = 0; b < codewords.size(); b++) {
      if (codewords[b].size() < k) throw Panic("Code size must be greater than or equal to K");
      for (size_t i = 0; i < k; i++) {
        if (b == 0) xs[i] = codewords[0][i].x.value;
        else if (codewords[b][i].x.value != xs[i]) throw Panic("decode_batch: codewords on different x coordinates");
        ys[b * k + i] = codewords[b][i].y.value;
      }
    }
    Context::global().check(ronk_poly_interpolate_batch_u64_host(Context::global().get(), F::ORDER, F::PRIMITIVE_ELEMENT().value,
                                                                 xs.data(), ys.data(), k, (uint32_t)codewords.size(), out.data()));
    std::vector<Message> msgs;
    for (size_t b = 0; b < codewords.size(); b++)
      msgs.emplace_back(Polynomial<Monomial, F>::from_raw(std::vector<uint64_t>(out.begin() + b * k, out.begin() + (b + 1) * k)));
    return msgs;
  }
};

}  // namespace codes

// ---------------------------------------------------------------------------------------------
// multi-GPU modes (SURVEY §8e): one Context per GPU; the library owns the NCCL communicator.  The host only
// carries the 128-byte id from rank 0 to the other ranks (MPI_Bcast, a TCP store …).
// ---------------------------------------------------------------------------------------------
namespace dist {

inline std::array<uint8_t, RONK_NCCL_UNIQUE_ID_BYTES> unique_id() {  // rank 0
  std::array<uint8_t, RONK_NCCL_UNIQUE_ID_BYTES> id{};
  const int rc = ronk_dist_unique_id(id.data());
  if (rc != RONK_OK) throw Error(rc, "ronk_dist_unique_id: libnccl.so.2 not available");
  return id;
}
inline void init(Context& c, const std::array<uint8_t, RONK_NCCL_UNIQUE_ID_BYTES>& id, int rank, int world) {
  c.check(ronk_dist_init(c.get(), id.data(), rank, world));
}
inline void finalize(Context& c) { c.check(ronk_dist_finalize(c.get())); }
// device pointers, as in the C ABI
inline std::pair<uint64_t, uint64_t> ntt_batch_sharded(Context& c, uint64_t p, uint64_t g, uint64_t* shard, uint32_t log_n,
                                                       uint64_t total_batch, bool inverse = false) {
  uint64_t lo = 0, hi = 0;
  c.check(ronk_ntt_u64_batch_sharded(c.get(), p, g, shard, log_n, total_batch, inverse ? 1 : 0, &lo, &hi));
  return {lo, hi};
}
inline void ntt(Context& c, uint64_t p, uint64_t g, uint64_t* local, uint32_t log_n, uint32_t batch = 1,
                int flavour = RONK_DIST_FUSED) {
  c.check(ronk_ntt_u64_dist(c.get(), p, g, local, log_n, batch, flavour));
}
// G = 2^log_g virtual ranks on one device (validation / capacity mode): data = [rank][batch][n/G]
inline void ntt_virtual(Context& c, uint64_t p, uint64_t g, uint64_t* data, uint32_t log_n, uint32_t batch, uint32_t log_g,
                        int flavour = RONK_DIST_FUSED) {
  c.check(ronk_ntt_u64_dist_virtual(c.get(), p, g, data, log_n, batch, log_g, flavour));
}
inline AffinePoint commit(Context& c, const uint8_t* points, const uint8_t* scalars, size_t n) {
  AffinePoint out;
  c.check(ronk_msm_pluto_ext_dist(c.get(), points, n, scalars, n, out.raw.data()));
  return out;
}

}  // namespace dist

}  // namespace ronk
