// ronk_internal.h — context object and launch helpers shared by the translation units of
// libronk_b200.so.  Not part of the public ABI (include/ronk_b200.h is).
#pragma once
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <map>
#include <string>
#include <tuple>
#include <type_traits>
#include <unordered_set>
#include <utility>
#include <vector>

#include "../../include/ronk_b200.h"
#include "field.cuh"

namespace ronk {

struct ProfRec {
  char name[32];
  cudaEvent_t start, stop;
};

// Owns one cudaMalloc allocation of T and frees it when destroyed; move-only.  Its user has bound the device, as every
// entry point does through DeviceGuard.
template <class T>
class DevBuf {
 public:
  DevBuf() = default;
  DevBuf(DevBuf&& o) noexcept : p_(o.p_) { o.p_ = nullptr; }
  DevBuf& operator=(DevBuf&& o) noexcept { reset(); std::swap(p_, o.p_); return *this; }
  ~DevBuf() { reset(); }
  // frees what it held and allocates count elements; a failure is reported as RONK_CUDA does (no message for a null ctx)
  int alloc(ronk_ctx* ctx, size_t count);
  T* get() const { return p_; }
  explicit operator bool() const { return p_ != nullptr; }
  void reset() { if (p_) { cudaFree(p_); p_ = nullptr; } }

 private:
  T* p_ = nullptr;
};

struct NttPlan {
  u64 p = 0, g = 0;
  u32 log_n = 0;
  bool two_pass = false;
  u32 log_n1 = 0, log_n2 = 0;
  DevBuf<u64> tw1;           // ω_{N1}^e (single pass: ω_n^e), twiddle form
  DevBuf<u64> tw2;           // ω_{N2}^e == ω_n^(e·N1)
  DevBuf<u64> tw1_2d[2];     // per-round 2-D tables of pass 1 / single (forward, inverse)
  DevBuf<u64> tw2_2d[2];     // per-round 2-D tables of pass 2
  DevBuf<u64> tw_lo;         // ω_n^x, x < N1
  DevBuf<u64> tw_hi_inv;     // ω_n^(y·N1) · n^-1
  u64 scale_inv = 0;         // n^-1, twiddle form (single-pass inverse)
  // full inter-pass twiddle tables ω_n^(±j2·k1) [· n^-1] in the pass-1 workspace layout, per direction and
  // per log2(C2) of that layout (built on first use; n words each)
  std::map<u32, DevBuf<u64>> tw_full[2];
  // three-pass 2^24 transform (ntt3_kernel.cuh): ω_256^x and the 64 Ki-entry pass-2 table, per direction
  DevBuf<u64> tw256[2], t2[2];
  DevBuf<u64> t1[2];  // optional n-word pass-1 twiddle table (log n ≤ RONK_NTT3_T1)
};

// The context's per-call device scratch (Frame below): device blocks, of which blocks[0, used) hold the live regions,
// the last of them in its first `top` bytes.
struct Scratch {
  struct Block {
    char* base;
    size_t bytes;
  };
  std::vector<Block> blocks;
  size_t used = 0;
  size_t top = 0;
};

}  // namespace ronk

// Tuning switches, read from the environment ONCE at ronk_ctx_create (never on the launch path).
struct ronk_tune {
  int ntt3_min_batch16 = 1; // RONK_NTT3_MIN_BATCH16: smallest batch of 2^16-point transforms that takes the 256-point-tile kernels
  int ntt16_cluster_max_batch = 2;  // RONK_NTT16_CLUSTER_MAX_BATCH: up to this many 2^16-point transforms go through ntt16c_kernel
                                    // (one launch, 16-CTA cluster per transform, DSMEM exchange, in place, no workspace); 0 = never.
                                    // The two were equal at batch 1–2 and the two-launch path won from batch 4 on
  int ntt3_ng1_tiles = 6;   // RONK_NTT3_NG1_TILES: grids below this many tiles per SM run one group per thread (256 threads per tile);
                            // 6 beat 3 on two 2^20-point transforms and was equal elsewhere
  int ntt3_split = 1;       // RONK_NTT3_SPLIT: 2^17 … 2^19 and 2^25 / 2^26 as a radix-2/4/8 register pass + interleaved 2^16- / 2^24-point tile transforms
  int ntt3_split_min16 = 1; // RONK_NTT3_SPLIT_MIN16: … for 2^17 … 2^19 only from this many 2^16-point sub-transforms on.  Even ONE
                            // transform gained, so 1
  int ntt3_mid = 1;         // RONK_NTT3_MID: 2^21 … 2^23-point transforms through the 256-point-tile kernels (first pass of 32 / 64 / 128 points)
  int ntt3_20 = 1;          // RONK_NTT3_20: 2^20-point transforms as 16 interleaved 2^16-point tile transforms + one radix-16 pass
  int ntt3_t1 = 20;         // RONK_NTT3_T1: largest log2 n whose first pass takes its twiddles ω_n^(k1·m) from an n-word table
                            // per direction (built at first use; no memory → stepped) instead of stepping them; 0 = never,
                            // 24 = every size (2^25 / 2^26 follow their 2^24-point sub-transforms).  On the H100 the
                            // 128 MiB table of 2^24 makes pass 1 HBM-bound (stepped with RONK_NTT3_EARLY_TW=0: 0.331 vs 0.356
                            // ms per transform), while the L2-resident 8 MiB table of 2^20 still pays (0.0294 vs 0.0309 ms;
                            // profiles/r04_ab_ntt3_t1_early_tw.txt); 2^21 … 2^23 were not timed and stay stepped
  int ntt3_pdl = 1;         // RONK_NTT3_PDL: programmatic dependent launch between the three passes
  int ntt3 = 1;             // RONK_NTT3: 2^24-point transforms as three passes of 256-point tiles (ntt3_kernel.cuh)
  int pdl = 1;              // RONK_PDL: programmatic dependent launch of pass 2 behind pass 1
  int pf_dist2 = 1;         // RONK_PF_DIST2: the same for pass 2 of the specialised kernel (round 0 fed from HBM)
  int pf_dist = 1;          // RONK_PF_DIST: pass-1 L2 prefetch distance in waves of co-resident CTAs (0 = off)
  int single_tile_log = 12; // RONK_SINGLE_TILE_LOG: preferred tile size when several small transforms share a tile
  int tile1 = 14, tile2 = 13, tile_adapt = 1;  // RONK_TILE1 / RONK_TILE2 / RONK_TILE_ADAPT
  int fast12 = 0;           // RONK_FAST12: the specialised 4096-point-per-tile kernel (ntt12_kernel.cuh) where it applies — opt-in:
                            // 20 % fewer instructions but slower (DESIGN.md §3.3); needs RONK_TW_TABLE=1 for pass 1
  int msm_split = 0;        // RONK_MSM_SPLIT: ≥ 2^22 terms: every other term to an L2-resident histogram (global RED)
  int msm_coord = 1;        // RONK_MSM_COORD: kzg::commit in group coordinates (two dot products mod 102 + one lookup); 0 = the paths below
  int msm_hist = 1;         // RONK_MSM_HIST: kzg::commit through the point-indexed histogram (1) or the bucket kernels (0)
  int tw_table = 0;         // RONK_TW_TABLE: inter-pass twiddles from an n-word table (1) or stepped w ← w·ρ (0)
  int tree_min = -1;        // RONK_TREE_MIN: smallest size that takes the subproduct-tree path of from_roots / multieval /
                            // interpolate where its transforms fit; -1 = the measured crossovers (poly.cu)
  int anyntt_min = -1;      // RONK_ANYNTT_MIN: smallest n that takes Bluestein in ronk_ntt_any_u64 where its convolution fits;
                            // -1 = the measured crossover (ntt_any.cu)
  long long crt_mul_min = -1;  // RONK_CRT_MUL_MIN: smallest da·db that takes the multi-modular path of ronk_poly_mul_u64 where it
                               // fits, whatever min(da, db) (64-bit: da·db reaches 2^52); -1 = the measured crossovers on
                               // da·db and min(da, db) (poly_crt.cu)
  int poly_batch_path = 0;  // RONK_POLY_BATCH_PATH: path of ronk_poly_mul_batch_u64 where it applies: 0 = the measured crossovers,
                            // 1 = schoolbook, 2 = transforms (fused up to its cap, multi-modular where no root fits), 3 = the
                            // batched transforms even where the fused kernel fits (poly_batch.cu)
  int divrem_batch_path = 0;  // RONK_DIVREM_BATCH_PATH: path of ronk_poly_divrem_batch_u64 from batch 2, for rows with nonzero
                              // top words and da ≥ db > 2: 0 = the measured rule, 1 = the literal kernel, 2 = Newton iteration
                              // wherever its transforms fit (poly.cu)
};

struct ronk_ctx {
  ~ronk_ctx();  // api.cu: what is not a DevBuf (events, the pipeline's streams, the scratch blocks, h_flag)
  int device = 0;
  ronk_tune tune;
  std::unordered_set<const void*> smem_attr_done;  // kernels whose >48 KiB dynamic-smem attribute is set on `device`
  cudaStream_t stream = nullptr;
  int sm_count = 132;
  std::string err;
  uint64_t launches = 0;
  bool prof = false;
  std::vector<ronk::ProfRec> prof_log;
  std::map<std::tuple<uint64_t, uint64_t, uint32_t>, ronk::NttPlan> plans;
  std::map<std::tuple<uint64_t, uint64_t, uint64_t>, ronk::DevBuf<uint64_t>> anyntt_spec;  // (p, g, n) → Bluestein spectrum, N words (ntt_any.cu)
  ronk::Scratch scratch;  // every per-call device buffer: transform workspaces, operands, staged _host arguments
  // two-slot host pipeline (ronk_ntt_u64_host_submit / _wait)
  cudaStream_t copy_in = nullptr, copy_out = nullptr;
  static constexpr int kSlots = 3;
  ronk::DevBuf<uint64_t> slot_buf[kSlots];
  size_t slot_bytes[kSlots] = {};
  cudaEvent_t ev_h2d[kSlots] = {}, ev_compute[kSlots] = {}, ev_d2h[kSlots] = {};
  bool slot_pending[kSlots] = {};
  int cluster16_state = 0;   // ntt16c_kernel: 0 = not probed, 1 = usable, -1 = the device refuses 16-CTA clusters of its footprint
  void* dist = nullptr;      // ronk::DistState (dist.cu): communicator, peer mappings, staging — null until ronk_dist_init
  ronk::DevBuf<uint16_t> msm_ytab;  // [20402]: y of the curve point in each histogram bin (msm.cu), built on first use
  ronk::DevBuf<uint32_t> msm_done;  // completion counter of msm_hist_finish_kernel + global histogram, built with msm_ytab
  ronk::DevBuf<uint32_t> msm_coord; // msm_coord_kernel: bintab[20404] | pttab[10404] | counter, Σa, Σb (msm.cu), built on first use
  ronk::DevBuf<uint8_t> pairing_tab;  // T[289²] of the Tate pairing on E[17], padded | μ17 list (pairing.cu), built on first use
  ronk::DevBuf<int> d_flag;  // device error flag
  int* h_flag = nullptr;  // pinned host mirror: h_flag[0] = error flag, h_flag[1..31] = small results (msm.cu)
};

namespace ronk {

inline int set_err(ronk_ctx* ctx, int code, const std::string& msg) {
  if (ctx) ctx->err = msg;
  return code;
}

#define RONK_CUDA(ctx, expr)                                                                  \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess)                                                                    \
      return ronk::set_err(ctx, _e == cudaErrorMemoryAllocation ? RONK_ENOMEM : RONK_ECUDA,   \
                           std::string(#expr ": ") + cudaGetErrorString(_e));                 \
  } while (0)

#define RONK_TRY(expr)          \
  do {                          \
    int _rc = (expr);           \
    if (_rc != RONK_OK) return _rc; \
  } while (0)

template <class T>
int DevBuf<T>::alloc(ronk_ctx* ctx, size_t count) {
  reset();
  T* p = nullptr;
  RONK_CUDA(ctx, cudaMalloc((void**)&p, count * sizeof(T)));
  p_ = p;
  return RONK_OK;
}

// Tables a context or plan keeps once built on first use: build() allocates them into the caller's local DevBufs and
// fills them on ctx->stream; the caller moves them into the context or plan only after build_tables returned RONK_OK.
// On failure ctx->stream is synchronised, since queued work may still touch the locals, which then free themselves.
template <class Build>
inline int build_tables(ronk_ctx* ctx, Build&& build) {
  const int rc = build();
  if (rc != RONK_OK) cudaStreamSynchronize(ctx->stream);
  return rc;
}
// The same for one table of count T: fill(ptr) fills it, and *slot takes it once filled.  optional: a table its user can
// do without; where its allocation fails, CUDA's error is cleared, *slot stays empty (the next call tries again) and the
// result is RONK_OK.
template <class T, class Fill>
inline int build_table(ronk_ctx* ctx, DevBuf<T>* slot, size_t count, Fill&& fill, bool optional = false) {
  DevBuf<T> tab;
  const int rc = tab.alloc(optional ? nullptr : ctx, count);
  if (rc != RONK_OK) {
    if (!optional) return rc;
    cudaGetLastError();
    return RONK_OK;
  }
  RONK_TRY(build_tables(ctx, [&] { return fill(tab.get()); }));
  *slot = std::move(tab);
  return RONK_OK;
}

// Binds the calling thread to the context's device for the duration of one C-ABI call and restores the
// caller's device on exit (contexts for several GPUs may coexist in one process; the caller — torch, a
// Rust host — keeps its own current device).  Every extern "C" entry point that takes a ctx opens with it,
// so allocations, attribute calls and launches inside the call all land on ctx->device.
struct DeviceGuard {
  int prev = -1;
  bool switched = false;
  explicit DeviceGuard(const ronk_ctx* ctx) {
    if (!ctx) return;
    if (cudaGetDevice(&prev) == cudaSuccess && prev != ctx->device) switched = cudaSetDevice(ctx->device) == cudaSuccess;
  }
  ~DeviceGuard() {
    if (switched) cudaSetDevice(prev);
  }
  DeviceGuard(const DeviceGuard&) = delete;
  DeviceGuard& operator=(const DeviceGuard&) = delete;
};

// Opt a kernel into > 48 KiB of dynamic shared memory, once per (context, kernel).
template <class K>
inline int ensure_smem_attr(ronk_ctx* ctx, K kernel, int bytes);

// Brackets a kernel launch with the launch counter and (optionally) profiling events.
struct LaunchScope {
  ronk_ctx* ctx;
  bool on;
  cudaEvent_t start = nullptr, stop = nullptr;
  const char* name;
  LaunchScope(ronk_ctx* c, const char* n) : ctx(c), on(c->prof), name(n) {
    ctx->launches++;  // the device is already bound by the entry point's DeviceGuard
    if (on) {
      cudaEventCreate(&start);
      cudaEventCreate(&stop);
      cudaEventRecord(start, ctx->stream);
    }
  }
  ~LaunchScope() {
    if (on) {
      cudaEventRecord(stop, ctx->stream);
      ProfRec r;
      std::memset(&r, 0, sizeof(r));
      std::snprintf(r.name, sizeof(r.name), "%s", name);
      r.start = start;
      r.stop = stop;
      ctx->prof_log.push_back(r);
    }
  }
};

template <class K>
inline int ensure_smem_attr(ronk_ctx* ctx, K kernel, int bytes) {
  const void* key = reinterpret_cast<const void*>(kernel);
  if (ctx->smem_attr_done.count(key)) return RONK_OK;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) return set_err(ctx, RONK_ECUDA, std::string("cudaFuncSetAttribute: ") + cudaGetErrorString(e));
  ctx->smem_attr_done.insert(key);
  return RONK_OK;
}

inline int check_launch(ronk_ctx* ctx, const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_err(ctx, RONK_ECUDA, std::string(what) + ": " + cudaGetErrorString(e));
  return RONK_OK;
}

// One kernel launch on the context's stream, counted and (when profiling) timed under `name`.  pdl: launch with
// programmatic dependent launch, so the kernel may start before its predecessor on the stream has finished (it waits
// at griddepcontrol.wait).  Not while profiling: the timing events between the kernels would defeat it.
template <class... KArgs, class... Args>
inline int launch(ronk_ctx* ctx, const char* name, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, bool pdl,
                  Args&&... args) {
  {
    LaunchScope ls(ctx, name);
    if (pdl && !ctx->prof) {
      cudaLaunchConfig_t cfg = {};
      cfg.gridDim = grid;
      cfg.blockDim = block;
      cfg.dynamicSmemBytes = smem;
      cfg.stream = ctx->stream;
      cudaLaunchAttribute attr[1];
      attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
      attr[0].val.programmaticStreamSerializationAllowed = 1;
      cfg.attrs = attr;
      cfg.numAttrs = 1;
      RONK_CUDA(ctx, cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...));
    } else {
      kernel<<<grid, block, smem, ctx->stream>>>(std::forward<Args>(args)...);
    }
  }
  return check_launch(ctx, name);
}

// Grid of a grid-stride kernel over n items: one per thread, at most per_sm CTAs per SM, at least one CTA.
inline int grid_for(const ronk_ctx* ctx, size_t n, size_t threads, size_t per_sm = 8) {
  size_t blocks = (n + threads - 1) / threads;
  const size_t cap = (size_t)ctx->sm_count * per_sm;
  if (blocks > cap) blocks = cap;
  if (blocks == 0) blocks = 1;
  return (int)blocks;
}

// A scope's share of the context's scratch stack: `Frame f(ctx); u64* X; RONK_TRY(f.take(&X, words));`.  Each take
// hands out a region above everything taken so far; the destructor gives back all the frame took.  A function takes
// what it needs and never has to know what its callees take.  The rules:
//  1. LIFO, no movement: a region is never moved or freed while its frame is alive, and never escapes its scope.
//  2. Every region starts on a 256-byte boundary, as a CUDA allocation does (msm_coord_kernel's vector path needs
//     16-byte aligned points), and spans at least 256 bytes, so that an empty request is still a valid pointer.
//  3. A request that does not fit the rest of the current block goes to the next block.  Where there is none, it
//     allocates one of its size.  Where the next block is too small, it frees that block and every one above it (no
//     live frame has a region there) and allocates one of its size.  Blocks come and go in stream order
//     (cudaMallocAsync / cudaFreeAsync on ctx->stream, from the device's default memory pool), so growing never makes
//     the host wait: cudaFree would wait for the device, and a small block left by one call (div_linear's chunk
//     sums) is outgrown by the next (dft's roots table) on a context fresh enough that its caller expects no wait.
//     The pool is shared by the process: a growth may reuse memory another stream freed and so order ctx->stream
//     behind that stream's work, as the device-wide wait of cudaFree did.
//  4. Blocks only grow, so a call whose requests fit the blocks held does no allocation, no free and no synchronise;
//     the blocks are freed in ronk_ctx_destroy.
//  5. A failed allocation is RONK_ENOMEM with ctx->err set (RONK_ECUDA where the device has no memory pools); CUDA's
//     sticky error is cleared.  The blocks a growth frees stay reserved until the stream reaches the free, so a
//     growth that runs out of memory synchronises ctx->stream, returns the pool's unused memory and tries once more:
//     near capacity it needs no more than the new block, as a synchronous free-then-allocate did.
//  6. A region given back may be handed to the very next kernel on ctx->stream while an earlier kernel that used it
//     is still queued: stream order makes that safe.  It holds because only the second and later kernels of one
//     transform or one commit are launched with programmatic dependent launch; a kernel that starts before its
//     predecessor ends must never be the first user of a region another call or scope gave back.
//  7. Nothing survives a call: every function writes its scratch before it reads it.
class Frame {
 public:
  ronk_ctx* const ctx;
  explicit Frame(ronk_ctx* c) : ctx(c), used_(c->scratch.used), top_(c->scratch.top) {}
  ~Frame() {
    ctx->scratch.used = used_;
    ctx->scratch.top = top_;
  }
  Frame(const Frame&) = delete;
  Frame& operator=(const Frame&) = delete;

  static constexpr size_t kAlign = 256;
  static size_t span(size_t bytes) { return bytes ? (bytes + kAlign - 1) / kAlign * kAlign : kAlign; }

  // *out = a region of `count` elements of T
  template <class T>
  int take(T** out, size_t count) {
    Scratch& s = ctx->scratch;
    const size_t bytes = span(count * sizeof(T));
    if (s.used == 0 || s.blocks[s.used - 1].bytes - s.top < bytes) {
      if (s.used < s.blocks.size() && s.blocks[s.used].bytes < bytes) {
        for (size_t i = s.used; i < s.blocks.size(); i++) cudaFreeAsync(s.blocks[i].base, ctx->stream);
        s.blocks.resize(s.used);
      }
      if (s.used == s.blocks.size()) {
        void* p = nullptr;
        cudaError_t e = cudaMallocAsync(&p, bytes, ctx->stream);
        if (e == cudaErrorMemoryAllocation) {
          cudaGetLastError();
          cudaMemPool_t pool;
          cudaStreamSynchronize(ctx->stream);
          if (cudaDeviceGetDefaultMemPool(&pool, ctx->device) == cudaSuccess) cudaMemPoolTrimTo(pool, 0);
          e = cudaMallocAsync(&p, bytes, ctx->stream);
        }
        if (e != cudaSuccess) {
          cudaGetLastError();
          return set_err(ctx, e == cudaErrorMemoryAllocation ? RONK_ENOMEM : RONK_ECUDA,
                         std::string("workspace allocation failed: ") + cudaGetErrorString(e));
        }
        s.blocks.push_back({(char*)p, bytes});
      }
      s.used++;
      s.top = 0;
    }
    *out = (T*)(s.blocks[s.used - 1].base + s.top);
    s.top += bytes;
    return RONK_OK;
  }

 private:
  const size_t used_, top_;
};

// The device error flag that kernels raise with atomicExch: cleared before a launch, read back (synchronising the
// stream) after it.
inline int reset_flag(ronk_ctx* ctx) {
  RONK_CUDA(ctx, cudaMemsetAsync(ctx->d_flag.get(), 0, sizeof(int), ctx->stream));
  return RONK_OK;
}
inline int read_flag(ronk_ctx* ctx, int* v) {
  RONK_CUDA(ctx, cudaMemcpyAsync(ctx->h_flag, ctx->d_flag.get(), sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  *v = *ctx->h_flag;
  return RONK_OK;
}

// The mapped pinned error flag, cleared: its device address for a kernel that raises it with a plain store.  The
// caller synchronises ctx->stream before it reads h_flag[0] (pairing.cu, sha256.cu).
inline int clear_flag(ronk_ctx* ctx, volatile u32** dev) {
  ((volatile u32*)ctx->h_flag)[0] = 0u;
  u32* d = nullptr;
  RONK_CUDA(ctx, cudaHostGetDevicePointer((void**)&d, (void*)ctx->h_flag, 0));
  *dev = d;
  return RONK_OK;
}

// One region of a _host call's arguments: `bytes` uploaded from `in` before the call when `in` is set, downloaded to
// `out` after a successful call when `out` is set, scratch when neither is.
struct Staged {
  size_t bytes;
  const void* in = nullptr;
  void* out = nullptr;
  u64* dev = nullptr;  // set by stage_in
};

// Carves the regions from one take of the _host entry point's frame, the outermost of the call, so that the scratch
// grows at most once for all of them, and enqueues the uploads on ctx->stream.  The frame must outlive stage_out.
template <size_t N>
inline int stage_in(Frame& f, Staged (&r)[N]) {
  size_t total = 0;
  for (const Staged& s : r) total += Frame::span(s.bytes);
  char* at = nullptr;
  RONK_TRY(f.take(&at, total));
  for (Staged& s : r) {
    s.dev = (u64*)at;
    at += Frame::span(s.bytes);
    if (s.in && s.bytes) RONK_CUDA(f.ctx, cudaMemcpyAsync(s.dev, s.in, s.bytes, cudaMemcpyHostToDevice, f.ctx->stream));
  }
  return RONK_OK;
}

// Ends a staged call whose device work returned rc: on RONK_OK copies the outputs back and synchronises; otherwise
// returns rc and leaves the host outputs unwritten.
template <size_t N>
inline int stage_out(ronk_ctx* ctx, int rc, const Staged (&r)[N]) {
  if (rc != RONK_OK) return rc;
  for (const Staged& s : r)
    if (s.out && s.bytes) RONK_CUDA(ctx, cudaMemcpyAsync(s.out, s.dev, s.bytes, cudaMemcpyDeviceToHost, ctx->stream));
  RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return RONK_OK;
}

// Whether the nx bytes at x and the ny bytes at y share a byte (never for a null or empty region).
inline bool bytes_overlap(const void* x, size_t nx, const void* y, size_t ny) {
  if (!x || !y || !nx || !ny) return false;
  const uintptr_t a = (uintptr_t)x, b = (uintptr_t)y;
  return a < b + ny && b < a + nx;
}

// ctx->msm_coord's group tables (msm.cu), built on the first call that needs them.
int msm_coord_tables(ronk_ctx* ctx);

// Whether the nx words at x and the ny words at y share a word.
inline bool overlaps(const u64* x, size_t nx, const u64* y, size_t ny) { return nx && ny && x < y + ny && y < x + nx; }

// ⌈log2 v⌉, capped at 63 (v ≤ 1 gives 0).
inline u32 log2_ceil(u64 v) {
  u32 k = 0;
  while (k < 63 && ((u64)1 << k) < v) k++;
  return k;
}

// Whether the power-of-two transforms take 2^log_n points over p: log_n ≤ 26 and 2^log_n divides p - 1.
inline bool pow2_fits(u64 p, u32 log_n) { return log_n <= 26 && (p - 1) % ((u64)1 << log_n) == 0; }

// Whether w, given w^n = 1 mod p, has order exactly n: w^(n/q) != 1 for every prime q dividing n.  Trial division, so
// under 2^16 steps for n ≤ 2^32.  Where it fails, two of the points ω^i, i < n, coincide (Reed–Solomon positions,
// barycentric nodes) and the reference divides by zero.
inline bool root_has_order(u64 w, u64 n, u64 p) {
  u64 r = n;
  for (u64 q = 2; r > 1; q++) {
    if (q * q > r) q = r;
    if (r % q) continue;
    if (h_powmod(w, n / q, p) == 1) return false;
    while (r % q == 0) r /= q;
  }
  return true;
}

int make_mont_field(ronk_ctx* ctx, u64 p, u64 g, bool inverse, MontField* out);  // ntt.cu
int validate_modulus(ronk_ctx* ctx, u64 p);                                       // field_ops.cu

// Runs fn(f) with the field policy of (p, g) and returns its result.  g is the generator whose roots of unity the call
// takes from the policy, or 0 when it takes none.  The Goldilocks policy hard-codes ω_16 = 2^156, a power of g = 7, so it
// serves Goldilocks with g = 7 or 0; every other (p, g) runs on a Montgomery policy built for it.
template <class Fn>
inline int with_field(ronk_ctx* ctx, u64 p, u64 g, bool inverse, Fn&& fn) {
  if (p == GL_P && (g == 0 || g == 7)) {
    GoldilocksField f;
    return fn(f);
  }
  MontField f;
  RONK_TRY(make_mont_field(ctx, p, g, inverse, &f));
  return fn(f);
}

// Internal device-pointer entry points used across translation units.
int ntt_device(ronk_ctx* ctx, u64 p, u64 g, u64* data, const u64* mul, u32 log_n, u32 batch, int inverse);
// ntt.cu: batch in-place coset transforms on s·H_n, s != 1, log_n >= 1 (arguments checked by ntt_coset.cu): one launch
// builds the factor tables in this call's scratch, then the transform runs with s^±j fused into its first or last pass.
int ntt_device_coset(ronk_ctx* ctx, u64 p, u64 g, u64* data, u32 log_n, u32 batch, u64 shift, int inverse);
// ntt.cu: the words of workspace a transform of batch × 2^log_n takes from the scratch on the single-tile and two-pass
// kernels (and on the 256-point-tile passes that coset transforms take)
size_t ntt_workspace_words(u32 log_n, u32 batch);
int ntt_device_shared_mul(ronk_ctx* ctx, u64 p, u64 g, const u64* src, u64* dst, const u64* mul, u32 log_n, u32 batch);
int ntt_device_bounded(ronk_ctx* ctx, u64 p, u64 g, const u64* src, u64 src_len, u64* dst, u64 dst_len, const u64* mul,
                       u32 log_n, int inverse);
// out[0, out_len) = a·b mod x^n - 1, n = 2^log_n, by three bounded transforms: a[0, la) → X, b[0, lb) → Y ⊙ X, the
// inverse of Y → out.  X and Y hold n words each.  a may be X, and out may be a, b or Y: a transform may run in place,
// and a and b are read by the first two transforms only.  Stream-ordered.
int product_bounded(ronk_ctx* ctx, u64 p, u64 g, const u64* a, u64 la, const u64* b, u64 lb, u32 log_n, u64* X, u64* Y,
                    u64* out, u64 out_len);
// poly_div.cu: dst[i] = i < n ? src[last - i] : 0 for i < dst_len (reverses, truncates and zero-fills in one pass), one
// launch profiled as `name`.
int reverse_words(ronk_ctx* ctx, const char* name, const u64* src, size_t last, size_t n, u64* dst, size_t dst_len);
// The single-tile plan of 2^log_n points (log_n ≤ 13): per-round twiddle tables (forward, inverse) and n^-1, twiddle form.
int ntt_single_tables(ronk_ctx* ctx, u64 p, u64 g, u32 log_n, const u64** fwd, const u64** inv, u64* scale_inv);
// poly.cu: nodes[i] = ω_n^i (plain residues), n ≤ 2^31 - 1; out[i] = Σ_j c_j xs[i]^j, one CTA per point
int roots_table(ronk_ctx* ctx, u64 p, u64 g, u64 n, u64* nodes);
int poly_eval_device(ronk_ctx* ctx, u64 p, const u64* c, size_t d, const u64* xs, size_t m, u64* out);
bool divrem_newton_fits(u64 p, u64 g, size_t da, size_t db);  // poly_div.cu
int divrem_newton_device(ronk_ctx* ctx, u64 p, u64 g, const u64* a, size_t da, const u64* b, size_t db, u64 top, u64* q,
                         u64* r);
// poly_div.cu, batches of rows (a, q, r: batch × da; b: batch × db, or db words when b_shared), top words nonzero:
// divrem_newton_rows runs Newton iteration on batched transforms (top = the shared divisor's top word; arguments checked
// by the caller, batch ≥ 2, scratch reserved from divrem_newton_rows_scratch; stream-ordered).
// divrem_newton_rows_transform_words: batch × the plan's larger transform.  divrem_top_inverses: out[2y] = b_y[db-1]^-1,
// out[2y + 1] = -b_y[0]·out[2y], one launch profiled as divrem_top_inv.
int divrem_newton_rows(ronk_ctx* ctx, u64 p, u64 g, const u64* a, size_t da, const u64* b, size_t db, bool b_shared, u32 batch,
                       u64 top, u64* q, u64* r);
size_t divrem_newton_rows_scratch(size_t da, size_t db, bool b_shared, u32 batch);
u64 divrem_newton_rows_transform_words(size_t da, size_t db, u32 batch);
int divrem_top_inverses(ronk_ctx* ctx, u64 p, const u64* b, size_t db, u32 batch, u64* out);
// G = hr^-1 mod x^L (hr: hl ≤ L words, g1 = hr[0]^-1); X, Y: 2^⌈log2(2L - 1)⌉ words each.  Stream-ordered.
int newton_inverse_device(ronk_ctx* ctx, u64 p, u64 g, const u64* hr, size_t hl, size_t L, u64 g1, u64* G, u64* X, u64* Y);
// Subproduct tree (poly_tree.cu) over k ≤ kTreeMaxLeaves points.  tree_fits: g != 0 and every transform of the plan
// (tree levels above the shared-memory kernels; with d > 0 the root's division of d words) a power of two dividing
// p - 1 and ≤ 2^26.  Arguments are checked by the caller.  from_roots with k ≤ kTreeLeaves launches no transform.
constexpr size_t kTreeLeaves = 64, kTreeMaxLeaves = (size_t)1 << 24;
bool tree_fits(u64 p, u64 g, size_t k, size_t d);
int tree_from_roots(ronk_ctx* ctx, u64 p, u64 g, const u64* xs, size_t k, u64* out);
// multieval and interpolate take `batch` rows over the one point set (c: batch × d, ys and out row-major); batch 1 is the
// single-row launch sequence.  tree_scratch_words: an upper bound on the words either takes from the context's scratch,
// its transforms' workspace included.
int tree_multieval(ronk_ctx* ctx, u64 p, u64 g, const u64* c, size_t d, u32 batch, const u64* xs, size_t m, u64* out);
int tree_interpolate(ronk_ctx* ctx, u64 p, u64 g, const u64* xs, const u64* ys, size_t k, u32 batch, u64* out);
size_t tree_scratch_words(const ronk_ctx* ctx, size_t k, size_t d, u32 batch, bool interp);
// poly_tree.cu: reverse_words over `batch` rows, dst[b·ds + i] = i < n ? src[b·ss + last - i] : 0, i < len, one launch
// profiled as tree_reverse; out[i] = (i + 1)·M[i + 1], i < k, one launch profiled as tree_deriv.
int reverse_rows(ronk_ctx* ctx, const u64* src, size_t ss, size_t last, size_t n, u64* dst, size_t ds, size_t len, u32 batch);
int poly_deriv(ronk_ctx* ctx, u64 p, const u64* M, size_t k, u64* out);
// poly.cu: the path of a non-empty batched multieval / interpolation (*tree) and its size checks, which read no
// pointer: RONK_EUNSUPPORTED past the envelope of ronk_poly_multieval_batch_u64 / ronk_poly_interpolate_batch_u64.
int multieval_path(ronk_ctx* ctx, u64 p, u64 g, size_t d, u32 batch, size_t m, bool* tree);
int interpolate_path(ronk_ctx* ctx, u64 p, u64 g, size_t k, u32 batch, bool* tree);
// grid.y of a kernel whose grid_x CTAs step over `rows` rows by gridDim.y: enough rows of CTAs to give every SM 8 (at
// least one row, at most `rows` and CUDA's 65535), so that each CTA serves several rows of a large batch and forms what
// the rows share once for all of them.
inline u32 grid_rows(const ronk_ctx* ctx, u64 rows, u64 grid_x) {
  const u64 fill = ((u64)ctx->sm_count * 8 + grid_x - 1) / grid_x;
  u64 y = rows < fill ? rows : fill;
  if (y > 65535) y = 65535;
  return y ? (u32)y : 1u;
}
// ntt_any.cu: ronk_ntt_any_u64 on device pointers, and its argument and path check (*path set on RONK_OK).
enum AnyNttPath { AN_POW2, AN_BLUESTEIN, AN_LITERAL, AN_NONE };
int anyntt_args(ronk_ctx* ctx, u64 p, u64 g, const void* data, u64 n, AnyNttPath* path);
int anyntt_device(ronk_ctx* ctx, u64 p, u64 g, u64* data, u64 n, u32 batch, int inverse);
// poly_crt.cu: the multi-modular product.  crt_mul_fits: g != 0, L = da + db - 1 ≤ kCrtMulMaxLen, no power of two ≥ L
// divides p - 1, and da·db and min(da, db) reach the crossovers.  crt_mul_device: c = a·b (L words) on device pointers, stream-ordered;
// arguments are checked by the caller.
constexpr size_t kCrtMulMaxLen = (size_t)1 << 26;
bool crt_mul_fits(const ronk_ctx* ctx, u64 p, u64 g, size_t da, size_t db);
int crt_mul_device(ronk_ctx* ctx, u64 p, const u64* a, size_t da, const u64* b, size_t db, u64* c);
// Batched products (poly_batch.cu): `batch` contiguous rows c[r] = a[r]·b[b_shared ? 0 : r], L = da + db - 1 words each.
// poly_mul_rows_pow2: on the fused kernel or the batched transforms over q, where a power of two N ≥ L divides q - 1
// (N ≤ 2^26, batch·N within poly_batch.cu's envelope).  crt_mul_rows_device (poly_crt.cu): the multi-modular path over
// the same rows.  *scratch_words: the words either takes from the context's scratch, its transforms' workspace included.
// Arguments are checked by the caller; stream-ordered; c is written by the last launch only.
int poly_mul_rows_pow2(ronk_ctx* ctx, u64 q, u64 g, const u64* a, size_t da, const u64* b, size_t db, bool b_shared,
                       u32 batch, u64* c);
size_t poly_mul_rows_pow2_scratch(const ronk_ctx* ctx, size_t da, size_t db, bool b_shared, u32 batch);
int crt_mul_rows_device(ronk_ctx* ctx, u64 p, const u64* a, size_t da, const u64* b, size_t db, bool b_shared, u32 batch,
                        u64* c);
size_t crt_mul_rows_scratch(const ronk_ctx* ctx, u64 p, size_t da, size_t db, bool b_shared, u32 batch);
// poly_batch.cu: dst[r·N + k] = k < d ? src[r·stride + k] : 0 (N = 2^log_n) over total = rows·N words, a grid-stride
// loop of PAD_THREADS-thread CTAs.  Zero-pads the rows of the batched product and of the LDE (ntt_coset.cu).
constexpr int PAD_THREADS = 256;
__global__ void __launch_bounds__(PAD_THREADS)
poly_rows_pad_kernel(const u64* __restrict__ src, u32 d, u64 stride, u32 log_n, u64 total, u64* __restrict__ dst);
// poly.cu: the schoolbook kernel over `batch` contiguous rows (b_stride = db, or 0 for one shared b).
int poly_mul_schoolbook_rows(ronk_ctx* ctx, u64 p, const u64* a, size_t da, const u64* b, size_t db, size_t b_stride,
                             u64 batch, u64* c);

}  // namespace ronk
