// dist.cu — the multi-GPU modes of the hot path behind the C ABI (SURVEY §8b/§8e), one process (or host thread)
// per GPU, NCCL over NVLink 5 / NVSwitch for the plumbing:
//
//   ronk_dist_unique_id / ronk_dist_init / ronk_dist_init_comm / ronk_dist_finalize
//       bootstrap: an ncclUniqueId made on rank 0 and carried to the other ranks by the host (MPI, a TCP store,
//       torch.distributed …), or an ncclComm_t the host already owns.  libnccl.so.2 is resolved with dlopen at
//       the first call, so the library loads (and every single-GPU entry point works) on a box without NCCL;
//       the dist entry points then return RONK_ENCCL.
//   ronk_ntt_u64_batch_sharded      independent transforms, contiguous batch ranges per rank, NO collective.
//   ronk_ntt_u64_dist               `batch` transforms of 2^log_n points each spread cyclically over the G ranks
//       (rank r holds a[r::G] of every transform).  Local 2^log_n / G-point transforms with the twiddle column
//       ω_n^(r·k') applied in their store phase, ONE exchange, then G-point butterflies across ranks — the top
//       log2 G stages of the transform.  ω_G is a power of two for G ≤ 16 (ω_16 = 2^156), so those butterflies
//       are shift networks: no general multiplication (round 1 spent O(G²) of them per output).
//       flavour RONK_DIST_NCCL : pack → grouped ncclSend/ncclRecv (all-to-all) → cross_rank_kernel on the
//                                received blocks;
//       flavour RONK_DIST_FUSED: every rank's local result sits in a buffer exported with CUDA IPC (handles
//                                exchanged through the communicator); after a stream-ordered barrier (a 4-byte
//                                ncclAllReduce) cross_rank_kernel reads the peers' blocks directly over NVLink
//                                (ld.global on peer-mapped addresses) — exchange and butterflies in ONE kernel,
//                                no staging buffer, no packing.
//   ronk_msm_pluto_ext_dist         kzg::commit over index-range shards: local commit (msm.cu), ncclAllGather of
//       the G partial points (4 bytes each), local sum with the reference's addition law.
//
// Output layout of ronk_ntt_u64_dist on rank s (m = n/G, blk = m/G): out[b][q][k''] = X_b[s·blk + k'' + m·q].
#include <dlfcn.h>
#include <nccl.h>
#include <unistd.h>

#include "msm_curve.cuh"
#include "ntt_kernel.cuh"
#include "ronk_internal.h"

namespace ronk {

// ---- NCCL through dlopen ---------------------------------------------------------------------------------
struct NcclApi {
  void* handle = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*CommCount)(const ncclComm_t, int*) = nullptr;
  ncclResult_t (*CommUserRank)(const ncclComm_t, int*) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  bool ok = false;
};

static NcclApi& nccl_api() {
  static NcclApi api;
  static bool tried = false;
  if (tried) return api;
  tried = true;
  // a host that already carries NCCL (torch bundles its own libnccl.so.2) gets that copy: same SONAME
  for (const char* name : {"libnccl.so.2", "libnccl.so"}) {
    api.handle = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
    if (api.handle) break;
  }
  if (!api.handle) return api;
  bool all = true;
  auto sym = [&](const char* n) {
    void* p = dlsym(api.handle, n);
    if (!p) all = false;
    return p;
  };
  api.GetUniqueId = (decltype(api.GetUniqueId))sym("ncclGetUniqueId");
  api.CommInitRank = (decltype(api.CommInitRank))sym("ncclCommInitRank");
  api.CommDestroy = (decltype(api.CommDestroy))sym("ncclCommDestroy");
  api.CommCount = (decltype(api.CommCount))sym("ncclCommCount");
  api.CommUserRank = (decltype(api.CommUserRank))sym("ncclCommUserRank");
  api.AllGather = (decltype(api.AllGather))sym("ncclAllGather");
  api.AllReduce = (decltype(api.AllReduce))sym("ncclAllReduce");
  api.Send = (decltype(api.Send))sym("ncclSend");
  api.Recv = (decltype(api.Recv))sym("ncclRecv");
  api.GroupStart = (decltype(api.GroupStart))sym("ncclGroupStart");
  api.GroupEnd = (decltype(api.GroupEnd))sym("ncclGroupEnd");
  api.GetErrorString = (decltype(api.GetErrorString))sym("ncclGetErrorString");
  api.ok = all;
  return api;
}

#define RONK_NCCL(ctx, expr)                                                                         \
  do {                                                                                               \
    ncclResult_t _r = (expr);                                                                        \
    if (_r != ncclSuccess)                                                                           \
      return ronk::set_err(ctx, RONK_ENCCL, std::string(#expr ": ") + nccl_api().GetErrorString(_r)); \
  } while (0)

// ---- per-context distributed state -------------------------------------------------------------------------
struct PeerBuf {            // what every rank publishes about its exchange buffer
  cudaIpcMemHandle_t handle;
  unsigned long long ptr;   // raw device pointer (valid for ranks living in the same process)
  long long pid;
  int device;
  int pad;
};

struct DistState {
  ncclComm_t comm = nullptr;
  bool owns_comm = false;
  int rank = 0, world = 1;
  u32 log_g = 0;
  // exchange buffer of the fused flavour (IPC-exported) and its peers' mappings
  u64* xbuf = nullptr;
  size_t xbuf_words = 0;
  u64* peer_ptr[16] = {};
  bool peer_opened[16] = {};
  // staging of the NCCL flavour
  DevBuf<u64> pack, recv;
  size_t stage_words = 0;
  DevBuf<int> barrier_word;      // 4 bytes for the stream-ordered barrier
  DevBuf<u32> gather;            // G words for the commit all-gather (+1 for the local word)
  std::map<std::tuple<u64, u64, u32>, DevBuf<u64>> twcol;  // (p, g, log_n) → ω_n^(rank·k'), k' < n/G
};

struct PeerPtrs {
  const u64* p[16];
};

// x[r] = src.p[r][b·bstride + off + k], r < G;  G-point DIF shift network;  out[b·ostride + q·blk + k] = X[q].
// The network leaves X[bitrev(j)] in x[j], so the store un-reverses.  One thread per (b, k).
template <class F, int LG>
__global__ void __launch_bounds__(256) cross_rank_kernel(const F f, const PeerPtrs src, u64* __restrict__ out, size_t blk,
                                                         u32 batch, size_t bstride, size_t off, size_t ostride) {
  constexpr int G = 1 << LG;
  const size_t total = (size_t)batch * blk;
  const size_t step = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += step) {
    const size_t b = i / blk, k = i - b * blk;
    u64 x[16];
#pragma unroll
    for (int r = 0; r < G; r++) x[r] = src.p[r][b * bstride + off + k];  // all G (peer) loads in flight together
    radix_network<LG, false>(f, x);
    u64* o = out + b * ostride + k;
#pragma unroll
    for (int j = 0; j < G; j++) {
      int q = 0;
#pragma unroll
      for (int t = 0; t < LG; t++) q |= ((j >> t) & 1) << (LG - 1 - t);
      o[(size_t)q * blk] = x[j];
    }
  }
}

// pack[s][b][k] = z[b][s·blk + k]   (the per-destination blocks of a batched local result, made contiguous)
__global__ void pack_blocks_kernel(const u64* __restrict__ z, u64* __restrict__ pack, size_t blk, u32 log_g, u32 batch) {
  const size_t m = blk << log_g, total = (size_t)batch * m;
  const size_t step = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += step) {
    const size_t b = i / m, rem = i - b * m, s = rem / blk, k = rem - s * blk;
    pack[(s * batch + b) * blk + k] = z[i];
  }
}

// one thread: sum of G packed points with the reference's addition law (curve/mod.rs:178-213)
__global__ void point_sum_kernel(const u32* __restrict__ pts, u32 count, volatile u32* host_result) {
  if (threadIdx.x || blockIdx.x) return;
  u32 acc = PT_INF;
  for (u32 i = 0; i < count; i++) acc = pt_add_w(acc, pts[i]);
  host_result[0] = acc;
}

static DistState* dist_of(ronk_ctx* ctx) { return reinterpret_cast<DistState*>(ctx->dist); }

static int dist_check(ronk_ctx* ctx, DistState** out) {
  if (!ctx) return RONK_EINVAL;
  DistState* d = dist_of(ctx);
  if (!d || !d->comm) return set_err(ctx, RONK_ENCCL, "ronk_dist_init has not been called on this context");
  *out = d;
  return RONK_OK;
}

// stream-ordered barrier across the ranks: a 4-byte all-reduce on the context's stream
static int dist_barrier(ronk_ctx* ctx, DistState* d) {
  RONK_NCCL(ctx, nccl_api().AllReduce(d->barrier_word.get(), d->barrier_word.get(), 1, ncclInt32, ncclSum, d->comm, ctx->stream));
  return RONK_OK;
}

static int dist_setup_common(ronk_ctx* ctx, DistState* d) {
  if (d->world < 1 || d->world > 16 || (d->world & (d->world - 1)))
    return set_err(ctx, RONK_EUNSUPPORTED, "world size must be a power of two ≤ 16");
  d->log_g = 0;
  while ((1 << d->log_g) < d->world) d->log_g++;
  RONK_TRY(d->barrier_word.alloc(ctx, 1));
  RONK_CUDA(ctx, cudaMemsetAsync(d->barrier_word.get(), 0, sizeof(int), ctx->stream));
  RONK_TRY(d->gather.alloc(ctx, 17));
  return RONK_OK;
}

static void dist_release_xbuf(DistState* d) {
  for (int r = 0; r < d->world; r++) {
    if (d->peer_opened[r] && d->peer_ptr[r]) cudaIpcCloseMemHandle(d->peer_ptr[r]);
    d->peer_ptr[r] = nullptr;
    d->peer_opened[r] = false;
  }
  if (d->xbuf) cudaFree(d->xbuf);
  d->xbuf = nullptr;
  d->xbuf_words = 0;
}

// (Re)allocate the IPC-exported exchange buffer and map every peer's: handles travel through the communicator.
static int dist_ensure_xbuf(ronk_ctx* ctx, DistState* d, size_t words) {
  if (d->xbuf_words >= words) return RONK_OK;
  RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  RONK_TRY(dist_barrier(ctx, d));  // nobody is still reading the old mapping
  RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  dist_release_xbuf(d);
  RONK_CUDA(ctx, cudaMalloc((void**)&d->xbuf, words * sizeof(u64)));
  d->xbuf_words = words;
  PeerBuf mine;
  std::memset(&mine, 0, sizeof(mine));
  RONK_CUDA(ctx, cudaIpcGetMemHandle(&mine.handle, d->xbuf));
  mine.ptr = (unsigned long long)(uintptr_t)d->xbuf;
  mine.pid = (long long)getpid();
  mine.device = ctx->device;
  DevBuf<PeerBuf> d_all;
  RONK_TRY(d_all.alloc(ctx, (size_t)d->world + 1));
  RONK_CUDA(ctx, cudaMemcpyAsync(d_all.get() + d->world, &mine, sizeof(mine), cudaMemcpyHostToDevice, ctx->stream));
  RONK_NCCL(ctx, nccl_api().AllGather(d_all.get() + d->world, d_all.get(), sizeof(PeerBuf), ncclUint8, d->comm, ctx->stream));
  std::vector<PeerBuf> all((size_t)d->world);
  RONK_CUDA(ctx, cudaMemcpyAsync(all.data(), d_all.get(), sizeof(PeerBuf) * (size_t)d->world, cudaMemcpyDeviceToHost,
                                 ctx->stream));
  RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  d_all.reset();
  for (int r = 0; r < d->world; r++) {
    if (r == d->rank) { d->peer_ptr[r] = d->xbuf; continue; }
    if (all[(size_t)r].pid == mine.pid) {
      // same process (one host thread per GPU): IPC handles cannot be opened where they were made — use the raw
      // pointer with peer access enabled
      int can = 0;
      cudaDeviceCanAccessPeer(&can, ctx->device, all[(size_t)r].device);
      if (!can) return set_err(ctx, RONK_EUNSUPPORTED, "no peer access between the devices of this process");
      cudaError_t e = cudaDeviceEnablePeerAccess(all[(size_t)r].device, 0);
      if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) RONK_CUDA(ctx, e);
      cudaGetLastError();
      d->peer_ptr[r] = (u64*)(uintptr_t)all[(size_t)r].ptr;
    } else {
      void* p = nullptr;
      RONK_CUDA(ctx, cudaIpcOpenMemHandle(&p, all[(size_t)r].handle, cudaIpcMemLazyEnablePeerAccess));
      d->peer_ptr[r] = (u64*)p;
      d->peer_opened[r] = true;
    }
  }
  return RONK_OK;
}

static int dist_ensure_stage(ronk_ctx* ctx, DistState* d, size_t words) {
  if (d->stage_words >= words) return RONK_OK;
  RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  d->pack.reset();
  d->recv.reset();
  d->stage_words = 0;
  RONK_TRY(d->pack.alloc(ctx, words));
  RONK_TRY(d->recv.alloc(ctx, words));
  d->stage_words = words;
  return RONK_OK;
}

// twiddle column ω_n^(rank·k'), k' < m, in the multiplier form f.mul expects (plain residues)
static int dist_twcol(ronk_ctx* ctx, DistState* d, u64 p, u64 g, u32 log_n, const u64** out) {
  DevBuf<u64>& tab = d->twcol[std::make_tuple(p, g, log_n)];  // empty until built
  const size_t m = ((size_t)1 << log_n) >> d->log_g;
  if (!tab) RONK_TRY(build_table(ctx, &tab, m, [&](u64* t) {
    const u64 w = h_powmod(g, (p - 1) >> log_n, p);
    return ronk_field_powers_u64(ctx, p, h_powmod(w, (u64)d->rank, p), 1 % p, t, m);
  }));
  *out = tab.get();
  return RONK_OK;
}

static int cross_rank(ronk_ctx* ctx, u64 p, u64 g, u32 log_g, const PeerPtrs& src, u64* out, size_t blk, u32 batch,
                      size_t bstride, size_t off, size_t ostride) {
  const int blocks = grid_for(ctx, (size_t)batch * blk, 256);
  return with_field(ctx, p, g, false, [&](const auto& f) {
    using F = std::decay_t<decltype(f)>;
    auto kernel = log_g == 1 ? cross_rank_kernel<F, 1> : log_g == 2 ? cross_rank_kernel<F, 2>
                : log_g == 3 ? cross_rank_kernel<F, 3> : cross_rank_kernel<F, 4>;
    return launch(ctx, "ntt_cross_rank", kernel, blocks, 256, 0, false, f, src, out, blk, batch, bstride, off, ostride);
  });
}

}  // namespace ronk

using namespace ronk;

extern "C" {

int ronk_dist_unique_id(uint8_t id[RONK_NCCL_UNIQUE_ID_BYTES]) {
  static_assert(RONK_NCCL_UNIQUE_ID_BYTES == NCCL_UNIQUE_ID_BYTES, "ncclUniqueId size");
  if (!id) return RONK_EINVAL;
  NcclApi& n = nccl_api();
  if (!n.ok) return RONK_ENCCL;
  ncclUniqueId u;
  if (n.GetUniqueId(&u) != ncclSuccess) return RONK_ENCCL;
  std::memcpy(id, &u, NCCL_UNIQUE_ID_BYTES);
  return RONK_OK;
}

static int dist_attach(ronk_ctx* ctx, ncclComm_t comm, bool owns, int rank, int world) {
  if (ctx->dist) return set_err(ctx, RONK_EINVAL, "context already has a communicator (ronk_dist_finalize first)");
  DistState* d = new DistState();
  d->comm = comm;
  d->owns_comm = owns;
  d->rank = rank;
  d->world = world;
  ctx->dist = d;
  const int rc = dist_setup_common(ctx, d);
  if (rc != RONK_OK) ronk_dist_finalize(ctx);
  return rc;
}

int ronk_dist_init(ronk_ctx* ctx, const uint8_t id[RONK_NCCL_UNIQUE_ID_BYTES], int rank, int world) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx || !id) return set_err(ctx, RONK_EINVAL, "null argument");
  if (world < 1 || rank < 0 || rank >= world) return set_err(ctx, RONK_EINVAL, "bad rank / world");
  NcclApi& n = nccl_api();
  if (!n.ok) return set_err(ctx, RONK_ENCCL, "libnccl.so.2 could not be loaded");
  ncclUniqueId u;
  std::memcpy(&u, id, NCCL_UNIQUE_ID_BYTES);
  ncclComm_t comm = nullptr;
  RONK_NCCL(ctx, n.CommInitRank(&comm, world, u, rank));
  return dist_attach(ctx, comm, true, rank, world);
}

int ronk_dist_init_comm(ronk_ctx* ctx, void* nccl_comm, int rank, int world) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx || !nccl_comm) return set_err(ctx, RONK_EINVAL, "null argument");
  NcclApi& n = nccl_api();
  if (!n.ok) return set_err(ctx, RONK_ENCCL, "libnccl.so.2 could not be loaded");
  int cw = 0, cr = -1;
  RONK_NCCL(ctx, n.CommCount((ncclComm_t)nccl_comm, &cw));
  RONK_NCCL(ctx, n.CommUserRank((ncclComm_t)nccl_comm, &cr));
  if (cw != world || cr != rank) return set_err(ctx, RONK_EINVAL, "rank / world do not match the communicator");
  return dist_attach(ctx, (ncclComm_t)nccl_comm, false, rank, world);
}

int ronk_dist_finalize(ronk_ctx* ctx) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx) return RONK_EINVAL;
  DistState* d = dist_of(ctx);
  if (!d) return RONK_OK;
  cudaStreamSynchronize(ctx->stream);
  dist_release_xbuf(d);
  if (d->comm && d->owns_comm && nccl_api().ok) nccl_api().CommDestroy(d->comm);
  delete d;
  ctx->dist = nullptr;
  return RONK_OK;
}

int ronk_dist_rank(ronk_ctx* ctx, int* rank, int* world) {
  DistState* d = nullptr;
  RONK_TRY(dist_check(ctx, &d));
  if (rank) *rank = d->rank;
  if (world) *world = d->world;
  return RONK_OK;
}

int ronk_dist_barrier(ronk_ctx* ctx) {
  ronk::DeviceGuard _dg(ctx);
  DistState* d = nullptr;
  RONK_TRY(dist_check(ctx, &d));
  return dist_barrier(ctx, d);
}

int ronk_dist_shard_range(uint64_t total, int rank, int world, uint64_t* lo, uint64_t* hi) {
  if (!lo || !hi || world < 1 || rank < 0 || rank >= world) return RONK_EINVAL;
  const uint64_t base = total / (uint64_t)world, rem = total % (uint64_t)world;
  const uint64_t r = (uint64_t)rank;
  *lo = r * base + (r < rem ? r : rem);
  *hi = *lo + base + (r < rem ? 1 : 0);
  return RONK_OK;
}

int ronk_ntt_u64_batch_sharded(ronk_ctx* ctx, uint64_t p, uint64_t g, uint64_t* shard, uint32_t log_n,
                               uint64_t total_batch, int inverse, uint64_t* lo_out, uint64_t* hi_out) {
  ronk::DeviceGuard _dg(ctx);
  DistState* d = nullptr;
  RONK_TRY(dist_check(ctx, &d));
  uint64_t lo = 0, hi = 0;
  if (ronk_dist_shard_range(total_batch, d->rank, d->world, &lo, &hi) != RONK_OK) return set_err(ctx, RONK_EINVAL, "bad shard");
  if (lo_out) *lo_out = lo;
  if (hi_out) *hi_out = hi;
  if (hi - lo > 0xFFFFFFFFull) return set_err(ctx, RONK_EUNSUPPORTED, "shard too large");
  return ntt_device(ctx, p, g, (u64*)shard, nullptr, log_n, (u32)(hi - lo), inverse);  // no collective on the data path
}

int ronk_ntt_u64_dist(ronk_ctx* ctx, uint64_t p, uint64_t g, uint64_t* local, uint32_t log_n, uint32_t batch, int flavour) {
  ronk::DeviceGuard _dg(ctx);
  DistState* d = nullptr;
  RONK_TRY(dist_check(ctx, &d));
  if (!local) return set_err(ctx, RONK_EINVAL, "null argument");
  RONK_TRY(validate_modulus(ctx, p));
  if (g == 0 || g >= p) return set_err(ctx, RONK_EINVAL, "generator out of range");
  if (log_n >= 64 || (p - 1) % ((u64)1 << log_n) != 0)
    return set_err(ctx, RONK_EINVAL, "n must divide p - 1 (no primitive n-th root of unity)");
  const u32 lg = d->log_g;
  if (log_n < 2 * lg) return set_err(ctx, RONK_EINVAL, "transform smaller than G² points");
  if (log_n - lg > 26) return set_err(ctx, RONK_EUNSUPPORTED, "local transform larger than 2^26");
  if (flavour != RONK_DIST_NCCL && flavour != RONK_DIST_FUSED) return set_err(ctx, RONK_EINVAL, "unknown flavour");
  if (batch == 0) return RONK_OK;
  if (lg == 0) return ntt_device(ctx, p, g, (u64*)local, nullptr, log_n, batch, 0);
  const u32 log_m = log_n - lg;
  const size_t m = (size_t)1 << log_m, blk = m >> lg, words = (size_t)batch * m;
  const int G = d->world;
  const u64* twcol = nullptr;
  if (d->rank) RONK_TRY(dist_twcol(ctx, d, p, g, log_n, &twcol));  // rank 0's column is all ones
  NcclApi& n = nccl_api();
  PeerPtrs src;
  for (int r = 0; r < 16; r++) src.p[r] = nullptr;
  if (flavour == RONK_DIST_FUSED) {
    RONK_TRY(dist_ensure_xbuf(ctx, d, words));
    // Z_r = NTT_m(a[r::G]) ⊙ ω_n^(r·k'), straight into the exported buffer
    if (log_m == 0) return set_err(ctx, RONK_EINVAL, "transform smaller than G² points");
    RONK_TRY(ntt_device_shared_mul(ctx, p, g, (const u64*)local, d->xbuf, twcol, log_m, batch));
    RONK_TRY(dist_barrier(ctx, d));  // every rank's Z is complete (stream-ordered; the host does not wait)
    for (int r = 0; r < G; r++) src.p[r] = d->peer_ptr[r];
    RONK_TRY(cross_rank(ctx, p, g, lg, src, (u64*)local, blk, batch, m, (size_t)d->rank * blk, m));
    return dist_barrier(ctx, d);     // peers have finished reading before anyone refills its buffer
  }
  RONK_TRY(dist_ensure_stage(ctx, d, words));
  RONK_TRY(ntt_device_shared_mul(ctx, p, g, (const u64*)local, (u64*)local, twcol, log_m, batch));
  const u64* sendbase = (const u64*)local;
  if (batch > 1) {  // the block for destination s is strided over the batch: make it contiguous first
    RONK_TRY(launch(ctx, "dist_pack", pack_blocks_kernel, grid_for(ctx, words, 256, 16), 256, 0, false, (const u64*)local,
                    d->pack.get(), blk, lg, batch));
    sendbase = d->pack.get();
  }
  const size_t chunk = (size_t)batch * blk;  // words per (source, destination) pair
  RONK_NCCL(ctx, n.GroupStart());
  for (int r = 0; r < G; r++) {
    RONK_NCCL(ctx, n.Send(sendbase + (size_t)r * chunk, chunk, ncclUint64, r, d->comm, ctx->stream));
    RONK_NCCL(ctx, n.Recv(d->recv.get() + (size_t)r * chunk, chunk, ncclUint64, r, d->comm, ctx->stream));
  }
  RONK_NCCL(ctx, n.GroupEnd());
  for (int r = 0; r < G; r++) src.p[r] = d->recv.get() + (size_t)r * chunk;
  return cross_rank(ctx, p, g, lg, src, (u64*)local, blk, batch, blk, 0, m);
}

// The same decomposition with G = 2^log_g VIRTUAL ranks on ONE device — no communicator, no IPC: `data` holds the G local
// slices rank-major ([rank][batch][n/G], slice r = a[r::G] of every transform) and receives the G local results in the
// layout ronk_ntt_u64_dist leaves on rank r ([batch][G][n/G²]).  Every kernel and every index formula of both
// exchange flavours runs exactly as in the multi-GPU call (local transforms with the twiddle column in the store phase,
// pack, cross_rank_kernel<log_g>); only the wire is replaced — device-to-device copies for the all-to-all, plain device
// pointers for the peer buffers.  It exists so that G = 4, 8, 16 can be validated on a single GPU
// (tests/test_gpu_ntt.py::test_virtual_rank_distributed_transform) and as a capacity mode for one device.
int ronk_ntt_u64_dist_virtual(ronk_ctx* ctx, uint64_t p, uint64_t g, uint64_t* data, uint32_t log_n, uint32_t batch,
                              uint32_t log_g, int flavour) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx || !data) return set_err(ctx, RONK_EINVAL, "null argument");
  RONK_TRY(validate_modulus(ctx, p));
  if (g == 0 || g >= p) return set_err(ctx, RONK_EINVAL, "generator out of range");
  if (log_n >= 64 || (p - 1) % ((u64)1 << log_n) != 0)
    return set_err(ctx, RONK_EINVAL, "n must divide p - 1 (no primitive n-th root of unity)");
  if (log_g < 1 || log_g > 4) return set_err(ctx, RONK_EINVAL, "2 <= G <= 16");
  if (log_n < 2 * log_g) return set_err(ctx, RONK_EINVAL, "transform smaller than G² points");
  if (log_n - log_g > 26) return set_err(ctx, RONK_EUNSUPPORTED, "local transform larger than 2^26");
  if (flavour != RONK_DIST_NCCL && flavour != RONK_DIST_FUSED) return set_err(ctx, RONK_EINVAL, "unknown flavour");
  if (batch == 0) return RONK_OK;
  const u32 log_m = log_n - log_g;
  const int G = 1 << log_g;
  const size_t m = (size_t)1 << log_m, blk = m >> log_g, words = (size_t)batch * m, chunk = (size_t)batch * blk;
  DevBuf<u64> z, tw, pack;
  RONK_TRY(z.alloc(ctx, (size_t)G * words));   // FUSED: the G exchange buffers; NCCL: the G receive buffers
  RONK_TRY(tw.alloc(ctx, m));
  if (flavour == RONK_DIST_NCCL) RONK_TRY(pack.alloc(ctx, words));
  const u64 w = h_powmod(g, (p - 1) >> log_n, p);
  for (int r = 0; r < G; r++) {   // Z_r = NTT_m(a[r::G]) ⊙ ω_n^(r·k')
    u64* local = (u64*)data + (size_t)r * words;
    const u64* twcol = nullptr;
    if (r) {
      RONK_TRY(ronk_field_powers_u64(ctx, p, h_powmod(w, (u64)r, p), 1 % p, tw.get(), m));
      twcol = tw.get();
    }
    if (flavour == RONK_DIST_FUSED) {
      RONK_TRY(ntt_device_shared_mul(ctx, p, g, local, z.get() + (size_t)r * words, twcol, log_m, batch));
    } else {
      RONK_TRY(ntt_device_shared_mul(ctx, p, g, local, local, twcol, log_m, batch));
      const u64* sendbase = local;
      if (batch > 1) {
        RONK_TRY(launch(ctx, "dist_pack", pack_blocks_kernel, grid_for(ctx, words, 256, 16), 256, 0, false, local, pack.get(), blk,
                        log_g, batch));
        sendbase = pack.get();
      }
      // the all-to-all: source r's chunk for destination s lands in s's receive buffer at slot r
      for (int s2 = 0; s2 < G; s2++)
        RONK_CUDA(ctx, cudaMemcpyAsync(z.get() + (size_t)s2 * words + (size_t)r * chunk, sendbase + (size_t)s2 * chunk,
                                       chunk * sizeof(u64), cudaMemcpyDeviceToDevice, ctx->stream));
    }
  }
  for (int r = 0; r < G; r++) {   // rank r's cross-rank stage
    PeerPtrs src;
    for (int q = 0; q < 16; q++) src.p[q] = nullptr;
    u64* local = (u64*)data + (size_t)r * words;
    if (flavour == RONK_DIST_FUSED) {
      for (int q = 0; q < G; q++) src.p[q] = z.get() + (size_t)q * words;
      RONK_TRY(cross_rank(ctx, p, g, log_g, src, local, blk, batch, m, (size_t)r * blk, m));
    } else {
      for (int q = 0; q < G; q++) src.p[q] = z.get() + (size_t)r * words + (size_t)q * chunk;
      RONK_TRY(cross_rank(ctx, p, g, log_g, src, local, blk, batch, blk, 0, m));
    }
  }
  RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));   // the scratch buffers are freed on return
  return RONK_OK;
}

int ronk_msm_pluto_ext_dist(ronk_ctx* ctx, const uint8_t* points, size_t n_points, const uint8_t* scalars,
                            size_t n_scalars, uint8_t out[4]) {
  ronk::DeviceGuard _dg(ctx);
  DistState* d = nullptr;
  RONK_TRY(dist_check(ctx, &d));
  if (!out) return set_err(ctx, RONK_EINVAL, "null argument");
  uint8_t mine[4];
  const int rc_local = ronk_msm_pluto_ext(ctx, points, n_points, scalars, n_scalars, mine);
  // every rank takes part in the collective even if its shard was rejected (the flag travels with the point)
  u32 word = (rc_local == RONK_OK) ? ((u32)mine[0] | ((u32)mine[1] << 8) | ((u32)mine[2] << 16) | ((u32)mine[3] << 24))
                                   : 0xFFFFFFFEu;  // not a valid packing: marks a failed shard
  u32* gather = d->gather.get();
  RONK_CUDA(ctx, cudaMemcpyAsync(gather + 16, &word, sizeof(u32), cudaMemcpyHostToDevice, ctx->stream));
  RONK_NCCL(ctx, nccl_api().AllGather(gather + 16, gather, 1, ncclUint32, d->comm, ctx->stream));
  u32 all[16];
  RONK_CUDA(ctx, cudaMemcpyAsync(all, gather, sizeof(u32) * (size_t)d->world, cudaMemcpyDeviceToHost, ctx->stream));
  RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  for (int r = 0; r < d->world; r++)
    if (all[r] == 0xFFFFFFFEu)
      return set_err(ctx, RONK_EINVAL, rc_local == RONK_OK ? std::string("a peer's shard holds an invalid term") : ctx->err);
  volatile u32* host = (volatile u32*)ctx->h_flag;
  u32* host_dev = nullptr;
  RONK_CUDA(ctx, cudaHostGetDevicePointer((void**)&host_dev, (void*)ctx->h_flag, 0));
  host[1] = PT_INF;
  RONK_TRY(launch(ctx, "point_sum", point_sum_kernel, 1, 32, 0, false, gather, (u32)d->world, host_dev + 1));
  RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  const u32 res = host[1];
  out[0] = (uint8_t)(res & 0xFF);
  out[1] = (uint8_t)((res >> 8) & 0xFF);
  out[2] = (uint8_t)((res >> 16) & 0xFF);
  out[3] = (uint8_t)(res >> 24);
  return RONK_OK;
}

}  // extern "C"
