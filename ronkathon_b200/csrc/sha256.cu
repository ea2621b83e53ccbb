// sha256.cu — batches of the reference's SHA-256 (src/hashes/sha.rs:88-201) and its Merkle tree (src/tree/merkle.rs):
// ronk_sha256, ronk_merkle_build_sha256, ronk_merkle_proofs_sha256, ronk_merkle_verify_sha256 and their _host twins
// (include/ronk_b200.h).  The hashing itself is sha256.cuh.
//
// - sha256_kernel: one thread per message, grid-stride.
// - merkle_span_kernel: one CTA of MERKLE_SPAN threads per span of MERKLE_SPAN consecutive nodes of one level.  The
//   first launch of a build hashes the leaves; each later one reads the nodes of the level the previous launch ended
//   on.  Either way the CTA then reduces its span through up to MERKLE_SPAN_LOG levels in shared memory, writing every
//   level's nodes to global.  A span of level b holds exactly the children of the span's nodes at the levels above, so
//   no CTA needs another's nodes, and the odd last node of a level lies in the last span.  A build is
//   1 + ⌈max(L − 9, 0) / 9⌉ launches.
// - merkle_proofs_kernel: one thread per (index, level).  merkle_verify_kernel: one thread per item.
// - Bad offsets, proof indices and side bytes raise the context's mapped error flag; each call synchronises once to read
//   it.  A thread whose input is bad reads nothing through it.
#include "ronk_internal.h"
#include "sha256.cuh"

namespace ronk {

constexpr int SHA_THREADS = 128;
// Nodes per CTA of a tree build: 512 digests of 32 bytes fill 16 KiB of shared memory and span 9 levels.
constexpr u32 MERKLE_SPAN_LOG = 9, MERKLE_SPAN = 1u << MERKLE_SPAN_LOG;
constexpr u64 SHA_MAX_DATA = (u64)1 << 40;
constexpr u32 MERKLE_MAX_DEPTH = 32;

// The levels of a tree of n leaves: level l (0 = leaves) holds size[l] = ⌈n / 2^l⌉ nodes from node off[l] of the node
// buffer on; depth = L = ⌈log2 n⌉ for n ≥ 2, else 0.
struct MerkleLevels {
  u64 size[MERKLE_MAX_DEPTH + 1];
  u64 off[MERKLE_MAX_DEPTH + 1];
  u32 depth;
};

static MerkleLevels merkle_levels(u64 n) {
  MerkleLevels lv = {};
  lv.depth = n >= 2 ? log2_ceil(n) : 0;
  u64 at = 0;
  for (u32 l = 0; l <= lv.depth; l++) {
    lv.size[l] = n ? ((n - 1) >> l) + 1 : 0;
    lv.off[l] = at;
    at += lv.size[l];
  }
  return lv;
}

static u64 merkle_total(const MerkleLevels& lv) { return lv.off[lv.depth] + lv.size[lv.depth]; }

// The big-endian bytes of h0 … h7 at p, any alignment.
__device__ __forceinline__ void store_digest(uint8_t* p, const u32 h[8]) {
  u32 b[8];
#pragma unroll
  for (int k = 0; k < 8; k++) b[k] = sha_bswap(h[k]);
  if (((uintptr_t)p & 15) == 0) {
    ((uint4*)p)[0] = make_uint4(b[0], b[1], b[2], b[3]);
    ((uint4*)p)[1] = make_uint4(b[4], b[5], b[6], b[7]);
  } else {
#pragma unroll
    for (int k = 0; k < 32; k++) p[k] = (uint8_t)(b[k / 4] >> (8 * (k % 4)));
  }
}

__device__ __forceinline__ void load_digest(const uint8_t* p, u32 h[8]) {
  if (((uintptr_t)p & 15) == 0) {
    const uint4 x = ((const uint4*)p)[0], y = ((const uint4*)p)[1];
    h[0] = x.x; h[1] = x.y; h[2] = x.z; h[3] = x.w; h[4] = y.x; h[5] = y.y; h[6] = y.z; h[7] = y.w;
  } else {
#pragma unroll
    for (int k = 0; k < 8; k++) h[k] = (u32)p[4 * k] | (u32)p[4 * k + 1] << 8 | (u32)p[4 * k + 2] << 16 | (u32)p[4 * k + 3] << 24;
  }
#pragma unroll
  for (int k = 0; k < 8; k++) h[k] = sha_bswap(h[k]);
}

// Message i of a batch is data[off[i], off[i+1]).  False, with nothing of data read, unless
// off[0] ≤ off[i] ≤ off[i+1] ≤ off[n] ≤ data_len: then no message of a batch with bad offsets is read outside
// [off[0], off[n]), and every bad batch has a thread that sees it.
__device__ __forceinline__ bool message_range(const u64* off, u64 n, u64 i, u64 data_len, u64* s, u64* e) {
  const u64 lo = off[0], hi = off[n];
  *s = off[i];
  *e = off[i + 1];
  return lo <= *s && *s <= *e && *e <= hi && hi <= data_len;
}

__global__ void __launch_bounds__(SHA_THREADS)
sha256_kernel(const uint8_t* data, u64 data_len, const u64* __restrict__ off, u64 n, uint8_t* out, volatile u32* flag) {
  const u64 stride = (u64)gridDim.x * SHA_THREADS;
  for (u64 i = (u64)blockIdx.x * SHA_THREADS + threadIdx.x; i < n; i += stride) {
    u64 s, e;
    if (!message_range(off, n, i, data_len, &s, &e)) {
      *flag = 1u;
      continue;
    }
    u32 h[8];
    sha_message(data + s, e - s, h);
    store_digest(out + 32 * i, h);
  }
}

// One span of level `base`: the leaves' digests (LEAVES) or the level's nodes, then `nlev` levels above them.
template <bool LEAVES>
__global__ void __launch_bounds__(MERKLE_SPAN)
merkle_span_kernel(const uint8_t* data, u64 data_len, const u64* __restrict__ off, uint8_t* nodes, MerkleLevels lv, u32 base,
                   u32 nlev, volatile u32* flag) {
  __shared__ u32 sm[8 * MERKLE_SPAN];  // word-major: sm[k·SPAN + i] is word k of node i, so a node pair costs 2-way conflicts
  const u32 t = threadIdx.x;
  const u64 first = (u64)blockIdx.x * MERKLE_SPAN;
  const u64 left = lv.size[base] - first;
  u32 cnt = left < MERKLE_SPAN ? (u32)left : MERKLE_SPAN;
  u32 h[8];
  if (t < cnt) {
    if (LEAVES) {
      u64 s, e;
      if (message_range(off, lv.size[0], first + t, data_len, &s, &e)) {
        sha_message(data + s, e - s, h);
      } else {
        *flag = 1u;
#pragma unroll
        for (int k = 0; k < 8; k++) h[k] = 0;
      }
      store_digest(nodes + 32 * (first + t), h);
    } else {
      load_digest(nodes + 32 * (lv.off[base] + first + t), h);
    }
#pragma unroll
    for (int k = 0; k < 8; k++) sm[k * MERKLE_SPAN + t] = h[k];
  }
  for (u32 l = 1; l <= nlev; l++) {
    const u32 next = (cnt + 1) / 2;
    __syncthreads();
    if (t < next) merkle_span_node(sm, MERKLE_SPAN, t, cnt, h);
    __syncthreads();
    if (t < next) {
#pragma unroll
      for (int k = 0; k < 8; k++) sm[k * MERKLE_SPAN + t] = h[k];
      store_digest(nodes + 32 * (lv.off[base + l] + (first >> l) + t), h);
    }
    cnt = next;
  }
}

__global__ void __launch_bounds__(SHA_THREADS)
merkle_proofs_kernel(const uint8_t* nodes, MerkleLevels lv, const u64* __restrict__ idx, u64 m, uint8_t* sib, uint8_t* sides,
                     volatile u32* flag) {
  const u64 total = m * lv.depth, stride = (u64)gridDim.x * SHA_THREADS;
  for (u64 t = (u64)blockIdx.x * SHA_THREADS + threadIdx.x; t < total; t += stride) {
    const u32 l = (u32)(t % lv.depth);
    const u64 x = idx[t / lv.depth] >> l, s = x ^ 1;
    if (s >= lv.size[l]) {  // merkle.rs:72-77 indexes past the level: the reference panics
      *flag = 1u;
      continue;
    }
    u32 h[8];
    load_digest(nodes + 32 * (lv.off[l] + s), h);
    store_digest(sib + 32 * t, h);
    sides[t] = (x & 1) ? 0 : 1;  // 0 = Left, 1 = Right
  }
}

__global__ void __launch_bounds__(SHA_THREADS)
merkle_verify_kernel(const uint8_t* root, const uint8_t* data, u64 data_len, const u64* __restrict__ off, u64 m,
                     const uint8_t* sib, const uint8_t* sides, u32 depth, uint8_t* ok, volatile u32* flag) {
  const u64 stride = (u64)gridDim.x * SHA_THREADS;
  u32 want[8];
  load_digest(root, want);
  for (u64 j = (u64)blockIdx.x * SHA_THREADS + threadIdx.x; j < m; j += stride) {
    u64 s, e;
    if (!message_range(off, m, j, data_len, &s, &e)) {
      *flag = 1u;
      ok[j] = 0;
      continue;
    }
    u32 h[8];
    sha_message(data + s, e - s, h);
    bool bad = false;
    for (u32 l = 0; l < depth; l++) {
      const uint8_t side = sides[j * depth + l];
      if (side > 1) {
        bad = true;
        break;
      }
      u32 x[8];
      load_digest(sib + 32 * (j * depth + l), x);
      if (side == 0) sha_node(x, h, h);  // Left: sibling ‖ hash (merkle.rs:89-93)
      else sha_node(h, x, h);
    }
    u32 diff = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) diff |= h[k] ^ want[k];
    if (bad) *flag = 1u;
    ok[j] = !bad && diff == 0;
  }
}

// Step (1) of the message entries' errors (ronk_sha256, ronk_merkle_build_sha256, ronk_merkle_verify_sha256): n
// messages over data_len bytes, out the output the call writes (null allowed only when n == 0).  device: the pointers
// are device pointers, which the kernels load offsets through as u64.
static int message_args(ronk_ctx* ctx, const uint8_t* data, u64 data_len, const u64* offsets, u64 n, const void* out,
                        bool device) {
  if (!ctx) return RONK_EINVAL;
  if ((data_len && !data) || (n && (!offsets || !out))) return set_err(ctx, RONK_EINVAL, "null argument");
  if (device && n && ((uintptr_t)offsets & 7)) return set_err(ctx, RONK_EINVAL, "offsets must be 8-byte aligned");
  if (n >> 32) return set_err(ctx, RONK_EUNSUPPORTED, "n at or above 2^32");
  if (data_len > SHA_MAX_DATA) return set_err(ctx, RONK_EUNSUPPORTED, "data_len above 2^40 bytes");
  return RONK_OK;
}

// The _host twins' check of the offsets, which the device entries make on the device.
static int host_offsets(ronk_ctx* ctx, const u64* off, u64 n, u64 data_len) {
  if (!n) return RONK_OK;
  for (u64 i = 0; i < n; i++)
    if (off[i] > off[i + 1]) return set_err(ctx, RONK_EINVAL, "offsets decrease");
  if (off[n] > data_len) return set_err(ctx, RONK_EINVAL, "offsets pass data_len");
  return RONK_OK;
}

// Step (4): the launches were enqueued by go(flag); wait for them and read the flag.
template <class Go>
static int run_flagged(ronk_ctx* ctx, const char* what, Go&& go) {
  volatile u32* flag = nullptr;
  RONK_TRY(clear_flag(ctx, &flag));
  RONK_TRY(go(flag));
  RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (ctx->h_flag[0]) return set_err(ctx, RONK_EINVAL, what);
  return RONK_OK;
}

}  // namespace ronk

using namespace ronk;

extern "C" {

int ronk_sha256(ronk_ctx* ctx, const uint8_t* data, uint64_t data_len, const uint64_t* offsets, size_t n, uint8_t* out) {
  ronk::DeviceGuard _dg(ctx);
  RONK_TRY(message_args(ctx, data, data_len, offsets, n, out, true));
  if (bytes_overlap(out, 32 * n, data, data_len) || bytes_overlap(out, 32 * n, offsets, 8 * (n + 1)))
    return set_err(ctx, RONK_EINVAL, "out overlaps an input");
  if (n == 0) return RONK_OK;
  return run_flagged(ctx, "offsets decrease or pass data_len", [&](volatile u32* flag) {
    return launch(ctx, "sha256", sha256_kernel, grid_for(ctx, n, SHA_THREADS), SHA_THREADS, 0, false, data, (u64)data_len,
                  offsets, (u64)n, out, flag);
  });
}

int ronk_merkle_build_sha256(ronk_ctx* ctx, const uint8_t* data, uint64_t data_len, const uint64_t* offsets, size_t n,
                             uint8_t* nodes) {
  ronk::DeviceGuard _dg(ctx);
  RONK_TRY(message_args(ctx, data, data_len, offsets, n, nodes, true));
  const MerkleLevels lv = merkle_levels(n);
  const u64 total = n ? merkle_total(lv) : 0;
  if (bytes_overlap(nodes, 32 * total, data, data_len) || bytes_overlap(nodes, 32 * total, offsets, 8 * (n + 1)))
    return set_err(ctx, RONK_EINVAL, "nodes overlap an input");
  if (n == 0) return RONK_OK;
  return run_flagged(ctx, "offsets decrease or pass data_len", [&](volatile u32* flag) {
    for (u32 base = 0;; base += MERKLE_SPAN_LOG) {
      const u32 nlev = std::min(lv.depth - base, MERKLE_SPAN_LOG);
      const int grid = (int)((lv.size[base] + MERKLE_SPAN - 1) / MERKLE_SPAN);
      if (base == 0)
        RONK_TRY(launch(ctx, "merkle_leaves", merkle_span_kernel<true>, grid, MERKLE_SPAN, 0, false, data, (u64)data_len,
                        offsets, nodes, lv, base, nlev, flag));
      else
        RONK_TRY(launch(ctx, "merkle_nodes", merkle_span_kernel<false>, grid, MERKLE_SPAN, 0, false, data, (u64)data_len,
                        offsets, nodes, lv, base, nlev, flag));
      if (base + nlev == lv.depth) return RONK_OK;
    }
  });
}

int ronk_merkle_proofs_sha256(ronk_ctx* ctx, const uint8_t* nodes, size_t n, const uint64_t* indices, size_t m,
                              uint8_t* siblings, uint8_t* sides) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx) return RONK_EINVAL;
  const MerkleLevels lv = merkle_levels(n >> 32 ? 0 : n);
  const u64 L = lv.depth;
  if (m && L && (!nodes || !indices || !siblings || !sides)) return set_err(ctx, RONK_EINVAL, "null argument");
  if (m && L && ((uintptr_t)indices & 7)) return set_err(ctx, RONK_EINVAL, "indices must be 8-byte aligned");
  if ((n >> 32) || (m >> 32)) return set_err(ctx, RONK_EUNSUPPORTED, "n or m at or above 2^32");
  const u64 total = n ? merkle_total(lv) : 0;
  if (bytes_overlap(siblings, 32 * m * L, nodes, 32 * total) || bytes_overlap(siblings, 32 * m * L, indices, 8 * m) ||
      bytes_overlap(sides, m * L, nodes, 32 * total) || bytes_overlap(sides, m * L, indices, 8 * m) ||
      bytes_overlap(sides, m * L, siblings, 32 * m * L))
    return set_err(ctx, RONK_EINVAL, "siblings or sides overlap an input or each other");
  if (m == 0 || L == 0) return RONK_OK;
  return run_flagged(ctx, "a proof index at which get_proof panics (merkle.rs:77)", [&](volatile u32* flag) {
    return launch(ctx, "merkle_proofs", merkle_proofs_kernel, grid_for(ctx, m * L, SHA_THREADS), SHA_THREADS, 0, false, nodes,
                  lv, indices, (u64)m, siblings, sides, flag);
  });
}

int ronk_merkle_verify_sha256(ronk_ctx* ctx, const uint8_t* root, const uint8_t* data, uint64_t data_len,
                              const uint64_t* offsets, size_t m, const uint8_t* siblings, const uint8_t* sides, uint32_t depth,
                              uint8_t* ok) {
  ronk::DeviceGuard _dg(ctx);
  RONK_TRY(message_args(ctx, data, data_len, offsets, m, ok, true));
  if (m && (!root || (depth && (!siblings || !sides)))) return set_err(ctx, RONK_EINVAL, "null argument");
  if (depth > MERKLE_MAX_DEPTH) return set_err(ctx, RONK_EUNSUPPORTED, "depth above 32");
  const u64 steps = (u64)m * depth;
  if (bytes_overlap(ok, m, root, 32) || bytes_overlap(ok, m, data, data_len) || bytes_overlap(ok, m, offsets, 8 * (m + 1)) ||
      bytes_overlap(ok, m, siblings, 32 * steps) || bytes_overlap(ok, m, sides, steps))
    return set_err(ctx, RONK_EINVAL, "ok overlaps an input");
  if (m == 0) return RONK_OK;
  return run_flagged(ctx, "offsets decrease or pass data_len, or a side byte other than 0 or 1", [&](volatile u32* flag) {
    return launch(ctx, "merkle_verify", merkle_verify_kernel, grid_for(ctx, m, SHA_THREADS), SHA_THREADS, 0, false, root, data,
                  (u64)data_len, offsets, (u64)m, siblings, sides, depth, ok, flag);
  });
}

int ronk_sha256_host(ronk_ctx* ctx, const uint8_t* data, uint64_t data_len, const uint64_t* offsets, size_t n, uint8_t* out) {
  ronk::DeviceGuard _dg(ctx);
  RONK_TRY(message_args(ctx, data, data_len, offsets, n, out, false));
  RONK_TRY(host_offsets(ctx, offsets, n, data_len));
  if (n == 0) return RONK_OK;
  Staged s[] = {{data_len, data}, {8 * (n + 1), offsets}, {32 * n, nullptr, out}};
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  return stage_out(ctx, ronk_sha256(ctx, (const uint8_t*)s[0].dev, data_len, s[1].dev, n, (uint8_t*)s[2].dev), s);
}

int ronk_merkle_build_sha256_host(ronk_ctx* ctx, const uint8_t* data, uint64_t data_len, const uint64_t* offsets, size_t n,
                                  uint8_t* nodes) {
  ronk::DeviceGuard _dg(ctx);
  RONK_TRY(message_args(ctx, data, data_len, offsets, n, nodes, false));
  RONK_TRY(host_offsets(ctx, offsets, n, data_len));
  if (n == 0) return RONK_OK;
  Staged s[] = {{data_len, data}, {8 * (n + 1), offsets}, {32 * merkle_total(merkle_levels(n)), nullptr, nodes}};
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  return stage_out(ctx, ronk_merkle_build_sha256(ctx, (const uint8_t*)s[0].dev, data_len, s[1].dev, n, (uint8_t*)s[2].dev), s);
}

int ronk_merkle_proofs_sha256_host(ronk_ctx* ctx, const uint8_t* nodes, size_t n, const uint64_t* indices, size_t m,
                                   uint8_t* siblings, uint8_t* sides) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx) return RONK_EINVAL;
  const MerkleLevels lv = merkle_levels(n >> 32 ? 0 : n);
  const u64 L = lv.depth;
  if (m && L && (!nodes || !indices || !siblings || !sides)) return set_err(ctx, RONK_EINVAL, "null argument");
  if ((n >> 32) || (m >> 32)) return set_err(ctx, RONK_EUNSUPPORTED, "n or m at or above 2^32");
  if (m == 0 || L == 0) return RONK_OK;
  Staged s[] = {{32 * merkle_total(lv), nodes}, {8 * m, indices}, {32 * m * L, nullptr, siblings}, {m * L, nullptr, sides}};
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  return stage_out(ctx,
                   ronk_merkle_proofs_sha256(ctx, (const uint8_t*)s[0].dev, n, s[1].dev, m, (uint8_t*)s[2].dev,
                                             (uint8_t*)s[3].dev),
                   s);
}

int ronk_merkle_verify_sha256_host(ronk_ctx* ctx, const uint8_t* root, const uint8_t* data, uint64_t data_len,
                                   const uint64_t* offsets, size_t m, const uint8_t* siblings, const uint8_t* sides,
                                   uint32_t depth, uint8_t* ok) {
  ronk::DeviceGuard _dg(ctx);
  RONK_TRY(message_args(ctx, data, data_len, offsets, m, ok, false));
  if (m && (!root || (depth && (!siblings || !sides)))) return set_err(ctx, RONK_EINVAL, "null argument");
  if (depth > MERKLE_MAX_DEPTH) return set_err(ctx, RONK_EUNSUPPORTED, "depth above 32");
  RONK_TRY(host_offsets(ctx, offsets, m, data_len));
  const u64 steps = (u64)m * depth;
  for (u64 i = 0; i < steps; i++)
    if (sides[i] > 1) return set_err(ctx, RONK_EINVAL, "a side byte other than 0 or 1");
  if (m == 0) return RONK_OK;
  Staged s[] = {{32, root}, {data_len, data}, {8 * (m + 1), offsets}, {32 * steps, siblings}, {steps, sides}, {m, nullptr, ok}};
  Frame fr(ctx);
  RONK_TRY(stage_in(fr, s));
  return stage_out(ctx,
                   ronk_merkle_verify_sha256(ctx, (const uint8_t*)s[0].dev, (const uint8_t*)s[1].dev, data_len, s[2].dev, m,
                                             (const uint8_t*)s[3].dev, (const uint8_t*)s[4].dev, depth, (uint8_t*)s[5].dev),
                   s);
}

}  // extern "C"
