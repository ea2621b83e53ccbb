// api.cu — context management, profiling and memory helpers of the C ABI (include/ronk_b200.h).
#include <cstdlib>

#include "ronk_internal.h"

using namespace ronk;

// The device is bound (ronk_ctx_destroy, ronk_ctx_create); the DevBuf members free the device memory after this body.
ronk_ctx::~ronk_ctx() {
  for (auto& r : prof_log) { cudaEventDestroy(r.start); cudaEventDestroy(r.stop); }
  for (int i = 0; i < kSlots; i++) {
    if (ev_h2d[i]) cudaEventDestroy(ev_h2d[i]);
    if (ev_compute[i]) cudaEventDestroy(ev_compute[i]);
    if (ev_d2h[i]) cudaEventDestroy(ev_d2h[i]);
  }
  if (copy_in) cudaStreamDestroy(copy_in);
  if (copy_out) cudaStreamDestroy(copy_out);
  for (auto& b : scratch.blocks) cudaFreeAsync(b.base, stream);
  cudaStreamSynchronize(stream);
  if (h_flag) cudaFreeHost(h_flag);
}

extern "C" {

const char* ronk_strerror(int code) {
  switch (code) {
    case RONK_OK: return "ok";
    case RONK_EINVAL: return "invalid argument (the reference would panic here)";
    case RONK_ECUDA: return "CUDA error";
    case RONK_ENOMEM: return "out of device memory";
    case RONK_ENCCL: return "collective error";
    case RONK_EUNSUPPORTED: return "unsupported configuration";
    default: return "unknown error";
  }
}

int ronk_ctx_create(ronk_ctx** out, int device, void* stream) {
  if (!out) return RONK_EINVAL;
  *out = nullptr;
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0) return RONK_ECUDA;  // no CPU fallback: fail loudly
  if (device < 0 || device >= count) return RONK_EINVAL;
  int prev = -1;
  cudaGetDevice(&prev);  // the caller's current device is restored before returning
  struct Restore {
    int d;
    ~Restore() { if (d >= 0) cudaSetDevice(d); }
  } restore{prev};
  if (cudaSetDevice(device) != cudaSuccess) return RONK_ECUDA;
  ronk_ctx* ctx = new ronk_ctx();
  ctx->device = device;
  auto env_int = [](const char* name, int dflt) {
    const char* s = getenv(name);
    return s ? atoi(s) : dflt;
  };
  ctx->tune.pf_dist = env_int("RONK_PF_DIST", 1);
  ctx->tune.pf_dist2 = env_int("RONK_PF_DIST2", 1);
  ctx->tune.pdl = env_int("RONK_PDL", 1);
  ctx->tune.ntt3 = env_int("RONK_NTT3", 1);
  ctx->tune.ntt3_pdl = env_int("RONK_NTT3_PDL", 1);
  ctx->tune.ntt3_t1 = env_int("RONK_NTT3_T1", 20);
  ctx->tune.ntt3_20 = env_int("RONK_NTT3_20", 1);
  ctx->tune.ntt3_mid = env_int("RONK_NTT3_MID", 1);
  ctx->tune.ntt3_split = env_int("RONK_NTT3_SPLIT", 1);
  ctx->tune.ntt3_split_min16 = env_int("RONK_NTT3_SPLIT_MIN16", 1);
  ctx->tune.ntt16_cluster_max_batch = env_int("RONK_NTT16_CLUSTER_MAX_BATCH", 2);
  ctx->tune.ntt3_ng1_tiles = env_int("RONK_NTT3_NG1_TILES", 6);
  ctx->tune.ntt3_min_batch16 = env_int("RONK_NTT3_MIN_BATCH16", 1);
  ctx->tune.single_tile_log = env_int("RONK_SINGLE_TILE_LOG", 12);
  ctx->tune.tile1 = env_int("RONK_TILE1", 14);
  ctx->tune.tile2 = env_int("RONK_TILE2", 13);
  ctx->tune.tile_adapt = env_int("RONK_TILE_ADAPT", 1);
  ctx->tune.fast12 = env_int("RONK_FAST12", 0);
  ctx->tune.tw_table = env_int("RONK_TW_TABLE", ctx->tune.fast12 ? 1 : 0);  // the specialised pass 1 reads the table
  ctx->tune.msm_coord = env_int("RONK_MSM_COORD", 1);
  ctx->tune.msm_hist = env_int("RONK_MSM_HIST", 1);
  ctx->tune.msm_split = env_int("RONK_MSM_SPLIT", 0);
  ctx->tune.tree_min = env_int("RONK_TREE_MIN", -1);
  ctx->tune.anyntt_min = env_int("RONK_ANYNTT_MIN", -1);
  const char* crt_min = getenv("RONK_CRT_MUL_MIN");
  ctx->tune.crt_mul_min = crt_min ? strtoll(crt_min, nullptr, 10) : -1;
  ctx->tune.poly_batch_path = env_int("RONK_POLY_BATCH_PATH", 0);
  ctx->tune.divrem_batch_path = env_int("RONK_DIVREM_BATCH_PATH", 0);
  ctx->stream = (cudaStream_t)stream;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) { delete ctx; return RONK_ECUDA; }
  ctx->sm_count = prop.multiProcessorCount;
  if (prop.major != 9 || prop.minor != 0) { delete ctx; return RONK_EUNSUPPORTED; }  // sm_90a-only binary: compute capability 9.0 alone
  if (ctx->d_flag.alloc(ctx, 1) != RONK_OK ||
      cudaHostAlloc((void**)&ctx->h_flag, 32 * sizeof(int), cudaHostAllocMapped) != cudaSuccess) {  // h_flag[0] + 31 words of small results
    delete ctx;
    return RONK_ENOMEM;
  }
  *out = ctx;
  return RONK_OK;
}

int ronk_ctx_destroy(ronk_ctx* ctx) {
  if (!ctx) return RONK_OK;
  ronk::DeviceGuard _dg(ctx);
  cudaStreamSynchronize(ctx->stream);
  if (ctx->dist) ronk_dist_finalize(ctx);
  delete ctx;
  return RONK_OK;
}


int ronk_ctx_set_stream(ronk_ctx* ctx, void* stream) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx) return RONK_EINVAL;
  RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  ctx->stream = (cudaStream_t)stream;
  return RONK_OK;
}

int ronk_sync(ronk_ctx* ctx) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx) return RONK_EINVAL;
  RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return RONK_OK;
}

const char* ronk_last_error(ronk_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }
uint64_t ronk_launch_count(ronk_ctx* ctx) { return ctx ? ctx->launches : 0; }

int ronk_prof_enable(ronk_ctx* ctx, int on) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx) return RONK_EINVAL;
  ctx->prof = on != 0;
  return RONK_OK;
}

int ronk_prof_fetch(ronk_ctx* ctx, char (*names)[32], float* ms, int max) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx) return 0;
  cudaStreamSynchronize(ctx->stream);
  int n = 0;
  for (auto& r : ctx->prof_log) {
    if (n < max) {
      float t = 0.f;
      cudaEventElapsedTime(&t, r.start, r.stop);
      if (names) std::memcpy(names[n], r.name, 32);
      if (ms) ms[n] = t;
      n++;
    }
    cudaEventDestroy(r.start);
    cudaEventDestroy(r.stop);
  }
  ctx->prof_log.clear();
  return n;
}

int ronk_dev_alloc(ronk_ctx* ctx, void** dptr, size_t bytes) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx || !dptr) return RONK_EINVAL;
  RONK_CUDA(ctx, cudaMalloc(dptr, bytes ? bytes : 1));
  return RONK_OK;
}
int ronk_dev_free(ronk_ctx* ctx, void* dptr) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx) return RONK_EINVAL;
  RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  RONK_CUDA(ctx, cudaFree(dptr));
  return RONK_OK;
}
int ronk_memcpy_h2d(ronk_ctx* ctx, void* dst_dev, const void* src_host, size_t bytes) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx) return RONK_EINVAL;
  RONK_CUDA(ctx, cudaMemcpyAsync(dst_dev, src_host, bytes, cudaMemcpyHostToDevice, ctx->stream));
  RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return RONK_OK;
}
int ronk_memcpy_d2h(ronk_ctx* ctx, void* dst_host, const void* src_dev, size_t bytes) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx) return RONK_EINVAL;
  RONK_CUDA(ctx, cudaMemcpyAsync(dst_host, src_dev, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return RONK_OK;
}

int ronk_memcpy_d2d(ronk_ctx* ctx, void* dst_dev, const void* src_dev, size_t bytes) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx) return RONK_EINVAL;
  RONK_CUDA(ctx, cudaMemcpyAsync(dst_dev, src_dev, bytes, cudaMemcpyDeviceToDevice, ctx->stream));
  return RONK_OK;
}

int ronk_ipc_export(ronk_ctx* ctx, const void* dptr, uint8_t handle[64]) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx || !dptr || !handle) return set_err(ctx, RONK_EINVAL, "null argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  cudaIpcMemHandle_t h;
  RONK_CUDA(ctx, cudaIpcGetMemHandle(&h, const_cast<void*>(dptr)));
  std::memcpy(handle, &h, 64);
  return RONK_OK;
}

int ronk_ipc_open(ronk_ctx* ctx, const uint8_t handle[64], void** dptr) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx || !dptr || !handle) return set_err(ctx, RONK_EINVAL, "null argument");
  cudaIpcMemHandle_t h;
  std::memcpy(&h, handle, 64);
  RONK_CUDA(ctx, cudaIpcOpenMemHandle(dptr, h, cudaIpcMemLazyEnablePeerAccess));
  return RONK_OK;
}

int ronk_ipc_close(ronk_ctx* ctx, void* dptr) {
  ronk::DeviceGuard _dg(ctx);
  if (!ctx) return RONK_EINVAL;
  RONK_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  RONK_CUDA(ctx, cudaIpcCloseMemHandle(dptr));
  return RONK_OK;
}

}  // extern "C"
