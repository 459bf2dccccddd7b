// estk_ctx.cu -- context, error text, version.
#include "estk_common.cuh"
#include <string.h>
#include <new>

static thread_local char g_estk_err[512] = "";

void estk_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_estk_err, sizeof(g_estk_err), fmt, ap);
  va_end(ap);
}

extern "C" int estk_version(void) { return ESTK_VERSION; }
extern "C" const char* estk_last_error(void) { return g_estk_err; }

extern "C" int estk_ctx_create(int device, estk_ctx** out) {
  ESTK_CHECK_ARG(out != nullptr, "estk_ctx_create: out is null");
  *out = nullptr;
  int count = 0;
  ESTK_CUDA(cudaGetDeviceCount(&count));
  ESTK_CHECK_ARG(device >= 0 && device < count, "estk_ctx_create: device %d of %d", device, count);
  ESTK_CUDA(cudaSetDevice(device));
  cudaDeviceProp prop;
  ESTK_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9) {
    estk_set_error("libestk is built for sm_90a (H100); device %d is sm_%d%d", device, prop.major,
                   prop.minor);
    return ESTK_ERR_UNSUPPORTED;
  }
  estk_ctx* c = new (std::nothrow) estk_ctx();
  if (!c) return ESTK_ERR_NOMEM;
  memset(c, 0, sizeof(*c));
  c->device = device;
  c->sm_count = prop.multiProcessorCount;
  c->cc_major = prop.major;
  c->cc_minor = prop.minor;
  c->max_grid = c->sm_count * 8;
  cudaError_t e = cudaSuccess;
  if (e == cudaSuccess) e = cudaMalloc(&c->cvals, sizeof(float) * ESTK_MAX_POPULATION);
  if (e == cudaSuccess) e = cudaMalloc(&c->partial, sizeof(float) * (size_t)c->max_grid * 1024);
  if (e == cudaSuccess)
    e = cudaMalloc(&c->eval_partial, sizeof(float) * (size_t)ESTK_MAX_POPULATION * 2 * kEvalMaxChunks);
  if (e == cudaSuccess) e = cudaMalloc(&c->counters, sizeof(unsigned int) * (ESTK_MAX_POPULATION + 8));
  if (e == cudaSuccess) e = cudaMalloc(&c->scalars, sizeof(double) * 8);
  if (e == cudaSuccess) e = cudaMemset(c->counters, 0, sizeof(unsigned int) * (ESTK_MAX_POPULATION + 8));
  if (e != cudaSuccess) {
    estk_set_error("estk_ctx_create: workspace allocation failed: %s", cudaGetErrorString(e));
    estk_ctx_destroy(c);
    return ESTK_ERR_NOMEM;
  }
  *out = c;
  return ESTK_OK;
}

extern "C" int estk_ctx_destroy(estk_ctx* c) {
  if (!c) return ESTK_OK;
  cudaFree(c->cvals);
  cudaFree(c->partial);
  cudaFree(c->eval_partial);
  cudaFree(c->counters);
  cudaFree(c->scalars);
  delete c;
  return ESTK_OK;
}

extern "C" int estk_ctx_info(estk_ctx* c, int* sm_count, int* cc_major, int* cc_minor) {
  ESTK_CHECK_ARG(c != nullptr, "estk_ctx_info: ctx is null");
  if (sm_count) *sm_count = c->sm_count;
  if (cc_major) *cc_major = c->cc_major;
  if (cc_minor) *cc_minor = c->cc_minor;
  return ESTK_OK;
}


// ------------------------------------------------------------------ peer memory (CUDA IPC)
// Device memory another process on the same node can map (estk.h: estk_rank_grad_xr_adam).
extern "C" int estk_peer_alloc(estk_ctx* ctx, int64_t bytes, void** ptr_out, unsigned char* handle_out) {
  ESTK_CHECK_ARG(ctx && ptr_out && handle_out && bytes > 0, "estk_peer_alloc: bad argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == ESTK_PEER_HANDLE_BYTES, "handle size");
  void* ptr = nullptr;
  ESTK_CUDA(cudaMalloc(&ptr, (size_t)bytes));
  cudaError_t e = cudaMemset(ptr, 0, (size_t)bytes);
  cudaIpcMemHandle_t h;
  if (e == cudaSuccess) e = cudaIpcGetMemHandle(&h, ptr);
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    cudaFree(ptr);
    estk_set_error("estk_peer_alloc: %s", cudaGetErrorString(e));
    return ESTK_ERR_CUDA;
  }
  memcpy(handle_out, &h, sizeof(h));
  *ptr_out = ptr;
  return ESTK_OK;
}

extern "C" int estk_peer_open(estk_ctx* ctx, const unsigned char* handle, void** ptr_out) {
  ESTK_CHECK_ARG(ctx && handle && ptr_out, "estk_peer_open: null argument");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, sizeof(h));
  ESTK_CUDA(cudaIpcOpenMemHandle(ptr_out, h, cudaIpcMemLazyEnablePeerAccess));
  return ESTK_OK;
}

extern "C" int estk_peer_close(estk_ctx* ctx, void* ptr) {
  ESTK_CHECK_ARG(ctx && ptr, "estk_peer_close: null argument");
  ESTK_CUDA(cudaIpcCloseMemHandle(ptr));
  return ESTK_OK;
}

extern "C" int estk_peer_free(estk_ctx* ctx, void* ptr) {
  ESTK_CHECK_ARG(ctx && ptr, "estk_peer_free: null argument");
  ESTK_CUDA(cudaFree(ptr));
  return ESTK_OK;
}
