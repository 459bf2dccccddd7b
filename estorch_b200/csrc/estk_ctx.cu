// estk_ctx.cu -- context, error text, version.
#include "estk_common.cuh"
#include "estk_sort.cuh"
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

static void free_workspace(estk_ctx* c) {
  cudaFree(c->cvals);
  cudaFree(c->eval_partial);
  cudaFree(c->counters);
  cudaFree(c->sort_ws);
  c->cvals = c->eval_partial = nullptr;
  c->counters = nullptr;
  c->sort_ws = nullptr;
  c->members = c->eval_floats = 0;
}

// The per-member buffers for `members` members and `eval_floats` evaluate partials, into `c`; the arrival
// counters are zero-filled on `stream` (every kernel that takes one leaves it at zero again).  On failure
// whatever was allocated is freed again and `c`'s buffers are null.
static cudaError_t alloc_workspace(estk_ctx* c, int64_t members, int64_t eval_floats, cudaStream_t stream) {
  const size_t counters = sizeof(unsigned int) * (size_t)(kCtxTicketSlots + members);
  c->cvals = c->eval_partial = nullptr;
  c->counters = nullptr;
  c->sort_ws = nullptr;
  cudaError_t e = cudaMalloc(&c->cvals, sizeof(float) * (size_t)members);
  if (e == cudaSuccess) e = cudaMalloc(&c->eval_partial, sizeof(float) * (size_t)eval_floats);
  if (e == cudaSuccess) e = cudaMalloc(&c->counters, counters);
  if (e == cudaSuccess) e = cudaMalloc(&c->sort_ws, estk_sort::workspace_bytes(members, 4, c->max_grid));
  if (e == cudaSuccess) e = cudaMemsetAsync(c->counters, 0, counters, stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(stream);   // zero before any launch on any stream
  if (e != cudaSuccess) {
    free_workspace(c);
    return e;
  }
  c->members = members;
  c->eval_floats = eval_floats;
  return e;
}

// Buffers replaced by a growth stay allocated until estk_ctx_destroy: a CUDA graph captured before the
// growth still points at them, and replaying it must not touch freed memory.
static void retire(estk_ctx* c, void* ptr) {
  if (c->n_retired == kCtxMaxRetired) {
    // (only after kCtxMaxRetired / 4 growths of one context) nothing in flight may still use them
    cudaDeviceSynchronize();
    for (int i = 0; i < c->n_retired; ++i) cudaFree(c->retired[i]);
    c->n_retired = 0;
  }
  c->retired[c->n_retired++] = ptr;
}

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
  cudaError_t e = cudaMalloc(&c->partial, sizeof(float) * (size_t)c->max_grid * 1024);
  if (e == cudaSuccess) e = cudaMalloc(&c->scalars, sizeof(double) * 8);
  if (e == cudaSuccess) e = alloc_workspace(c, kCtxInitialMembers, kCtxInitialMembers * 2 * kEvalMaxChunks, 0);
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
  free_workspace(c);
  for (int i = 0; i < c->n_retired; ++i) cudaFree(c->retired[i]);
  cudaFree(c->partial);
  cudaFree(c->scalars);
  delete c;
  return ESTK_OK;
}

int estk_ctx_reserve(estk_ctx* c, int64_t members, int64_t eval_floats, cudaStream_t stream, const char* who) {
  if (members <= c->members && eval_floats <= c->eval_floats) return ESTK_OK;
  cudaStreamCaptureStatus capture = cudaStreamCaptureStatusNone;
  ESTK_CUDA(cudaStreamIsCapturing(stream, &capture));
  if (capture != cudaStreamCaptureStatusNone) {
    estk_set_error("%s: the context workspace must grow (%lld members, %lld evaluate partials; it holds %lld, %lld), "
                   "which is not possible while the stream is captured into a CUDA graph: run the same call once "
                   "before capturing it", who, (long long)members, (long long)eval_floats, (long long)c->members,
                   (long long)c->eval_floats);
    return ESTK_ERR_NOMEM;
  }
  if (members < c->members) members = c->members;
  if (eval_floats < c->eval_floats) eval_floats = c->eval_floats;
  members = (members + 1023) / 1024 * 1024;
  int prev = 0;
  ESTK_CUDA(cudaGetDevice(&prev));
  ESTK_CUDA(cudaSetDevice(c->device));
  // the new buffers first: on failure the context keeps the ones it has
  estk_ctx grown = *c;
  const cudaError_t e = alloc_workspace(&grown, members, eval_floats, stream);
  cudaSetDevice(prev);
  if (e != cudaSuccess) {
    cudaGetLastError();   // an allocation failure is not sticky: clear it for the caller's next launch
    estk_set_error("%s: growing the context workspace to %lld members, %lld evaluate partials failed: %s", who,
                   (long long)members, (long long)eval_floats, cudaGetErrorString(e));
    return ESTK_ERR_NOMEM;
  }
  retire(c, c->cvals);
  retire(c, c->eval_partial);
  retire(c, c->counters);
  retire(c, c->sort_ws);
  c->cvals = grown.cvals;
  c->eval_partial = grown.eval_partial;
  c->counters = grown.counters;
  c->sort_ws = grown.sort_ws;
  c->members = grown.members;
  c->eval_floats = grown.eval_floats;
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
