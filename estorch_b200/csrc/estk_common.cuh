// estk_common.cuh -- shared host/device helpers for libestk (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include "estk.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "libestk is written for sm_90a (H100) only"
#endif

// ---------------------------------------------------------------- errors
void estk_set_error(const char* fmt, ...);

#define ESTK_CHECK_ARG(cond, ...)                         \
  do {                                                    \
    if (!(cond)) {                                        \
      estk_set_error(__VA_ARGS__);                        \
      return ESTK_ERR_INVALID;                            \
    }                                                     \
  } while (0)

#define ESTK_CUDA(call)                                                          \
  do {                                                                           \
    cudaError_t e_ = (call);                                                     \
    if (e_ != cudaSuccess) {                                                     \
      estk_set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_),     \
                     __FILE__, __LINE__);                                        \
      return ESTK_ERR_CUDA;                                                      \
    }                                                                            \
  } while (0)

#define ESTK_ALIGNED16(p) ((((uintptr_t)(p)) & 15u) == 0)

// estk_mlp_desc.activation: the fifteen defined codes (each hidden kind ReLU / Tanh / ELU / SiLU /
// LeakyReLU x output identity / Tanh with the squared error, and x identity output with the cross-entropy)
static inline bool estk_act_valid(int a) {
  const int h = a & 0xff, rest = a & ~0xff;
  const bool hidden = h == ESTK_ACT_RELU || h == ESTK_ACT_TANH || h == ESTK_ACT_ELU || h == ESTK_ACT_SILU ||
                      h == ESTK_ACT_LEAKY_RELU;
  return hidden && (rest == 0 || rest == ESTK_ACT_OUT_TANH || rest == ESTK_LOSS_XENT);
}

#ifdef __CUDACC__
// y / d rounded to nearest-even in fp32 -- the bits of the IEEE divide y / d -- for d >= 1 or d = +inf,
// without the out-of-line slow path of div.rn.f32 (its calls in the unrolled 64-element epilogue cost
// the cluster kernel's bf16 consumer spills; the streamed wgmma kernel, at 255 registers, spills with
// this form instead and keeps div.rn).  r = 1/d to ~2^-52 by two fp64 Newton steps from rcp.approx, then
// q = y * r in fp64 (relative error < 2^-51) rounded once to fp32.  That rounding is exact: a quotient of
// two 24-bit floats that is not a float is at least 2^-49 (relative) from every fp32 rounding boundary,
// and never on one.  d = +inf (y < -88.7 in SiLU) gives y * 0, the IEEE y / inf; NaNs propagate.
__device__ __forceinline__ float estk_div_rn_ge1(float y, float d) {
  const double dd = d;
  double r;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(dd));
  r = fma(r, fma(-dd, r, 1.0), r);
  r = fma(r, fma(-dd, r, 1.0), r);
  return d == INFINITY ? y * 0.f : __double2float_rn((double)y * r);
}

// The hidden activation H = activation & 0xff on the fp32 value y = acc + bias (estk.h states the
// arithmetic).  H is a compile-time constant, so an epilogue carries no branch on it.  CALL_FREE_DIV:
// SiLU divides with estk_div_rn_ge1 instead of div.rn -- the same bits, another register footprint.
template <int H, bool CALL_FREE_DIV = false>
__device__ __forceinline__ float estk_hidden_act(float y) {
  static_assert(H == ESTK_ACT_RELU || H == ESTK_ACT_TANH || H == ESTK_ACT_ELU || H == ESTK_ACT_SILU ||
                H == ESTK_ACT_LEAKY_RELU, "undefined hidden activation");
  if constexpr (H == ESTK_ACT_TANH) return tanhf(y);
  else if constexpr (H == ESTK_ACT_ELU) return y > 0.f ? y : expm1f(y);
  else if constexpr (H == ESTK_ACT_SILU) {
    const float d = 1.0f + expf(-y);
    return CALL_FREE_DIV ? estk_div_rn_ge1(y, d) : __fdiv_rn(y, d);
  }
  else if constexpr (H == ESTK_ACT_LEAKY_RELU) return y > 0.f ? y : y * 0.01f;
  else return fmaxf(y, 0.f);
}
#endif

// ---------------------------------------------------------------- context
static const int kCtxMaxRetired = 80;   // 16 growths of the 5 workspace buffers
// The per-member buffers are sized for kCtxInitialMembers at estk_ctx_create and grown by
// estk_ctx_reserve when a call needs more (a population beyond that, or a wider evaluate).
struct estk_ctx {
  int device;
  int sm_count;
  int cc_major, cc_minor;
  int max_grid;            // sm_count * 8: upper bound on any persistent grid
  int64_t members;         // capacity of cvals / counters / sort_ws, in members
  int64_t eval_floats;     // capacity of eval_partial, in floats
  int64_t slab_floats;     // capacity of eval_slab, in floats (0 until a streamed evaluate needs it)
  float* cvals;            // [members] blended centred ranks (fp32)
  float* partial;          // [max_grid * 1024] split-over-pairs partial sums
  float* eval_partial;     // [eval_floats] loss partials of the evaluate kernels
  float* eval_slab;        // [slab_floats] per-CTA activations of the streamed fp32 evaluate
  unsigned int* counters;  // [kCtxTicketSlots + members]: kernel tickets, then self-resetting arrival counters
  void* sort_ws;           // estk_sort::workspace_bytes(members, 4, max_grid) bytes: radix-sort buffers
  double* scalars;         // [8] small fp64 scratch (||archive||_F, ...)
  void* retired[kCtxMaxRetired];  // buffers replaced by growth, freed at estk_ctx_destroy (earlier graphs use them)
  int n_retired;
};
static const int kEvalMaxChunks = 64;   // the tensor-core evaluate writes up to 2 * kEvalMaxChunks partials per member
static const int64_t kCtxInitialMembers = 32768;
// counters[0 .. kCtxTicketSlots): last-CTA tickets at fixed slots; the per-member counters follow
static const int kCtxTicketSlots = 8;
static const int kTicketClampAdam = 0;
static const int kTicketTrackBest = 1;
static inline unsigned int* estk_member_counters(estk_ctx* c) { return c->counters + kCtxTicketSlots; }

// Grows the context workspace to at least `members` members (cvals, arrival counters, sort buffers),
// `eval_floats` evaluate partials and `slab_floats` activation-slab floats; no-op when it is large
// enough.  Growth allocates new buffers and waits on `stream` for their zero-filled counters; the old
// buffers stay allocated until estk_ctx_destroy (graphs captured before keep working), and stay in use
// if the allocation fails (ESTK_ERR_NOMEM).
// Refused with ESTK_ERR_NOMEM while `stream` is being captured into a CUDA graph.
int estk_ctx_reserve(estk_ctx* c, int64_t members, int64_t eval_floats, cudaStream_t stream, const char* who,
                     int64_t slab_floats = 0);

// ---------------------------------------------------------------- evaluate back ends
// estk_eval_mlp and estk_eval_conv_vbn check their arguments once, then hand the call to the
// kernel file of the requested precision.  A centre call (offsets == NULL) arrives with table =
// theta, pairs = 1, sigma = 0 and no minus outputs; buffers the precision does not read are null.
struct EvalMlpCall {
  estk_mlp_desc desc;
  int precision;  // ESTK_PREC_*
  const float* theta;
  const uint16_t* theta16;
  const float* table;
  const uint16_t* table16;
  const int64_t* offsets;
  const int32_t* order;
  int pairs;
  float sigma;
  const float* obs;
  const float* target;
  int B;
  float* ret_plus;
  float* ret_minus;
  float* bc_plus;
  float* bc_minus;
  int bc_obs, bc_dim;
  float* centre_out;
};
int eval_mlp_tc(estk_ctx* ctx, const EvalMlpCall& c, cudaStream_t stream);     // estk_eval_mlp_tc.cu
// ESTK_PREC_F16_ANY on a shape the cluster kernel does not serve (estk_eval_mlp_tc_stream.cu); the
// shapes it serves: every valid desc, B >= 1 (else 0 and the reason in *why)
int eval_mlp_tc_stream(estk_ctx* ctx, const EvalMlpCall& c, cudaStream_t stream);
int eval_mlp_tc_stream_supported(const estk_mlp_desc& d, int B, const char** why);

struct EvalConvCall {
  int A, R, B;  // n_actions, ref_batch, batch
  const float* theta;
  const float* table;
  const uint16_t* table16;
  const int64_t* offsets;
  const int32_t* order;
  int pairs;
  float sigma;
  const float* xref;
  const float* obs;
  const float* target;
  float* ret_plus;
  float* ret_minus;
  void* scratch;
};
int64_t eval_conv_tc_scratch_per_cta(int R, int B);                              // estk_eval_conv_tc.cu
int eval_conv_tc(estk_ctx* ctx, const EvalConvCall& c, cudaStream_t stream);

// ---------------------------------------------------------------- hashing
// splitmix64 finaliser; must stay in lock-step with oracle/es_oracle.py:mix64
// and estorch_b200/noise.py.
__host__ __device__ __forceinline__ uint64_t estk_mix64(uint64_t z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
#define ESTK_GEN_MUL 0xD1342543DE82EF95ull

// ---------------------------------------------------------------- loads
#ifdef __CUDACC__
// streaming 128-bit read of the noise table: read-only path, do not pollute L1
// (every byte is used exactly once per CTA); default L2 policy on purpose --
// table rows of one generation overlap and are re-read by other CTAs.
__device__ __forceinline__ float4 ld_noise4(const float4* p) {
  float4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p));
  return v;
}
// the same for the fp16 copy of the table: 8 values per 128-bit load
__device__ __forceinline__ uint4 ld_noise4h(const uint4* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}
// d = a * b + c, element-wise (two IEEE fp32 fmas)
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
  return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}
__device__ __forceinline__ float ld_noise1(const float* p) {
  float v;
  asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ int warp_sum_i(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
#endif
