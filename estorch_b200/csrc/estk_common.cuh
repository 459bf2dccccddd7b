// estk_common.cuh -- shared host/device helpers for libestk (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <algorithm>
#include <climits>
#include <type_traits>
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

// ---------------------------------------------------------------- compile-time value lists
// The values a kernel template parameter is instantiated over.  estk_dispatch(list, v, f) calls the generic
// lambda f with std::integral_constant<int, V> for the V of the list that equals v, and with the first value
// of the list (the default) when none does.  f is instantiated for every value of its list, so a kernel with
// two such parameters nests two dispatches over the two lists, and the instantiations are exactly their product.
template <int... V> struct EstkValues {};
template <int... V> __host__ __device__ constexpr bool estk_in(EstkValues<V...>, int v) { return ((v == V) || ...); }
template <int D, int... V, class F> auto estk_dispatch(EstkValues<D, V...>, int v, F&& f) {
  decltype(f(std::integral_constant<int, D>{})) r{};
  const bool hit = ((v == V ? (r = f(std::integral_constant<int, V>{}), true) : false) || ...);
  return hit ? r : f(std::integral_constant<int, D>{});
}
// bits 0-7 of estk_mlp_desc.activation: the hidden kinds (ReLU, the default, first) and the recurrent cells
using EstkHiddenKinds = EstkValues<ESTK_ACT_RELU, ESTK_ACT_TANH, ESTK_ACT_ELU, ESTK_ACT_SILU, ESTK_ACT_LEAKY_RELU>;
using EstkCells = EstkValues<ESTK_CELL_GRU, ESTK_CELL_LSTM>;
// bits 8-23 of a dense MLP code with a return (output activation | loss), and the output bits alone of an
// ESTK_ACTIONS code (an MLP or a recurrent cell step)
using EstkDenseOutLoss = EstkValues<0, ESTK_ACT_OUT_TANH, ESTK_LOSS_XENT, ESTK_LOSS_ACCURACY>;
using EstkActionOutputs = EstkValues<0, ESTK_ACT_OUT_TANH>;

// estk_mlp_desc.activation: the forty defined codes (each hidden kind of EstkHiddenKinds and each recurrent
// cell of EstkCells x output identity / Tanh with the squared error, x identity output with the cross-entropy,
// and x output identity / Tanh with ESTK_ACTIONS; each hidden kind, not a cell, x identity output with the
// accuracy)
static inline bool estk_act_valid(int a) {
  const int h = a & 0xff, rest = a & ~0xff;
  const bool actions = rest == ESTK_ACTIONS || rest == (ESTK_ACT_OUT_TANH | ESTK_ACTIONS);
  const bool cell = estk_in(EstkCells{}, h);
  const bool known = estk_in(EstkHiddenKinds{}, h) || cell;
  return known && (rest == 0 || rest == ESTK_ACT_OUT_TANH || rest == ESTK_LOSS_XENT || actions ||
                   (rest == ESTK_LOSS_ACCURACY && !cell));
}
// the loss field is ESTK_LOSS_ACCURACY: the count of correct rows needs B < 2^24 to stay exact in fp32
static inline bool estk_loss_accuracy(int code) { return (code & 0xff0000) == ESTK_LOSS_ACCURACY; }
static const int kAccuracyMaxB = (1 << 24) - 1;
// The estk_eval_mlp back end of an activation code: n_conv != 0 in bits 24-31 the convolutional evaluate;
// a defined code whose loss field is ESTK_ACTIONS (no return, the outputs themselves) one step of the MLP or
// of the recurrent cell in bits 0-7; a defined recurrent cell code with a return the sequence evaluate;
// anything else the dense MLP evaluate, which refuses an undefined code.
enum EvalRoute { kRouteDense, kRouteCnn, kRouteActions, kRouteActionsCell, kRouteSequence };
static inline EvalRoute estk_eval_route(int a) {
  if ((a >> 24) & 0xff) return kRouteCnn;
  if (!estk_act_valid(a)) return kRouteDense;
  const bool cell = estk_in(EstkCells{}, a & 0xff);
  if ((a & 0xff0000) == ESTK_ACTIONS) return cell ? kRouteActionsCell : kRouteActions;
  return cell ? kRouteSequence : kRouteDense;
}
// The output head of a code with a return, a compile-time parameter of the sequence and convolutional
// evaluates: identity, tanhf, or the logits of the cross-entropy (which takes precedence over the Tanh bit)
// or of the accuracy.  kHeadAct | kHeadIdentity or kHeadTanh: the act variant of the convolutional kernel
// (estk_act_cnn), which writes the outputs instead of scoring them.
constexpr int kHeadIdentity = 0, kHeadTanh = 1, kHeadXent = 2, kHeadAccuracy = 3, kHeadAct = 4;
static inline int estk_head(int code) {
  return estk_loss_accuracy(code) ? kHeadAccuracy : (code & ESTK_LOSS_XENT) ? kHeadXent
       : (code & ESTK_ACT_OUT_TANH) ? kHeadTanh : kHeadIdentity;
}
using EstkSeqHeads = EstkValues<kHeadIdentity, kHeadXent, kHeadTanh>;
using EstkCnnHeads = EstkValues<kHeadIdentity, kHeadXent, kHeadAccuracy, kHeadTanh, kHeadAct | kHeadTanh,
                                kHeadAct | kHeadIdentity>;
// Rows per sign in one work item of the fp32 act kernels (an environment population): B itself up to 2, then
// 4, then 8 -- one instantiation per value of EstkChunkRows.
static inline int estk_chunk_rows(int B) { return B <= 1 ? 1 : B <= 2 ? 2 : B <= 4 ? 4 : 8; }
using EstkChunkRows = EstkValues<1, 2, 4, 8>;

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
  static_assert(estk_in(EstkHiddenKinds{}, H), "undefined hidden activation");
  if constexpr (H == ESTK_ACT_TANH) return tanhf(y);
  else if constexpr (H == ESTK_ACT_ELU) return y > 0.f ? y : expm1f(y);
  else if constexpr (H == ESTK_ACT_SILU) {
    const float d = 1.0f + expf(-y);
    return CALL_FREE_DIV ? estk_div_rn_ge1(y, d) : __fdiv_rn(y, d);
  }
  else if constexpr (H == ESTK_ACT_LEAKY_RELU) return y > 0.f ? y : y * 0.01f;
  else return fmaxf(y, 0.f);
}

// the recurrent cells' s(v) = 1.0f / (1.0f + expf(-v)) with an IEEE divide (estk.h); the step and the
// sequence kernels share it, so their outputs are the same bits
__device__ __forceinline__ float estk_sigmoid_rn(float v) { return __fdiv_rn(1.f, 1.f + expf(-v)); }
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

#ifdef __CUDACC__
// The launch of an fp32 evaluate whose per-item activations live in shared memory when they fit, else in a
// per-CTA slab of the context workspace (the same kernel code with slab = true, P::slab pointing there).
struct SlabLaunch {
  bool slab;                   // the activations are in the slab
  int64_t items;               // work items; in shared memory each has its own CTA
  size_t smem_shared;          // dynamic shared memory of the shared-memory kernel
  size_t smem_slab;            // ... and of the slab kernel
  int64_t slab_per_cta;        // slab floats of one CTA
  int64_t members, eval_floats;  // estk_ctx_reserve's; both 0: the call reserves on the slab path only
  int64_t slab_cap;            // > 0: the grid's slab stays within this many floats, down to one CTA
};
// The slab grid is persistent: the resident CTAs (by the occupancy of the slab kernel), at most `items`, and
// at most slab_cap / slab_per_cta.  `bind` runs after the reservation, so it can take workspace pointers.
template <class P, class Bind>
int estk_launch_eval(estk_ctx* ctx, void (*shared_kern)(P), void (*slab_kern)(P), P& p, const SlabLaunch& l,
                     int threads, cudaStream_t stream, const char* who, Bind bind) {
  void (*const kern)(P) = l.slab ? slab_kern : shared_kern;
  const size_t smem = l.slab ? l.smem_slab : l.smem_shared;
  ESTK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int64_t grid = l.items < INT_MAX ? l.items : INT_MAX;
  if (l.slab) {
    int per_sm = 0;
    ESTK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, threads, smem));
    grid = std::min<int64_t>(l.items, (int64_t)ctx->sm_count * std::max(per_sm, 1));
    if (l.slab_cap > 0) grid = std::min<int64_t>(grid, std::max<int64_t>(1, l.slab_cap / l.slab_per_cta));
  }
  if (l.members || l.eval_floats || l.slab) {
    const int rc = estk_ctx_reserve(ctx, l.members, l.eval_floats, stream, who, l.slab ? grid * l.slab_per_cta : 0);
    if (rc) return rc;
  }
  p.slab = l.slab ? ctx->eval_slab : nullptr;
  bind();
  kern<<<(int)grid, threads, smem, stream>>>(p);
  ESTK_CUDA(cudaGetLastError());
  return ESTK_OK;
}
#endif

// ---------------------------------------------------------------- evaluate back ends
// estk_eval_mlp checks the precision code, builds this record once and hands it to the back end of the
// activation code (estk_eval_route), which makes its own argument checks.  A centre call (offsets == NULL)
// carries pairs = 1, sigma = 0 and null table, table16, order and minus outputs; centre_out is carried as
// passed, so that every back end can refuse it on a centre call.  The dense MLP evaluate then puts theta
// (and theta16) in place of the table and nulls the 16-bit buffers its precision does not read.
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
// the first checks of both ESTK_ACTIONS back ends: fp32 only, the pointers, the bc layout, no
// centre_return_out (target and the returns are not part of the call; estk_eval_mlp_act.cu)
int eval_actions_check(estk_ctx* ctx, const EvalMlpCall& c);
// the checks of both back ends that return a loss (the sequence and the convolutional evaluate), in two
// groups so that each back end's own ESTK_ERR_UNSUPPORTED checks can run between them (estk_eval_rnn_seq.cu):
// eval_returns_supported: fp32 only, no centre_return_out (ESTK_ERR_UNSUPPORTED);
// eval_returns_check: the pointers, the bc layout, B and pairs (ESTK_ERR_INVALID)
int eval_returns_supported(const EvalMlpCall& c, const char* who);
int eval_returns_check(estk_ctx* ctx, const EvalMlpCall& c, const char* who);
// kRouteActions: eval_actions_check, its own checks, then the act-mode kernel (estk_eval_mlp_act.cu)
int eval_mlp_actions(estk_ctx* ctx, const EvalMlpCall& c, cudaStream_t stream);
// kRouteActionsCell: eval_actions_check, then one step of the cell + head kernel (estk_act_rnn.cu)
int eval_rnn_actions(estk_ctx* ctx, const EvalMlpCall& c, cudaStream_t stream);
// kRouteSequence: its own argument checks, then the sequence evaluate over obs [B][T][in] (estk_eval_rnn_seq.cu)
int eval_rnn_sequence(estk_ctx* ctx, const EvalMlpCall& c, cudaStream_t stream);
// kRouteCnn: its own argument checks, then the convolutional evaluate over obs [B][c][h][w] (estk_eval_cnn.cu)
int eval_cnn(estk_ctx* ctx, const EvalMlpCall& c, cudaStream_t stream);
// The layers of a packed convolutional descriptor (include/estk.h): layer l maps [cin][hin][win] to
// [cout][ho][wo] with K = cin*k*k taps per output, its weight [cout][K] then bias [cout] at wbase (a Linear is
// the 1x1 convolution of its flattened input); maxact the largest layer output per image.
// eval_cnn_parse (estk_eval_cnn.cu) fills it by the fp32 route's rules; every malformed field is ESTK_ERR_INVALID.
struct EstkCnnLayer {
  int cin, hin, win, cout, k, s, pad, ho, wo, K;
  int64_t wbase;
};
struct EstkCnnShape {
  EstkCnnLayer layer[ESTK_MAX_LAYERS];
  int n_layers, in_size, out, maxact;
};
int eval_cnn_parse(const estk_mlp_desc& d, int n_conv, EstkCnnShape& s, const char* who);
// The activation-code checks of both convolutional routes (estk_eval_cnn.cu): n_conv in 1..7 and a defined code
// (ESTK_ERR_INVALID), and a dense code with a return -- ESTK_ACTIONS and the recurrent cells are `route_rc`; then
// B < 2^24 with the accuracy (ESTK_ERR_INVALID)
int eval_cnn_code_check(int code, int route_rc, const char* who);
int eval_cnn_batch_check(int code, int B, const char* who);
// ESTK_PREC_F16_ANY on a shape the cluster kernel does not serve (estk_eval_mlp_tc_stream.cu); the
// shapes it serves: every valid desc, B >= 1 (else 0 and the reason in *why)
int eval_mlp_tc_stream(estk_ctx* ctx, const EvalMlpCall& c, cudaStream_t stream);
int eval_mlp_tc_stream_supported(const estk_mlp_desc& d, int B, const char** why);

// estk_eval_conv_vbn's arguments as passed (a centre call included), for both of its paths
struct EvalConvCall {
  int precision;  // ESTK_PREC_*
  int A, R, B;    // n_actions (with ESTK_ACTIONS: the whole n_actions | ESTK_ACTIONS code), ref_batch, batch
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
  int64_t scratch_bytes;
};
int64_t eval_conv_tc_scratch_per_cta(int R, int B);                              // estk_eval_conv_tc.cu
int eval_conv_tc(estk_ctx* ctx, const EvalConvCall& c, cudaStream_t stream);
// estk_eval_conv_vbn with n_actions | ESTK_ACTIONS: its own argument checks, then the stats and / or act
// kernels (estk_act_conv.cu); target is not part of the call, scratch holds the per-member VBN stats
int eval_conv_actions(estk_ctx* ctx, const EvalConvCall& c, cudaStream_t stream);

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
#include <cuda_fp16.h>
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
__device__ __forceinline__ float ld_noise1h(const uint16_t* p) {
  unsigned short v;
  asm volatile("ld.global.nc.L1::no_allocate.u16 %0, [%1];" : "=h"(v) : "l"(p));
  return __half2float(__ushort_as_half(v));
}

// One pair's noise row: the fp32 table, its exact fp16 copy, or theta itself for the centre (sigma 0).
// A kernel that reads the fp32 table only passes table16 = nullptr, and the fp16 branch folds away.
struct NoiseRow {
  const float* t32;
  const uint16_t* t16;
  __device__ __forceinline__ float operator()(int64_t i) const { return t16 ? ld_noise1h(t16 + i) : ld_noise1(t32 + i); }
};
__device__ __forceinline__ NoiseRow noise_row(const float* theta, const float* table, const uint16_t* table16,
                                              const int64_t* offsets, int j) {
  if (offsets == nullptr) return NoiseRow{theta, nullptr};
  const int64_t toff = offsets[j];
  return table16 ? NoiseRow{nullptr, table16 + toff} : NoiseRow{table + toff, nullptr};
}
// Parameter idx of both members of a pair: W+ = theta + (sigma*t) and W- = theta - (sigma*t), each with the
// evaluate's two roundings, so W- has the bits of theta + (-sigma)*t (estk.h)
__device__ __forceinline__ void estk_form_pm(const float* theta, const NoiseRow& row, float sigma, int64_t idx,
                                             float& wp, float& wm) {
  const float th = __ldg(theta + idx);
  const float ep = __fmul_rn(sigma, row(idx));
  wp = __fadd_rn(th, ep);
  wm = __fsub_rn(th, ep);
}
// ... and of one member, for a thread that serves one sign
__device__ __forceinline__ float estk_form_sign(const float* theta, const NoiseRow& row, float sigma, int64_t idx,
                                                bool minus) {
  const float th = __ldg(theta + idx);
  const float ep = __fmul_rn(sigma, row(idx));
  return minus ? __fsub_rn(th, ep) : __fadd_rn(th, ep);
}

// The return of a pair whose loss is split over `items` work items (CTAs, or chunks of a persistent CTA).
// part = [2][n] partials of the pair (+ then -); each is stored and __threadfence'd by its writer before a
// barrier, after which one thread of the work item arrives on the pair's counter.  The last arrival finishes:
// a fence that orders its reads of the other work items' partials, the in-order fold of each sign (include/
// estk.h states it: the bits do not depend on the schedule), ret = -(sum / denom), and the counter back to 0
// for the next launch.  The finish is a macro, not a function: the fold loop then stays the kernel's own loop,
// which nvcc unrolls as it did before the finish was shared (an inlined function's loop is unrolled
// differently, and the kernel's SASS would change).
__device__ __forceinline__ bool estk_pair_arrive(unsigned int* counter, int items) {
  return atomicAdd(counter, 1u) == (unsigned int)items - 1;
}
#define ESTK_PAIR_FINISH(part, n, denom, ret_plus, ret_minus, j, counter)                                   \
  do {                                                                                                      \
    __threadfence();                                                                                        \
    const float* const pf_ = (part);                                                                        \
    float sp_ = 0.f, sm_ = 0.f;                                                                             \
    for (int i_ = 0; i_ < (n); ++i_) { sp_ += __ldcg(pf_ + i_); sm_ += __ldcg(pf_ + (n) + i_); }          \
    const float d_ = (denom);                                                                               \
    (ret_plus)[j] = -(sp_ / d_);                                                                            \
    if (ret_minus) (ret_minus)[j] = -(sm_ / d_);                                                            \
    *(counter) = 0u;                                                                                        \
  } while (0)
// The order of torch.argmax on (value, index) pairs: a NaN is above every number (the lower index wins between
// two NaNs) and the lower index wins a tie.  It is a total order, so folding the pairs of a row in any order
// and any grouping, from (-INFINITY, INT_MAX), leaves the first index of the maximum (ESTK_LOSS_ACCURACY).
__device__ __forceinline__ void estk_argmax_fold(float& m, int& i, float v, int k) {
  const bool better = v != v ? (m == m || k < i) : (m == m && (v > m || (v == m && k < i)));
  if (better) { m = v; i = k; }
}
// The loss of one row of an fp32 evaluate's row pass: the outputs y(0 .. C) (a loader of the row's columns from
// shared memory or the slab) against the target row t[0 .. C), in column order.  kHeadXent: the cross-entropy
// m + log sum exp(y - m) times sum t, minus sum t*y; any other head: the squared error sum (y - t)^2.  Only
// where the kernel keeps its SASS: the dense and streamed MLP kernels' accuracy and the convolutional kernel's
// scores are their own lines (with this helper inlined, their registers are allocated differently).
template <int HEAD, class Y>
__device__ __forceinline__ float estk_row_loss(Y y, const float* t, int C) {
  if constexpr (HEAD == kHeadXent) {
    float m = -INFINITY;
    for (int c = 0; c < C; ++c) m = fmaxf(m, y(c));
    float s = 0.f, st = 0.f, sty = 0.f;
    for (int c = 0; c < C; ++c) {
      const float v = y(c), tv = __ldg(t + c);
      s += expf(v - m);
      st += tv;
      sty = fmaf(tv, v, sty);
    }
    return fmaf(m + logf(s), st, -sty);
  } else {
    float s = 0.f;
    for (int c = 0; c < C; ++c) {
      const float d = y(c) - __ldg(t + c);
      s = fmaf(d, d, s);
    }
    return s;
  }
}
// The fold across the four lanes of a quad (lane distance 1, then 2): every lane ends with the quad's result.
// All 32 lanes of the warp take part.
__device__ __forceinline__ void estk_argmax_quad(float& m, int& i) {
#pragma unroll
  for (int o = 1; o <= 2; o <<= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, m, o);
    const int oi = __shfl_xor_sync(0xffffffffu, i, o);
    estk_argmax_fold(m, i, om, oi);
  }
}
// The label of a target row t[0..C) for the four lanes of a quad (q = lane & 3): lane q folds its quarter of the
// columns, four loads in flight; every lane returns the first index of the row's maximum.  C = 0 reads nothing
// (a row past the batch).
__device__ __forceinline__ int estk_quad_label(const float* t, int C, int q) {
  const int qs = (C + 3) / 4, c1 = min(C, (q + 1) * qs);
  float m = -INFINITY;
  int i = INT_MAX;
#pragma unroll 4
  for (int c = q * qs; c < c1; ++c) estk_argmax_fold(m, i, __ldg(t + c), c);
  estk_argmax_quad(m, i);
  return i;
}
__device__ __forceinline__ int warp_sum_i(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// One step of Welford's mean / variance update for the n-th sample y (inv = 1.f / n, correctly rounded):
// d = y - mean, mean += d * inv, m2 += d * (y - mean); the unbiased variance is m2 / (n - 1).  Where every y
// is the same, d is 0 from the second sample on and the variance is exactly 0.
__device__ __forceinline__ void welford_add(float y, float inv, float& mean, float& m2) {
  const float d = y - mean;
  mean = fmaf(d, inv, mean);
  m2 = fmaf(d, y - mean, m2);
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
