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

// ---------------------------------------------------------------- context
struct estk_ctx {
  int device;
  int sm_count;
  int cc_major, cc_minor;
  int max_grid;            // sm_count * 8: upper bound on any persistent grid
  float* cvals;            // [ESTK_MAX_POPULATION] blended centred ranks (fp32)
  float* partial;          // [max_grid * 1024] split-over-pairs partial sums
  float* eval_partial;     // [ESTK_MAX_POPULATION * 2 * kEvalMaxChunks] loss partials
  unsigned int* counters;  // [ESTK_MAX_POPULATION + 8] self-resetting arrival counters (+ kernel tickets)
  double* scalars;         // [8] small fp64 scratch (||archive||_F, ...)
};
static const int kEvalMaxChunks = 64;   // the tensor-core evaluate writes up to 2 * kEvalMaxChunks partials per member

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
