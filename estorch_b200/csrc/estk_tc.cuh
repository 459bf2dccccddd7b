// estk_tc.cuh -- raw PTX wrappers shared by the tensor-core evaluate kernel (sm_90a):
// mbarriers, warpgroup MMA (wgmma) and its shared-memory descriptors, the 128B-swizzle address
// map and the 16-bit packing conversions.
#pragma once
#include "estk_common.cuh"
#include <cuda_bf16.h>
#include <cuda_fp16.h>

namespace {

constexpr int kMaxW = 512;            // max layer width (K and N) of the tensor-core path
constexpr int kBlockK = 64;           // 16-bit elements per 128-byte swizzle row

// ------------------------------------------------------------------ PTX helpers
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// generic-proxy st.shared -> visible to the async proxy (wgmma reads of smem)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ uint4 ld_noise4u(const uint4* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}

// wgmma shared-memory matrix descriptor: K-major, SWIZZLE_128B, 8-row core-matrix groups 1024 B apart
// (start>>4 [0,14), LBO>>4 [16,30) (unused for swizzled K-major), SBO>>4 [32,46), layout 1 = 128B swizzle [62,64))
__device__ __forceinline__ uint64_t make_sw128_desc(uint32_t smem_addr) {
  return (uint64_t)((smem_addr >> 4) & 0x3FFFu) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}
// byte offset of the 16-byte chunk (row r, chunk c8 of 8 16-bit values) inside a swizzled [rows x 64] tile
__device__ __forceinline__ uint32_t sw128_offset(int r, int c8) {
  return (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + ((c8 ^ (r & 7)) << 4));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator accesses across the asynchronous MMAs
__device__ __forceinline__ void fence_acc(float (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D[64 x 128] (+)= A[64 x 16] * B[128 x 16]^T, both operands K-major in shared memory, fp32 accumulators;
// 16-bit operands: fp16 (F16) or bf16
template <bool F16>
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
#define ESTK_WG_D8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
#define ESTK_WG_ASM(TYPE)                                                                                        \
  asm volatile(                                                                                                  \
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"                                                                \
      "wgmma.mma_async.sync.aligned.m64n128k16.f32." TYPE "." TYPE " "                                           \
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,"  \
      "%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53," \
      "%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n}"                                     \
      : ESTK_WG_D8(0), ESTK_WG_D8(8), ESTK_WG_D8(16), ESTK_WG_D8(24), ESTK_WG_D8(32), ESTK_WG_D8(40),            \
        ESTK_WG_D8(48), ESTK_WG_D8(56)                                                                           \
      : "l"(da), "l"(db), "r"(accumulate))
  if constexpr (F16) ESTK_WG_ASM("f16");
  else ESTK_WG_ASM("bf16");
#undef ESTK_WG_ASM
#undef ESTK_WG_D8
}
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
// relu(x) rounded to bf16, two at a time (ReLU fused into the conversion)
__device__ __forceinline__ uint32_t pack_bf16_relu(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.relu.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
// fp16 variants (saturating: an activation beyond +-65504 becomes +-65504, not inf)
__device__ __forceinline__ uint32_t pack_f16(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
__device__ __forceinline__ uint32_t pack_f16_relu(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.relu.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
__device__ __forceinline__ float2 unpack_f16(uint32_t h2) {
  return __half22float2(*reinterpret_cast<const __half2*>(&h2));
}
template <bool F16> __device__ __forceinline__ uint32_t pack16(float lo, float hi) {
  return F16 ? pack_f16(lo, hi) : pack_bf16(lo, hi);
}
template <bool F16> __device__ __forceinline__ uint32_t pack16_relu(float lo, float hi) {
  return F16 ? pack_f16_relu(lo, hi) : pack_bf16_relu(lo, hi);
}
__device__ __forceinline__ void st_shared_v4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ uint4 ld_shared_v4u(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ float4 ld_shared_v4(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ void named_bar_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
__device__ __forceinline__ void st_shared_u32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}


}  // namespace
