// estk_rank_grad.cu -- kernel 2 of the ES generation: centred-rank transform of
// the P returns, the weighted noise reduction g = (1/P) sum_j w_j T[off_j:off_j+n]
// and the negate/clamp/Adam update, as ONE cooperative persistent launch.
//
// Replaces (reference file:line, /root/reference/estorch/estorch.py):
//   _compute_ranks :22-26, _center_function :15-20, rank_transformation :28-39
//   ES._calculate_grad :174-179 (+ NS :419-425, NSR :542-549, NSRA :640-648)
//   grad scatter + clamp :236-244, optimizer.step() :245 (torch Adam)
//
// Roofline: HBM-bound by the noise stream.  Algorithmic bytes per launch =
// 4*n*pairs_local (each pair's unit-normal row once; the reference's torch.mm
// reads both [eps; -eps] halves, 2x this) + 28*n (theta/m/v read+write, g) + 8*P.
//
// Decomposition: grid = CS column-splits x PS pair-splits, all CTAs co-resident.
//   phase A  bit-exact integer ranks, stable by index on ties: P <= 8192 every warp
//            counts over keys in shared memory (O(P^2) compares total); larger P
//            a grid-wide radix sort (estk_sort.cuh).  Centres in fp64 -> fp32 and
//            blends reward/novelty rows                             -> grid.sync
//   phase B  CTA (cs, ps) owns float4 columns [c0,c1) and sorted pair slots
//            [s0,s1): 128-bit read-only loads, fp32 FMA into registers, 16
//            independent loads in flight per thread (128 KB per SM: the kernel is
//            latency-bound at the L2, bytes in flight set its rate).  With PS == 1 every CTA
//            walks all pairs in the same (offset-sorted) order, so rows that
//            overlap in the table are served from L2 instead of HBM.
//   phase C  PS == 1: epilogue straight from registers.  PS > 1: partial sums
//            to the workspace -> grid.sync -> fixed-order sum -> epilogue
//            (deterministic; no atomics anywhere).
#include "estk_common.cuh"
#include "estk_sort.cuh"
#include <cooperative_groups.h>
#include <cuda_fp16.h>
#include <type_traits>
namespace cg = cooperative_groups;

namespace {

constexpr int kPairTile = 256;  // pair weights / offsets staged per shared-memory refill

struct RankGradParams {
  const float* returns;
  const float* novelty;  // nullable
  float w_rew, w_nov;
  int P, pairs;          // global population / pair count
  int pair_begin, pairs_local;
  const float* table;      // fp32 table, or null when table16 is given
  const uint16_t* table16; // exact fp16 copy of the table (half the bytes, identical values)
  int world;               // > 1: `returns` / `novelty` are laid out rank-major [world][2][pairs/world]
                           // (the all-gather of each rank's (+,-) halves, no re-ordering copy)
  const int64_t* offsets;  // [pairs_local]
  const int32_t* order;    // [pairs_local] nullable
  int64_t n, n4;
  int CS, PS;
  estk_sort::Workspace sort;  // phase A for P > 8192: radix-sort buffers (context workspace)
  float* cvals;    // [P] workspace
  float* partial;  // [PS * n4 * 4] workspace (PS > 1)
  int32_t* ranks_out;
  int32_t* ranks2_out;
  // epilogue
  int fused_adam;       // 1: Adam in place; 0: raw sum -> grad_sum_out
  float* grad_sum_out;  // [n] (fused_adam == 0)
  float* grad_out;      // [n] nullable: g (fused) -- the reference's un-negated estimate
  float* theta;
  float* m;
  float* v;
  estk_state* state;
  estk_adam_desc adam;
  // cross-GPU reduction over peer memory (estk_rank_grad_xr_adam): xr = world size (0: off)
  int xr, xr_rank;
  unsigned char* peer[ESTK_MAX_PEERS];   // every rank's workspace as mapped here; [xr_rank] is this GPU's own
};

// Layout of a cross-GPU workspace (bytes).  Flags first, then the two gradient images.
constexpr int64_t kXrEpochOff = 0;        // uint32: launches completed by the owner (advanced by the kernel itself)
constexpr int64_t kXrCtaCountOff = 128;   // uint32: CTAs of the owner that reached the current barrier
constexpr int64_t kXrArriveOff = 256;     // uint32 arrive[ESTK_MAX_PEERS]: slot q is written by rank q only
constexpr int64_t kXrDataOff = 4096;      // float gsum[nq * 4]  (this rank's partial sum), then float gtot[nq * 4]
__host__ __device__ inline int64_t xr_image_bytes(int64_t n) { return ((n + 3) / 4 * 16 + 255) / 256 * 256; }

struct AdamScalars {
  float lerp_coef, b2, one_minus_b2, bc2_sqrt, eps, neg_step, wd, clamp, inv_div;
  int lerp_big;      // lerp_coef = w = 1 - beta1 (0), or w - 1 with the new gradient as the fma's addend (1)
};

// The launch-wide scalars of adam_elem for Adam step t (t = 0: gradient only, no bias corrections).
// torch.optim.Adam takes 1 - beta1 / 1 - beta2 / -lr/bc1 in fp64 and rounds them to fp32 when they meet
// the fp32 tensors; lerp_ picks its form once from the fp32 weight (ATen lerp: small while |w| < 0.5).
__device__ __forceinline__ AdamScalars adam_scalars(const estk_adam_desc& d, int P, int64_t t) {
  AdamScalars a;
  a.inv_div = (float)P;
  a.clamp = d.clamp;
  const float w = (float)(1.0 - d.beta1);
  a.lerp_big = fabsf(w) >= 0.5f;
  a.lerp_coef = a.lerp_big ? __fsub_rn(w, 1.f) : w;
  a.b2 = (float)d.beta2;
  a.one_minus_b2 = (float)(1.0 - d.beta2);
  a.eps = (float)d.eps;
  a.wd = (float)d.weight_decay;
  a.bc2_sqrt = 1.f; a.neg_step = 0.f;
  if (t > 0) {
    a.bc2_sqrt = (float)sqrt(1.0 - pow(d.beta2, (double)t));
    a.neg_step = (float)(-(d.lr / (1.0 - pow(d.beta1, (double)t))));
  }
  return a;
}

// Order-preserving 32-bit image of a return: -0 maps to +0 (they compare equal), every NaN to 0xffffffff
// (after +inf: numpy's argsort puts NaN last).  image(a) < image(b) <=> a sorts before b.
__device__ __forceinline__ uint32_t rank_image(float v) {
  v = __fadd_rn(v, 0.f);
  const uint32_t b = __float_as_uint(v);
  return v != v ? 0xffffffffu : ((b & 0x80000000u) ? ~b : (b | 0x80000000u));
}

__device__ __forceinline__ float centre(int rank, int P) {
  // estorch.py:17-19 in float64, cast to fp32 at :176
  return (float)((double)rank / (double)(P - 1) - 0.5);
}

// torch.optim.Adam single-tensor update on one element (torch/optim/adam.py:
// add :429, lerp_ :457, mul_/addcmul_ :476, sqrt/div/add_ :543, addcdiv_ :545), operation for
// operation as ATen's vectorised CPU kernels round it: three of them are single fmas there
// (add with alpha: fma(wd, theta, g); lerp_: fma(w, g - m, m), or fma(w - 1, g - m, g) for
// |w| >= 0.5; addcmul_: fma((1 - beta2) g, g, beta2 v)), every other operation is rounded on its
// own (explicit intrinsics: no contraction).  m and v are therefore torch's bits; theta is too
// wherever torch's own sqrt is correctly rounded (__fsqrt_rn always is; torch's CPU sqrt is
// occasionally one ulp off).
__device__ __forceinline__ void adam_elem(float sum, const AdamScalars& a, float& th, float& m,
                                          float& v, float* g_out) {
  const float g = __fdiv_rn(sum, a.inv_div);  // inv_div holds (float)P
  if (g_out) *g_out = g;
  float gp = -g;                               // estorch.py:239
  if (a.clamp > 0.f) gp = fminf(fmaxf(gp, -a.clamp), a.clamp);  // :243
  if (a.wd != 0.f) gp = __fmaf_rn(a.wd, th, gp);
  m = __fmaf_rn(a.lerp_coef, __fsub_rn(gp, m), a.lerp_big ? gp : m);
  v = __fmaf_rn(__fmul_rn(a.one_minus_b2, gp), gp, __fmul_rn(v, a.b2));
  const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), a.bc2_sqrt), a.eps);
  th = __fadd_rn(th, __fdiv_rn(__fmul_rn(a.neg_step, m), denom));
}

__device__ __forceinline__ void epilogue(const RankGradParams& p, const AdamScalars& a,
                                         int64_t col4, float4 s, bool raw) {
  const int64_t k = col4 * 4;
  const bool full = (k + 3 < p.n);
  if (raw) {
    if (full) {
      reinterpret_cast<float4*>(p.grad_sum_out)[col4] = s;
    } else {
      const float sv[4] = {s.x, s.y, s.z, s.w};
      for (int e = 0; e < 4 && k + e < p.n; ++e) p.grad_sum_out[k + e] = sv[e];
    }
    return;
  }
  float sv[4] = {s.x, s.y, s.z, s.w};
  float th[4], mm[4], vv[4], gg[4];
  if (full) {
    const float4 t4 = reinterpret_cast<const float4*>(p.theta)[col4];
    const float4 m4 = reinterpret_cast<const float4*>(p.m)[col4];
    const float4 v4 = reinterpret_cast<const float4*>(p.v)[col4];
    th[0] = t4.x; th[1] = t4.y; th[2] = t4.z; th[3] = t4.w;
    mm[0] = m4.x; mm[1] = m4.y; mm[2] = m4.z; mm[3] = m4.w;
    vv[0] = v4.x; vv[1] = v4.y; vv[2] = v4.z; vv[3] = v4.w;
#pragma unroll
    for (int e = 0; e < 4; ++e) adam_elem(sv[e], a, th[e], mm[e], vv[e], &gg[e]);
    reinterpret_cast<float4*>(p.theta)[col4] = make_float4(th[0], th[1], th[2], th[3]);
    reinterpret_cast<float4*>(p.m)[col4] = make_float4(mm[0], mm[1], mm[2], mm[3]);
    reinterpret_cast<float4*>(p.v)[col4] = make_float4(vv[0], vv[1], vv[2], vv[3]);
    if (p.grad_out) reinterpret_cast<float4*>(p.grad_out)[col4] = make_float4(gg[0], gg[1], gg[2], gg[3]);
  } else {
    for (int e = 0; e < 4 && k + e < p.n; ++e) {
      float t = p.theta[k + e], m_ = p.m[k + e], v_ = p.v[k + e], g_;
      adam_elem(sv[e], a, t, m_, v_, &g_);
      p.theta[k + e] = t; p.m[k + e] = m_; p.v[k + e] = v_;
      if (p.grad_out) p.grad_out[k + e] = g_;
    }
  }
}

// Phase X of rank_grad_kernel (estk_rank_grad_xr_adam): this GPU's partial gradient sum is complete in its own
// workspace; sum over the GPUs through peer memory, then apply the (replicated) Adam step.  Inlined into the XR
// instantiations only (out of line it copied the 400-byte parameter block to local memory in every thread: 9 us).
__device__ __forceinline__ void xr_phase(const RankGradParams& p, const AdamScalars& adam, int kThreads) {
  const int tid = threadIdx.x;
  const int W = p.xr, me = p.xr_rank;
  unsigned char* mine = p.peer[me];
  const uint32_t epoch = *reinterpret_cast<volatile const uint32_t*>(mine + kXrEpochOff);   // block 0 advances it
  const int64_t img = xr_image_bytes(p.n);                                                  // after the LAST grid.sync
  const int64_t nq = (p.n + 3) / 4;
  const int64_t gstride = (int64_t)gridDim.x * kThreads;
  // A barrier over the GPUs (and over the CTAs of this one), called by every thread of the grid.  `value` only
  // grows (two per launch); slot q of a rank's arrive[] is written by rank q alone.  No grid.sync: every CTA
  // counts itself in, the last one tells the peers, and every CTA watches this GPU's own arrive[] words.
  uint32_t* cta_count = reinterpret_cast<uint32_t*>(mine + kXrCtaCountOff);
  auto gpu_barrier = [&](uint32_t value, bool remote_stores) {
    __syncthreads();                 // this CTA's stores happen-before thread 0's fence, which is cumulative over them
    if (tid == 0) {
      // partial sums in this GPU's own memory are visible to NVLink readers once they are in its L2 (gpu scope);
      // stores INTO the peers' memory must have been performed there (system scope)
      if (remote_stores) __threadfence_system(); else __threadfence();
      if (atomicAdd(cta_count, 1u) == gridDim.x - 1) {      // every CTA of this GPU is past its stores
        *reinterpret_cast<volatile uint32_t*>(cta_count) = 0u;   // re-arm (nobody counts again before the peers answer)
        __threadfence_system();                               // release: fence, then relaxed flag stores
        for (int q = 0; q < W; ++q) {
          uint32_t* there = reinterpret_cast<uint32_t*>(p.peer[q] + kXrArriveOff) + me;
          asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(there), "r"(value) : "memory");
        }
      }
    }
    if (tid < W) {
      const uint32_t* here = reinterpret_cast<const uint32_t*>(mine + kXrArriveOff) + tid;
      uint32_t seen;
      const long long t0 = clock64();
      for (;;) {
        asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(seen) : "l"(here) : "memory");
        if ((int32_t)(seen - value) >= 0) break;
        if (clock64() - t0 > (20ll << 30)) __trap();   // ~10 s: a peer never arrived; fail instead of hanging the GPU
      }
      __threadfence_system();        // acquire side, once
    }
    __syncthreads();
  };
  gpu_barrier(2 * epoch + 1, false);
  // reduce-scatter + all-gather of slice `me`: float4 columns [q0, q1); the sum runs in rank order on every GPU
  {
    const int64_t q0 = (int64_t)me * nq / W, q1 = (int64_t)(me + 1) * nq / W;
    for (int64_t c = q0 + (int64_t)blockIdx.x * kThreads + tid; c < q1; c += gstride) {
      float4 sum = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int qb = 0; qb < W; qb += 4) {          // four loads over NVLink in flight per thread
        float4 t[4];
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (qb + e < W) {
            const float4* src = reinterpret_cast<const float4*>(p.peer[qb + e] + kXrDataOff) + c;
            asm volatile("ld.volatile.global.v4.f32 {%0,%1,%2,%3}, [%4];"
                         : "=f"(t[e].x), "=f"(t[e].y), "=f"(t[e].z), "=f"(t[e].w) : "l"(src) : "memory");
          }
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (qb + e < W) {
            if (qb + e == 0) { sum = t[0]; continue; }
            sum.x = __fadd_rn(sum.x, t[e].x); sum.y = __fadd_rn(sum.y, t[e].y);
            sum.z = __fadd_rn(sum.z, t[e].z); sum.w = __fadd_rn(sum.w, t[e].w);
          }
      }
      for (int q = 0; q < W; ++q) reinterpret_cast<float4*>(p.peer[q] + kXrDataOff + img)[c] = sum;
    }
  }
  gpu_barrier(2 * epoch + 2, true);
  {
    const float4* gtot = reinterpret_cast<const float4*>(mine + kXrDataOff + img);
    for (int64_t c = (int64_t)blockIdx.x * kThreads + tid; c < nq; c += gstride)
      epilogue(p, adam, c, __ldcg(gtot + c), false);
  }
  if (blockIdx.x == 0 && tid == 0) *reinterpret_cast<volatile uint32_t*>(mine + kXrEpochOff) = epoch + 1;
}

// Phase A for P > 8192, one column: a stable grid-wide radix sort of (rank_image(value), member) in member
// order, so equal images keep index order; rank[member] = its sorted position (O(P) per pass instead of the
// O(P^2) count).  `second`: blend into cvals (the novelty column).
template <int T>
__device__ __forceinline__ void sort_ranks_body(const float* vals, int32_t* ranks_out, float* cvals, float w_rew, float w_nov,
                                        bool second, int P, int world, void* k0, void* k1, uint32_t* v0,
                                        uint32_t* v1, uint32_t* hist, uint32_t* total, uint32_t* s_sort) {
  cg::grid_group grid = cg::this_grid();
  estk_sort::Workspace ws;
  ws.keys[0] = k0; ws.keys[1] = k1; ws.vals[0] = v0; ws.vals[1] = v1; ws.hist = hist; ws.total = total;
  const int pairs = P / 2;
  const int pl = pairs / max(world, 1);
  auto pos_of = [&](int m) { const int sg = m / pairs, g = m % pairs; return ((g / pl) * 2 + sg) * pl + g % pl; };
  auto load = [&](int m) { return rank_image(__ldg(vals + (world > 1 ? pos_of(m) : m))); };
  const int b = estk_sort::grid_sort<uint32_t, T>(grid, ws, P, 32, load, s_sort);
  const uint32_t* member = b ? v1 : v0;
  for (int s = blockIdx.x * T + threadIdx.x; s < P; s += gridDim.x * T) {
    const int i = (int)__ldcg(member + s);
    if (ranks_out) ranks_out[i] = s;
    if (!second) {
      cvals[i] = centre(s, P);
    } else {
      // estorch.py:645-646; cvals[i] was written by some thread before the sort's grid.syncs
      cvals[i] = __fadd_rn(__fmul_rn(w_rew, __ldcg(cvals + i)), __fmul_rn(w_nov, centre(s, P)));
    }
  }
}

// The 512-thread kernels (up to 128 registers, phase B near the limit) call the sort out of line, with its
// arguments by value, so that none of its state enters phase B's register allocation; the 256-thread kernels
// (80 registers) inline it -- there the call's saved registers would spill instead.
template <int T>
__device__ __noinline__ void sort_ranks_call(const float* vals, int32_t* ranks_out, float* cvals, float w_rew,
                                             float w_nov, bool second, int P, int world, void* k0, void* k1,
                                             uint32_t* v0, uint32_t* v1, uint32_t* hist, uint32_t* total,
                                             uint32_t* s_sort) {
  sort_ranks_body<T>(vals, ranks_out, cvals, w_rew, w_nov, second, P, world, k0, k1, v0, v1, hist, total, s_sort);
}

template <int T>
__device__ __forceinline__ void sort_ranks(const float* vals, int32_t* ranks_out, float* cvals, float w_rew,
                                           float w_nov, bool second, int P, int world, void* k0, void* k1,
                                           uint32_t* v0, uint32_t* v1, uint32_t* hist, uint32_t* total,
                                           uint32_t* s_sort) {
  if constexpr (T == 512)
    sort_ranks_call<T>(vals, ranks_out, cvals, w_rew, w_nov, second, P, world, k0, k1, v0, v1, hist, total, s_sort);
  else
    sort_ranks_body<T>(vals, ranks_out, cvals, w_rew, w_nov, second, P, world, k0, k1, v0, v1, hist, total, s_sort);
}

// SORT: phase A by the grid-wide radix sort (P > 8192) instead of the shared-memory count (P <= 8192)
template <int NC, int T, int LOADS = 8, bool T16 = false, bool XR = false, bool SORT = false>
__global__ void __launch_bounds__(T, T == 256 ? 3 : 1) rank_grad_kernel(const RankGradParams p) {
  constexpr int kThreads = T;
  cg::grid_group grid = cg::this_grid();
  const int tid = threadIdx.x;
  const int lane = tid & 31;
  __shared__ __align__(16) float s_w[kPairTile];
  __shared__ AdamScalars s_adam;
  extern __shared__ __align__(16) unsigned long long s_key_raw[];   // [P] keys, or the sort's scratch (SORT)
  uint64_t* s_key = reinterpret_cast<uint64_t*>(s_key_raw);

  // ---- Adam scalars (read adam_step BEFORE the first grid.sync; block 0
  //      publishes the increment after the last one, so there is no race)
  int64_t adam_t = 0;
  if (p.fused_adam) adam_t = p.state->adam_step + 1;
  if (tid == 0) s_adam = adam_scalars(p.adam, p.P, adam_t);

  // ---- phase A: ranks.  rank_i = #{j: r_j < r_i} + #{j < i: r_j == r_i}
  //      numpy's argsort order (estorch.py:25): NaN sorts last, NaNs among themselves by index.
  {
    const int warps = kThreads >> 5;
    const int gwarp = blockIdx.x * warps + (tid >> 5);
    const int nwarps = gridDim.x * warps;
    // member index <-> position in `returns` (identity on one GPU; rank-major otherwise)
    const int pl = p.pairs / max(p.world, 1);
    auto pos_of = [&](int m) { const int sg = m / p.pairs, g = m % p.pairs; return ((g / pl) * 2 + sg) * pl + g % pl; };
    auto member_of = [&](int q) { const int r = q / (2 * pl), rem = q - r * 2 * pl; return (rem / pl) * p.pairs + r * pl + rem % pl; };
    if constexpr (!SORT) {
      // P <= 8192: every CTA builds one 64-bit key per member in shared memory -- (order-preserving image
      // of the fp32 value) << 32 | member index -- so that rank_i = #{j: key_j < key_i}: one shared-memory
      // load and one 64-bit compare per (i, j), ties and the rank-major index arithmetic folded into the key.
      auto count = [&](const float* vals, int32_t* ranks_out, bool second) {
        __syncthreads();                                     // the previous column's keys are no longer read
        for (int q = tid; q < p.P; q += kThreads)
          s_key[q] = ((uint64_t)rank_image(__ldg(vals + q)) << 32) | (uint32_t)(p.world > 1 ? member_of(q) : q);
        __syncthreads();
        for (int i = gwarp; i < p.P; i += nwarps) {
          const uint64_t ki = s_key[p.world > 1 ? pos_of(i) : i];
          int cnt = 0;
#pragma unroll 4
          for (int j = lane; j < p.P; j += 32) cnt += s_key[j] < ki;
          cnt = warp_sum_i(cnt);
          if (lane == 0) {
            if (ranks_out) ranks_out[i] = cnt;
            if (!second) {
              p.cvals[i] = centre(cnt, p.P);
            } else {
              // estorch.py:645-646  w*c(reward) + (1-w)*c(novelty), fp32, two roundings + add
              p.cvals[i] = __fadd_rn(__fmul_rn(p.w_rew, p.cvals[i]), __fmul_rn(p.w_nov, centre(cnt, p.P)));
            }
          }
        }
      };
      count(p.returns, p.ranks_out, false);
      if (p.novelty) count(p.novelty, p.ranks2_out, true);   // the same lane 0 wrote cvals[i] just above
    } else {
      // P > 8192: a stable grid-wide radix sort (sort_ranks)
      uint32_t* s_sort = reinterpret_cast<uint32_t*>(s_key_raw);
      const estk_sort::Workspace& w = p.sort;
      sort_ranks<kThreads>(p.returns, p.ranks_out, p.cvals, p.w_rew, p.w_nov, false, p.P, p.world, w.keys[0],
                           w.keys[1], w.vals[0], w.vals[1], w.hist, w.total, s_sort);
      if (p.novelty)
        sort_ranks<kThreads>(p.novelty, p.ranks2_out, p.cvals, p.w_rew, p.w_nov, true, p.P, p.world, w.keys[0],
                             w.keys[1], w.vals[0], w.vals[1], w.hist, w.total, s_sort);
      (void)gwarp; (void)nwarps; (void)member_of;
    }
  }
  __threadfence();
  grid.sync();

  // ---- phase B: weighted noise reduction
  const int cs = blockIdx.x % p.CS;
  const int ps = blockIdx.x / p.CS;
  const int64_t c0 = (int64_t)cs * p.n4 / p.CS;
  const int64_t c1 = (int64_t)(cs + 1) * p.n4 / p.CS;
  const int s0 = (int)((int64_t)ps * p.pairs_local / p.PS);
  const int s1 = (int)((int64_t)(ps + 1) * p.pairs_local / p.PS);
  // valid: written before the __syncthreads in grid.sync; read from shared memory where the epilogue
  // needs it, so that none of it is held in registers through phase B
  const AdamScalars& adam = s_adam;
  const bool raw_out = !p.fused_adam || XR;   // phases B / C leave the raw sum in grad_sum_out
  if constexpr (T16) {
    // fp16 table: a 128-bit load carries 8 noise values; same 16 loads in flight per thread, half the
    // bytes per pair row.  Columns are counted in vectors of 8 elements (p.n4 holds ceil(n/8) here).
    // The loop is issue-bound once the bytes are halved (ncu: 60 % issue-active), so it is written for
    // instruction count: one 64-bit add per address (64-bit byte offset of the pair row + this thread's 64-bit
    // column base: any table length), pair offsets / weights fetched four at a time, two fp32 FMAs per instruction
    // (fma.rn.f32x2: each lane an IEEE fma, so the sums are bit-identical to the fp32-table kernel), and
    // the number of live columns of a thread resolved once per pair tile instead of once per load.
    __shared__ __align__(16) uint64_t s_off[kPairTile];   // 64-bit byte offset of each staged pair's row
    const char* tabb = reinterpret_cast<const char*>(p.table16);
    for (int64_t cbase = c0; cbase < c1; cbase += (int64_t)kThreads * NC) {
      int64_t col[NC];
      bool act[NC];
      const char* cb[NC];
      float2 acc[NC][4];
      int na = 0;
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        col[c] = cbase + (int64_t)c * kThreads + tid;
        act[c] = col[c] < c1;       // monotone in c: the live columns of a thread are c < na
        na += act[c] ? 1 : 0;
        cb[c] = tabb + (act[c] ? col[c] : c0) * 16;   // a dead lane of a live warp re-reads column c0 (one sector)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[c][e] = make_float2(0.f, 0.f);
      }
      const int na_w = __reduce_max_sync(0xffffffffu, na);   // warp-uniform: no divergence inside the pair loop
      for (int sbase = s0; sbase < s1; sbase += kPairTile) {
        const int cnt = min(kPairTile, s1 - sbase);
        __syncthreads();
        for (int t = tid; t < cnt; t += kThreads) {
          const int jl = p.order ? p.order[sbase + t] : (sbase + t);
          const int jg = p.pair_begin + jl;
          s_w[t] = __fsub_rn(__ldcg(p.cvals + jg), __ldcg(p.cvals + jg + p.pairs));
          s_off[t] = (uint64_t)p.offsets[jl] * 2;           // byte offset of the row in the fp16 table
        }
        __syncthreads();
        constexpr int U = LOADS / NC;
        static_assert(U % 4 == 0, "pair offsets / weights are fetched four at a time");
        auto row = [](const char* base, uint64_t off) { return reinterpret_cast<const uint4*>(base + off); };
        auto fma8 = [](float2 (&a)[4], float2 w, const uint4& t) {
          a[0] = ffma2(w, __half22float2(*reinterpret_cast<const __half2*>(&t.x)), a[0]);
          a[1] = ffma2(w, __half22float2(*reinterpret_cast<const __half2*>(&t.y)), a[1]);
          a[2] = ffma2(w, __half22float2(*reinterpret_cast<const __half2*>(&t.z)), a[2]);
          a[3] = ffma2(w, __half22float2(*reinterpret_cast<const __half2*>(&t.w)), a[3]);
        };
        auto body = [&](auto na_tag) {
          constexpr int NA = decltype(na_tag)::value;
          int jj = 0;
          for (; jj + U <= cnt; jj += U) {
            uint4 t[U][NA];
#pragma unroll
            for (int q = 0; q < U / 4; ++q) {
              const ulonglong2 o01 = *reinterpret_cast<const ulonglong2*>(s_off + jj + 4 * q);
              const ulonglong2 o23 = *reinterpret_cast<const ulonglong2*>(s_off + jj + 4 * q + 2);
              const uint64_t ov[4] = {o01.x, o01.y, o23.x, o23.y};
#pragma unroll
              for (int e = 0; e < 4; ++e)
#pragma unroll
                for (int c = 0; c < NA; ++c) t[4 * q + e][c] = ld_noise4h(row(cb[c], ov[e]));
            }
            __syncwarp();   // scheduling fence: all U x NA loads are issued before the first one is consumed
                            // (bytes in flight set the rate; without it ptxas interleaves loads and FMAs)
#pragma unroll
            for (int q = 0; q < U / 4; ++q) {
              const float4 w4 = *reinterpret_cast<const float4*>(s_w + jj + 4 * q);
              const float wv[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
              for (int e = 0; e < 4; ++e)
#pragma unroll
                for (int c = 0; c < NA; ++c) fma8(acc[c], make_float2(wv[e], wv[e]), t[4 * q + e][c]);
            }
          }
          for (; jj < cnt; ++jj) {
            const float w = s_w[jj];
#pragma unroll
            for (int c = 0; c < NA; ++c) fma8(acc[c], make_float2(w, w), ld_noise4h(row(cb[c], s_off[jj])));
          }
        };
        static_assert(NC <= 2, "one loop body per possible number of live columns");
        if (na_w == NC) body(std::integral_constant<int, NC>{});
        else if (NC > 1 && na_w == 1) body(std::integral_constant<int, 1>{});
      }
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        if (!act[c]) continue;
        const float4 lo = make_float4(acc[c][0].x, acc[c][0].y, acc[c][1].x, acc[c][1].y);
        const float4 hi = make_float4(acc[c][2].x, acc[c][2].y, acc[c][3].x, acc[c][3].y);
        if (p.PS == 1) {
          epilogue(p, adam, col[c] * 2, lo, raw_out);
          if (col[c] * 8 + 4 < p.n) epilogue(p, adam, col[c] * 2 + 1, hi, raw_out);
        } else {
          float4* part = reinterpret_cast<float4*>(p.partial) + ((int64_t)ps * p.n4 + col[c]) * 2;
          part[0] = lo; part[1] = hi;
        }
      }
    }
  } else {
  // fp32 table: each row as its 32-bit float4 index offsets[j] / 4, exact for every table of at most
  // ESTK_MAX_TABLE_LEN = 2^34 entries (64-bit byte offsets here cost 1.7x the time at n = 1,001,760)
  __shared__ __align__(16) uint32_t s_off4[kPairTile];
  const float4* tab4 = reinterpret_cast<const float4*>(p.table);
  for (int64_t cbase = c0; cbase < c1; cbase += (int64_t)kThreads * NC) {
    int64_t col[NC];
    bool act[NC];
    float4 acc[NC];
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      col[c] = cbase + (int64_t)c * kThreads + tid;
      act[c] = col[c] < c1;
      acc[c] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    for (int sbase = s0; sbase < s1; sbase += kPairTile) {
      const int cnt = min(kPairTile, s1 - sbase);
      __syncthreads();
      for (int t = tid; t < cnt; t += kThreads) {
        const int jl = p.order ? p.order[sbase + t] : (sbase + t);
        const int jg = p.pair_begin + jl;
        // (c_j) * eps_j + (c_{j+pairs}) * (-eps_j)  ==  (c_j - c_{j+pairs}) * eps_j
        s_w[t] = __fsub_rn(__ldcg(p.cvals + jg), __ldcg(p.cvals + jg + p.pairs));
        s_off4[t] = (uint32_t)(p.offsets[jl] >> 2);
      }
      __syncthreads();
      constexpr int U = LOADS / NC;  // LOADS independent 16-byte loads in flight per thread
      int jj = 0;
      for (; jj + U <= cnt; jj += U) {
        float4 t[U][NC];
#pragma unroll
        for (int u = 0; u < U; ++u)
#pragma unroll
          for (int c = 0; c < NC; ++c)
            if (act[c]) t[u][c] = ld_noise4(tab4 + (size_t)s_off4[jj + u] + col[c]);
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const float w = s_w[jj + u];
#pragma unroll
          for (int c = 0; c < NC; ++c)
            if (act[c]) {
              acc[c].x = fmaf(w, t[u][c].x, acc[c].x);
              acc[c].y = fmaf(w, t[u][c].y, acc[c].y);
              acc[c].z = fmaf(w, t[u][c].z, acc[c].z);
              acc[c].w = fmaf(w, t[u][c].w, acc[c].w);
            }
        }
      }
      for (; jj < cnt; ++jj) {
        const float w = s_w[jj];
#pragma unroll
        for (int c = 0; c < NC; ++c)
          if (act[c]) {
            const float4 t = ld_noise4(tab4 + (size_t)s_off4[jj] + col[c]);
            acc[c].x = fmaf(w, t.x, acc[c].x);
            acc[c].y = fmaf(w, t.y, acc[c].y);
            acc[c].z = fmaf(w, t.z, acc[c].z);
            acc[c].w = fmaf(w, t.w, acc[c].w);
          }
      }
    }
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      if (!act[c]) continue;
      if (p.PS == 1) {
        epilogue(p, adam, col[c], acc[c], raw_out);
      } else {
        reinterpret_cast<float4*>(p.partial)[(int64_t)ps * p.n4 + col[c]] = acc[c];
      }
    }
  }
  }

  // ---- phase C: fixed-order sum of the pair-split partials (float4 granularity in both layouts:
  //      the fp16-table path stores two float4 per 8-element vector)
  if (p.PS > 1) {
    __threadfence();
    grid.sync();
    const int64_t nq = T16 ? p.n4 * 2 : p.n4;        // float4 columns per partial row
    const int64_t gstride = (int64_t)gridDim.x * kThreads;
    for (int64_t col4 = (int64_t)blockIdx.x * kThreads + tid; col4 < nq; col4 += gstride) {
      if (col4 * 4 >= p.n) continue;
      float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int q = 0; q < p.PS; ++q) {
        const float4 t = __ldcg(reinterpret_cast<const float4*>(p.partial) + (int64_t)q * nq + col4);
        s.x += t.x; s.y += t.y; s.z += t.z; s.w += t.w;
      }
      epilogue(p, adam, col4, s, raw_out);
    }
  }

  // ---- phase X: sum over the GPUs through peer memory, then the replicated Adam step
  if constexpr (XR) xr_phase(p, adam, kThreads);   // (only the XR instantiations pay for its registers)
  if (p.fused_adam && blockIdx.x == 0 && tid == 0) p.state->adam_step = adam_t;
}

__global__ void __launch_bounds__(256) clamp_adam_kernel(const RankGradParams p, unsigned int* ticket) {
  __shared__ AdamScalars s_adam;
  const bool do_adam = p.theta != nullptr;
  int64_t adam_t = 0;
  if (do_adam) adam_t = p.state->adam_step + 1;
  if (threadIdx.x == 0) s_adam = adam_scalars(p.adam, p.P, adam_t);
  __syncthreads();
  const AdamScalars a = s_adam;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < p.n; k += stride) {
    const float sum = p.grad_sum_out[k];
    if (do_adam) {
      float t = p.theta[k], m_ = p.m[k], v_ = p.v[k], g_;
      adam_elem(sum, a, t, m_, v_, &g_);
      p.theta[k] = t; p.m[k] = m_; p.v[k] = v_;
      if (p.grad_out) p.grad_out[k] = g_;
    } else {
      float gp = -__fdiv_rn(sum, a.inv_div);
      if (a.clamp > 0.f) gp = fminf(fmaxf(gp, -a.clamp), a.clamp);
      p.grad_out[k] = gp;
    }
  }
  // every CTA read adam_step before taking a ticket, so the last one to finish may publish the
  // incremented counter (no CTA can observe it) and re-arm the ticket
  if (do_adam) {
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence();
      if (atomicAdd(ticket, 1u) == gridDim.x - 1) {
        p.state->adam_step = adam_t;
        *ticket = 0u;
      }
    }
  }
}

template <int NC, int T, int LOADS = 8, bool T16 = false, bool XR = false>
int launch_rank_grad(estk_ctx* ctx, RankGradParams& p, cudaStream_t stream) {
  constexpr int kThreads = T;
  int occ = 0;
  constexpr size_t kKeyBytesMax = 64 * 1024;             // P <= 8192 (BASELINE config 3); larger: radix sort
  static bool attr_set[64] = {};                         // per device: one process may drive several GPUs
  const int dev = ctx->device & 63;
  if (!attr_set[dev]) {
    ESTK_CUDA(cudaFuncSetAttribute(rank_grad_kernel<NC, T, LOADS, T16, XR>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)kKeyBytesMax));
    attr_set[dev] = true;
  }
  const bool sort = (size_t)p.P * 8 > kKeyBytesMax;
  const size_t key_bytes = sort ? 0 : (size_t)p.P * 8;
  // the geometry (hence the fp32 summation order) is the count kernel's at P > 8192 as well
  ESTK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, rank_grad_kernel<NC, T, LOADS, T16, XR>, kThreads, key_bytes));
  if (occ < 1) {
    estk_set_error("rank_grad_kernel<%d> cannot be resident", NC);
    return ESTK_ERR_CUDA;
  }
  if (occ > 1024 / kThreads) occ = 1024 / kThreads;  // <= 1024 threads x 8 x 16 B in flight per SM
  if (kThreads == 256 && occ > 3) occ = 3;           // the same geometry (hence the same fp32 sums) with and without XR
  const int gmax = occ * ctx->sm_count;
  const int64_t n4 = p.n4;
  if (n4 >= (int64_t)ctx->sm_count * 512) {
    // enough columns to keep every SM busy without splitting pairs
    p.PS = 1;
    p.CS = gmax;
  } else {
    p.CS = (int)((n4 + kThreads - 1) / kThreads);
    int ps = gmax / p.CS;
    const int ps_cap = (p.pairs_local + 15) / 16;  // >= 16 pair rows per CTA
    if (ps > ps_cap) ps = ps_cap;
    if (ps < 1) ps = 1;
    p.PS = ps;
    if ((int64_t)p.PS * n4 * (T16 ? 8 : 4) > (int64_t)ctx->max_grid * 1024) {
      estk_set_error("rank_grad: partial workspace too small (PS=%d n4=%lld)", p.PS, (long long)n4);
      return ESTK_ERR_NOMEM;
    }
  }
  const int grid = p.CS * p.PS;
  void* args[] = {(void*)&p};
  if (!sort) {
    ESTK_CUDA(cudaLaunchCooperativeKernel((void*)rank_grad_kernel<NC, T, LOADS, T16, XR>, dim3(grid), dim3(kThreads), args,
                                          key_bytes, stream));
    return ESTK_OK;
  }
  constexpr size_t kSortBytes = estk_sort::smem_bytes(kThreads);
  int occ_sort = 0;
  ESTK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_sort, rank_grad_kernel<NC, T, LOADS, T16, XR, true>,
                                                          kThreads, kSortBytes));
  if (occ_sort < occ) {
    estk_set_error("rank_grad_kernel<%d> (sorting ranks): %d CTAs per SM resident, the geometry needs %d", NC,
                   occ_sort, occ);
    return ESTK_ERR_CUDA;
  }
  p.sort = estk_sort::workspace_of(ctx);
  ESTK_CUDA(cudaLaunchCooperativeKernel((void*)rank_grad_kernel<NC, T, LOADS, T16, XR, true>, dim3(grid), dim3(kThreads),
                                        args, kSortBytes, stream));
  return ESTK_OK;
}

// Checks the arguments every rank + gradient launch shares and fills their fields of `p`.
int init_common(RankGradParams& p, estk_ctx* ctx, const float* returns, const float* novelty, float w_rew,
                float w_nov, int P, int world, const float* table, const uint16_t* table16, const int64_t* offsets,
                const int32_t* order, int pair_begin, int pairs_local, int64_t n, int32_t* ranks_out,
                int32_t* ranks2_out, cudaStream_t stream, const char* who) {
  ESTK_CHECK_ARG(ctx && returns && offsets, "%s: null argument", who);
  ESTK_CHECK_ARG((table == nullptr) != (table16 == nullptr), "%s: exactly one of table / table16 must be given", who);
  ESTK_CHECK_ARG(P >= 2 && (P % 2) == 0 && P <= ESTK_MAX_POPULATION,
                 "%s: population_size %d must be even, >= 2 and <= %d", who, P, ESTK_MAX_POPULATION);
  ESTK_CHECK_ARG(n > 0, "%s: n must be positive", who);
  ESTK_CHECK_ARG(ESTK_ALIGNED16(table ? (const void*)table : (const void*)table16),
                 "%s: noise table must be 16-byte aligned", who);
  ESTK_CHECK_ARG(world >= 1 && (P / 2) % world == 0, "%s: world=%d does not divide %d pairs", who, world, P / 2);
  ESTK_CHECK_ARG(pair_begin >= 0 && pairs_local > 0 && pair_begin + pairs_local <= P / 2,
                 "%s: local pairs [%d,+%d) outside %d", who, pair_begin, pairs_local, P / 2);
  const int rc = estk_ctx_reserve(ctx, P, 0, stream, who);
  if (rc) return rc;
  p = {};
  p.returns = returns; p.novelty = novelty; p.w_rew = w_rew; p.w_nov = w_nov;
  p.P = P; p.pairs = P / 2; p.pair_begin = pair_begin; p.pairs_local = pairs_local;
  p.table = table; p.table16 = table16; p.world = world; p.offsets = offsets; p.order = order;
  p.n = n; p.n4 = (n + 3) / 4;
  p.cvals = ctx->cvals; p.partial = ctx->partial;
  p.ranks_out = ranks_out; p.ranks2_out = ranks2_out;
  return ESTK_OK;
}

// The in-place Adam epilogue's fields (estk_rank_grad_adam, estk_rank_grad_xr_adam).
int init_adam(RankGradParams& p, float* theta, float* m, float* v, estk_state* state, const estk_adam_desc* adam,
              float* grad_out, const char* who) {
  ESTK_CHECK_ARG(theta && m && v && state && adam, "%s: null optimizer argument", who);
  ESTK_CHECK_ARG(ESTK_ALIGNED16(theta) && ESTK_ALIGNED16(m) && ESTK_ALIGNED16(v) && (!grad_out || ESTK_ALIGNED16(grad_out)),
                 "%s: theta/m/v/grad_out must be 16-byte aligned", who);
  p.fused_adam = 1; p.grad_out = grad_out;
  p.theta = theta; p.m = m; p.v = v; p.state = state; p.adam = *adam;
  return ESTK_OK;
}

int dispatch(estk_ctx* ctx, RankGradParams& p, cudaStream_t stream) {
  // Large n: 512-thread CTAs, four float4 columns per thread (one CTA per SM), so that a CTA
  // covers its whole column slice in ONE pass over the (offset-sorted) pair list -- all CTAs then
  // walk the table in lock-step, which is what makes overlapping rows hit L2.
  if (p.table16) {                     // fp16 table: columns are 8-element vectors
    p.n4 = (p.n + 7) / 8;
    if (p.xr > 0) {
      if (p.n4 >= (int64_t)ctx->sm_count * 512) return launch_rank_grad<2, 512, 16, true, true>(ctx, p, stream);
      return launch_rank_grad<1, 256, 8, true, true>(ctx, p, stream);
    }
    if (p.n4 >= (int64_t)ctx->sm_count * 512) return launch_rank_grad<2, 512, 16, true>(ctx, p, stream);
    return launch_rank_grad<1, 256, 8, true>(ctx, p, stream);
  }
  if (p.n4 >= (int64_t)ctx->sm_count * 512)
    return launch_rank_grad<4, 512, 16>(ctx, p, stream);   // 16 x 16 B in flight per thread = 128 KB per SM
  return launch_rank_grad<1, 256>(ctx, p, stream);
}

}  // namespace

extern "C" int estk_rank_grad_adam(estk_ctx* ctx, const float* returns, const float* novelty,
                                   float w_rew, float w_nov, int32_t P, const float* table, const uint16_t* table16,
                                   const int64_t* offsets, const int32_t* order, int64_t n,
                                   float* theta, float* m, float* v, estk_state* state,
                                   const estk_adam_desc* adam, int32_t* ranks_out,
                                   int32_t* ranks2_out, float* grad_out, void* stream) {
  const char* who = "estk_rank_grad_adam";
  RankGradParams p;
  int rc = init_common(p, ctx, returns, novelty, w_rew, w_nov, P, 1, table, table16, offsets, order, 0, P / 2, n,
                       ranks_out, ranks2_out, (cudaStream_t)stream, who);
  if (!rc) rc = init_adam(p, theta, m, v, state, adam, grad_out, who);
  return rc ? rc : dispatch(ctx, p, (cudaStream_t)stream);
}

extern "C" int estk_rank_grad(estk_ctx* ctx, const float* returns, const float* novelty,
                              float w_rew, float w_nov, int32_t P, int32_t world, const float* table,
                              const uint16_t* table16, const int64_t* offsets, const int32_t* order,
                              int32_t pair_begin, int32_t pairs_local, int64_t n, float* grad_sum_out,
                              int32_t* ranks_out, int32_t* ranks2_out, void* stream) {
  RankGradParams p;
  const int rc = init_common(p, ctx, returns, novelty, w_rew, w_nov, P, world, table, table16, offsets, order,
                             pair_begin, pairs_local, n, ranks_out, ranks2_out, (cudaStream_t)stream,
                             "estk_rank_grad");
  if (rc) return rc;
  ESTK_CHECK_ARG(grad_sum_out && ESTK_ALIGNED16(grad_sum_out), "estk_rank_grad: grad_sum_out null or unaligned");
  p.fused_adam = 0; p.grad_sum_out = grad_sum_out;
  return dispatch(ctx, p, (cudaStream_t)stream);
}

extern "C" int64_t estk_xr_workspace_bytes(int64_t n) { return n > 0 ? kXrDataOff + 2 * xr_image_bytes(n) : 0; }

extern "C" int estk_rank_grad_xr_adam(estk_ctx* ctx, const float* returns, const float* novelty,
                                      float w_rew, float w_nov, int32_t P, int32_t world, int32_t rank,
                                      const uint16_t* table16, const int64_t* offsets, const int32_t* order,
                                      int32_t pair_begin, int32_t pairs_local, int64_t n,
                                      void* const* peer_ws, float* theta, float* m, float* v,
                                      estk_state* state, const estk_adam_desc* adam,
                                      int32_t* ranks_out, int32_t* ranks2_out, float* grad_out, void* stream) {
  const char* who = "estk_rank_grad_xr_adam";
  ESTK_CHECK_ARG(table16 != nullptr, "%s: null table16", who);
  ESTK_CHECK_ARG(world >= 2 && world <= ESTK_MAX_PEERS && rank >= 0 && rank < world,
                 "%s: world=%d rank=%d (2 <= world <= %d)", who, world, rank, ESTK_MAX_PEERS);
  ESTK_CHECK_ARG(peer_ws != nullptr, "%s: null peer_ws", who);
  RankGradParams p;
  int rc = init_common(p, ctx, returns, novelty, w_rew, w_nov, P, world, nullptr, table16, offsets, order,
                       pair_begin, pairs_local, n, ranks_out, ranks2_out, (cudaStream_t)stream, who);
  if (!rc) rc = init_adam(p, theta, m, v, state, adam, grad_out, who);
  if (rc) return rc;
  p.xr = world; p.xr_rank = rank;
  for (int q = 0; q < world; ++q) {
    ESTK_CHECK_ARG(peer_ws[q] && ESTK_ALIGNED16(peer_ws[q]), "%s: peer workspace %d null or unaligned", who, q);
    p.peer[q] = static_cast<unsigned char*>(peer_ws[q]);
  }
  p.grad_sum_out = reinterpret_cast<float*>(p.peer[rank] + kXrDataOff);   // this rank's partial sum
  return dispatch(ctx, p, (cudaStream_t)stream);
}

extern "C" int estk_clamp_adam(estk_ctx* ctx, const float* grad_sum, int32_t P, int64_t n,
                               float* theta, float* m, float* v, estk_state* state,
                               const estk_adam_desc* adam, float* grad_out, void* stream) {
  ESTK_CHECK_ARG(ctx && grad_sum && adam, "estk_clamp_adam: null argument");
  ESTK_CHECK_ARG(P >= 2 && n > 0, "estk_clamp_adam: bad P/n");
  const bool do_adam = theta != nullptr;
  ESTK_CHECK_ARG(do_adam ? (m && v && state) : (grad_out != nullptr),
                 "estk_clamp_adam: need theta+m+v+state, or grad_out alone");
  RankGradParams p = {};
  p.P = P; p.n = n;
  p.grad_sum_out = const_cast<float*>(grad_sum);
  p.grad_out = grad_out; p.theta = theta; p.m = m; p.v = v; p.state = state; p.adam = *adam;
  int blocks = (int)((n + 255) / 256);
  if (blocks > ctx->sm_count * 8) blocks = ctx->sm_count * 8;
  clamp_adam_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(p, ctx->counters + kTicketClampAdam);
  ESTK_CUDA(cudaGetLastError());
  return ESTK_OK;
}
