// estk_eval_mlp_tc.cu -- kernel 1 of the ES generation (population evaluate) on the Hopper
// tensor cores: warpgroup MMA (wgmma), 16-bit operands / fp32 accumulation.
//
// Same contract as estk_eval_mlp (estk_eval_mlp.cu; reference estorch.py:187-202 +
// Policy.forward examples/cartpole_es.py:14-20 + synthetic agent of SURVEY 8d),
// for policies whose dense layers are worth a GEMM.
//
// Work unit ("task") = (antithetic pair j, sign s, chunk of 64 observations), one CTA.  Per layer
//   D[obs, out] = H[obs, in] * W_s[out, in]^T       (wgmma m64n128k16, N tiles of 128)
//   A  activations H, 64 rows, 16-bit, K-major, 128B-swizzled, resident in shared memory:
//      two buffers (64 KB each) swapped per layer, so a layer's output never overwrites its input;
//   B  W_s = theta + s*sigma*eps, formed ON THE FLY by producer warps into a ring of
//      [128 x 64] stages (16 KB) -- the perturbed weights never exist in global memory;
//   D  64 x 128 fp32 in the registers of the consumer warpgroup; the epilogue adds the bias,
//      applies ReLU and rounds to 16 bits straight into the other activation buffer.  The last
//      layer is fused with the squared-error reduction (and the behaviour characterisation).
// Operand modes (template MODE):
//   kModeBF16   bf16 operands formed from fp32 theta + fp32 table (one FMA in fp32, one rounding)
//   kModeBF16S  bf16 operands formed from bf16 shadows of theta and table (fma.rn.bf16x2)
//   kModeF16    fp16 operands (11-bit significand, the TF32 class) from fp32 theta and the EXACT
//               16-bit copy of the noise table: W16 = rn_f16(theta + s*sigma*eps), sum in fp32; the
//               observations enter layer 0 as x_hi + x_lo (two fp16 k-block sets, same B tile)
// Warp roles: warpgroup 0 = consumer (MMA issue + epilogue), warps 4..11 = weight producers in
// two groups of four, each group forming every other stage of the flattened
// (task, layer, N tile, k-block) sequence.  full / empty mbarriers per ring stage.  Persistent:
// CTAs loop over tasks; the two signs of a pair run on neighbouring CTAs at the same time, so
// the second read of the noise row is an L2 hit.
#include "estk_tc.cuh"
#include <type_traits>

namespace {

constexpr int kRows = 64;                          // observation rows per CTA (wgmma M)
constexpr int kTileN = 128;                        // wgmma N
constexpr int kHBlockBytes = kRows * kBlockK * 2;  // one [64 x 64] 16-bit k-block of activations = 8 KB
constexpr int kHBytes = (kMaxW / kBlockK) * kHBlockBytes;   // 64 KB per activation buffer
constexpr int kStageBytes = kTileN * kBlockK * 2;  // one [128 x 64] 16-bit B stage = 16 KB
constexpr int kStages = 5;
constexpr int kProdWarps = 8, kProdGroups = 2, kProdGroupWarps = kProdWarps / kProdGroups;
constexpr int kPT = 32 * kProdGroupWarps;          // threads per producer group
constexpr int kThreadsTC = 128 + 32 * kProdWarps;  // 384
constexpr int kModeBF16 = 0, kModeBF16S = 1, kModeF16 = 2;

struct EvalTCParams {
  estk_mlp_desc desc;
  const float* theta;
  const float* table;
  const uint16_t* theta16;  // bf16 shadows of theta / table (kModeBF16S)
  const uint16_t* table16;  // bf16 shadow (kModeBF16S) or exact fp16 copy (kModeF16) of the table
  const int64_t* offsets;   // null => centre evaluation
  const int32_t* order;
  int pairs;
  float sigma;
  const float* obs;
  const float* target;
  int B, chunks;            // chunks of kRows observations
  float* ret_plus;
  float* ret_minus;
  float* bc_plus;
  float* bc_minus;
  int bc_obs, bc_dim;
  float* partial;           // [pairs*2 + 1][chunks]
  unsigned int* counters;   // [pairs*2 + 1]
  float* centre_out;        // optional: also evaluate theta itself (sigma = 0) into centre_out[0]
  int n_centre;             // number of leading centre tasks (0 or chunks)
  int n_tasks;              // n_centre + pairs * n_signs * chunks
  int n_signs;              // 2, or 1 for the centre evaluation
  int mode;
};

struct Layer { int K, N; int64_t wbase, bbase; };

// task -> (slot, sign, chunk); the first n_centre tasks evaluate theta itself
struct TaskId { int slot, sgn, chunk; bool centre; };
__device__ __forceinline__ TaskId decode_task(const EvalTCParams& p, int task, bool all_centre) {
  TaskId t;
  if (task < p.n_centre) { t.slot = 0; t.sgn = 0; t.chunk = task; t.centre = true; return t; }
  const int q = task - p.n_centre;
  t.chunk = q % p.chunks;
  t.sgn = (q / p.chunks) % p.n_signs;
  t.slot = q / (p.chunks * p.n_signs);
  t.centre = all_centre;
  return t;
}

template <int MODE>
__global__ void __launch_bounds__(kThreadsTC, 1) eval_mlp_tc_kernel(const EvalTCParams p) {
  constexpr bool S16 = (MODE == kModeBF16S), F16 = (MODE == kModeF16);
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sH = smem;                                  // 2 activation buffers x 8 k-blocks x 8 KB
  uint8_t* sB = sH + 2 * kHBytes;                      // ring
  float* sBias = reinterpret_cast<float*>(sB + kStages * kStageBytes);   // [512], one layer at a time
  uint64_t* bar_full = reinterpret_cast<uint64_t*>(sBias + kMaxW);      // [kStages] stage formed
  uint64_t* bar_empty = bar_full + kStages;                             // [kStages] stage consumed
  float* s_loss = reinterpret_cast<float*>(bar_empty + kStages);        // [4]
  __shared__ Layer lay[ESTK_MAX_LAYERS];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int L = p.desc.n_layers;
  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(smem_u32(bar_full + s), kProdGroupWarps);
      mbar_init(smem_u32(bar_empty + s), 4);
    }
    fence_barrier_init();
    int64_t pb = 0;
    for (int l = 0; l < L; ++l) {
      lay[l].K = p.desc.dims[l];
      lay[l].N = p.desc.dims[l + 1];
      lay[l].wbase = pb;
      lay[l].bbase = pb + (int64_t)lay[l].K * lay[l].N;
      pb = lay[l].bbase + lay[l].N;
    }
  }
  __syncthreads();
  const bool centre = (p.offsets == nullptr);

  if (warp < 4) {
    // =================================================================== consumer warpgroup
    const int tid = threadIdx.x;                     // 0..127
    const int r0 = warp * 16 + (lane >> 2);          // accumulator rows r0 and r0 + 8
    const int cq = (lane & 3) * 2;                   // accumulator columns 8j + cq, +1
    uint32_t kst = 0;                                // global stage index
    for (int task = blockIdx.x; task < p.n_tasks; task += gridDim.x) {
      const TaskId tk = decode_task(p, task, centre);
      const int chunk = tk.chunk, sgn = tk.sgn, slot = tk.slot;
      const int j = (!tk.centre && p.order) ? p.order[slot] : slot;
      const float* trow = tk.centre ? p.theta : p.table + p.offsets[j];
      const float ssig = tk.centre ? 0.f : (sgn ? -p.sigma : p.sigma);
      float* bc = (tk.centre && !centre) ? nullptr : (sgn ? p.bc_minus : p.bc_plus);
      // ---- this CTA's observations as the layer-0 A operand (buffer 0)
      {
        const int K0 = lay[0].K, per_row = K0 / 8;
        for (int it = tid; it < kRows * per_row; it += 128) {
          const int r = it / per_row, c = it % per_row;
          const float* src = p.obs + (size_t)(chunk * kRows + r) * K0 + c * 8;
          const float4 x0 = __ldg(reinterpret_cast<const float4*>(src));
          const float4 x1 = __ldg(reinterpret_cast<const float4*>(src + 4));
          const uint32_t addr = smem_u32(sH + (c >> 3) * kHBlockBytes) + sw128_offset(r, c & 7);
          const uint32_t h0 = pack16<F16>(x0.x, x0.y), h1 = pack16<F16>(x0.z, x0.w);
          const uint32_t h2 = pack16<F16>(x1.x, x1.y), h3 = pack16<F16>(x1.z, x1.w);
          st_shared_v4(addr, h0, h1, h2, h3);
          if constexpr (F16) {
            // x_lo = rn_f16(x - x_hi): the observation enters layer 0 with ~22 significant bits
            const float2 f0 = unpack_f16(h0), f1 = unpack_f16(h1), f2 = unpack_f16(h2), f3 = unpack_f16(h3);
            st_shared_v4(addr + (K0 / kBlockK) * kHBlockBytes, pack_f16(x0.x - f0.x, x0.y - f0.y),
                         pack_f16(x0.z - f1.x, x0.w - f1.y), pack_f16(x1.x - f2.x, x1.y - f2.y),
                         pack_f16(x1.z - f3.x, x1.w - f3.y));
          }
        }
      }
      float loss = 0.f;
      for (int l = 0; l < L; ++l) {
        const int K = lay[l].K, N = lay[l].N;
        const bool last = (l == L - 1);
        const uint32_t h_in = smem_u32(sH + (l & 1) * kHBytes);
        const uint32_t h_out = smem_u32(sH + ((l + 1) & 1) * kHBytes);
        named_bar_sync(1, 128);          // previous layer's epilogue (bias reads) done
        for (int o = tid; o < N; o += 128)
          sBias[o] = fmaf(ssig, ld_noise1(trow + lay[l].bbase + o), __ldg(p.theta + lay[l].bbase + o));
        fence_proxy_async();             // this layer's input (generic-proxy stores) -> wgmma
        named_bar_sync(1, 128);          // ... by every thread; bias[] published
        const int lo_kb = (F16 && l == 0) ? K / kBlockK : 0;   // layer 0 in fp16: x_lo k-blocks
        for (int n0 = 0; n0 < N; n0 += kTileN) {
          const int width = min(kTileN, N - n0);
          float d[64];                     // the first MMA of the tile overwrites (scale-d = 0)
          uint32_t prev = 0;
          // NP = 2: layer 0 in fp16, x_lo on the same B tile (a separate instantiation, so that no
          // wgmma sits under a branch)
          auto k_loop = [&](auto np_tag) {
            constexpr int NP = decltype(np_tag)::value;
            for (int kb = 0; kb < K / kBlockK; ++kb, ++kst) {
              const uint32_t stage = kst % kStages, phase = (kst / kStages) & 1u;
              mbar_wait(smem_u32(bar_full + stage), phase);
              const uint32_t a_addr = h_in + kb * kHBlockBytes, b_addr = smem_u32(sB + stage * kStageBytes);
              wgmma_fence();
#pragma unroll
              for (int pass = 0; pass < NP; ++pass) {
                const uint32_t a = a_addr + pass * lo_kb * kHBlockBytes;
#pragma unroll
                for (int k = 0; k < kBlockK / 16; ++k)
                  wgmma_m64n128k16<F16>(d, make_sw128_desc(a + k * 32), make_sw128_desc(b_addr + k * 32),
                                        (kb | k | pass) != 0 ? 1u : 0u);
              }
              wgmma_commit();
              wgmma_wait<1>();             // the previous stage's MMAs are done: release its slot
              if (kb > 0 && lane == 0) mbar_arrive(smem_u32(bar_empty + prev));
              prev = stage;
            }
          };
          if (F16 && lo_kb) k_loop(std::integral_constant<int, 2>{});
          else k_loop(std::integral_constant<int, 1>{});
          wgmma_wait<0>();
          fence_acc(d);
          if (lane == 0) mbar_arrive(smem_u32(bar_empty + prev));
          // ---- epilogue of the tile
#pragma unroll
          for (int jb = 0; jb < kTileN / 8; ++jb) {
            if (jb * 8 < width) {
              const int col = n0 + jb * 8 + cq;
              const float2 bv = *reinterpret_cast<const float2*>(sBias + col);
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int r = r0 + 8 * h;
                const float y0 = d[jb * 4 + 2 * h] + bv.x, y1 = d[jb * 4 + 2 * h + 1] + bv.y;
                if (last) {
                  const int b = chunk * kRows + r;
                  const float2 t = __ldg(reinterpret_cast<const float2*>(p.target + (size_t)b * N + col));
                  const float e0 = y0 - t.x, e1 = y1 - t.y;
                  loss = fmaf(e0, e0, loss);
                  loss = fmaf(e1, e1, loss);
                  if (bc && b < p.bc_obs) {
                    const int64_t idx = (int64_t)b * N + col;
                    if (idx < p.bc_dim) bc[(size_t)j * p.bc_dim + idx] = y0;
                    if (idx + 1 < p.bc_dim) bc[(size_t)j * p.bc_dim + idx + 1] = y1;
                  }
                } else {
                  st_shared_u32(h_out + (col >> 6) * kHBlockBytes + sw128_offset(r, (col & 63) >> 3) + (col & 7) * 2,
                                pack16_relu<F16>(y0, y1));
                }
              }
            }
          }
        }
      }
      // ---- squared-error partial of this CTA; the last arriver combines them in fixed order
      loss = warp_sum_f(loss);
      if (lane == 0) s_loss[warp] = loss;
      named_bar_sync(1, 128);
      if (tid == 0) {
        const float tot = (s_loss[0] + s_loss[1]) + (s_loss[2] + s_loss[3]);
        const int parts = p.chunks;
        const bool folded = tk.centre && !centre;                 // centre task riding in a population launch
        const int cell = folded ? p.pairs * 2 : slot * 2 + sgn;
        float* part = p.partial + (size_t)cell * parts;
        part[chunk] = tot;
        __threadfence();
        const unsigned int arrived = atomicAdd(p.counters + cell, 1u);
        if (arrived == (unsigned int)parts - 1) {
          __threadfence();
          float s = 0.f;
          for (int c = 0; c < parts; ++c) s += __ldcg(part + c);
          const float r = -(s / ((float)p.B * (float)lay[L - 1].N));
          if (folded) p.centre_out[0] = r;
          else if (sgn) p.ret_minus[j] = r;
          else p.ret_plus[j] = r;
          p.counters[cell] = 0u;
        }
      }
    }
  } else {
    // =================================================================== weight producers
    // Group g forms stages g, g+G, g+2G, ... of the flattened (task, layer, N tile, k-block)
    // sequence.  Item `it` of a stage = tile row it/8, 16-byte output chunk it%8 (8 weights).
    const int pwarp = warp - 4;
    const int pgroup = pwarp / kProdGroupWarps;
    const int ptid = (pwarp % kProdGroupWarps) * 32 + lane;
    constexpr int kBatch = (MODE == kModeBF16) ? 4 : 8;    // items whose loads are in flight together
    int cached_task = -1;
    const float* trow = p.theta;
    const uint16_t* trow16 = nullptr;
    float ssig = 0.f;
    int task = blockIdx.x, l = 0, n0 = 0, kb = 0;
    auto advance = [&]() -> bool {
      if (++kb >= lay[l].K / kBlockK) {
        kb = 0;
        n0 += kTileN;
        if (n0 >= lay[l].N) {
          n0 = 0;
          if (++l == L) { l = 0; task += gridDim.x; }
        }
      }
      return task < p.n_tasks;
    };
    bool has = task < p.n_tasks;
    for (int sk = 0; sk < pgroup && has; ++sk) has = advance();
    uint32_t kst = pgroup;
    while (has) {
      if (task != cached_task) {            // two dependent global loads: once per task, not per stage
        cached_task = task;
        const TaskId tk = decode_task(p, task, centre);
        const int jj = (!tk.centre && p.order) ? p.order[tk.slot] : tk.slot;
        trow = tk.centre ? p.theta : p.table + p.offsets[jj];
        trow16 = tk.centre ? (S16 ? p.theta16 : nullptr) : p.table16 + p.offsets[jj];
        ssig = tk.centre ? 0.f : (tk.sgn ? -p.sigma : p.sigma);
      }
      const uint32_t stage = kst % kStages, phase = (kst / kStages) & 1u;
      const uint32_t sbase = smem_u32(sB + stage * kStageBytes);
      const int K = lay[l].K;
      const int n_items = min(kTileN, lay[l].N - n0) * 8;
      const int64_t rbase = lay[l].wbase + (int64_t)n0 * K + kb * kBlockK;
      bool waited = false;
      for (int it0 = 0; it0 < n_items; it0 += kBatch * kPT) {
        float4 th[kBatch][2], ep[kBatch][2];
        uint4 t16[kBatch], e16[kBatch];
        // every load of the batch is issued up front ...
#pragma unroll
        for (int u = 0; u < kBatch; ++u) {
          const int it = it0 + u * kPT + ptid;
          if (it < n_items) {
            const int64_t off = rbase + (int64_t)(it >> 3) * K + (it & 7) * 8;
            if constexpr (S16) {
              t16[u] = ld_noise4u(reinterpret_cast<const uint4*>(p.theta16 + off));
              e16[u] = ld_noise4u(reinterpret_cast<const uint4*>(trow16 + off));
            } else if constexpr (F16) {
              th[u][0] = ld_noise4(reinterpret_cast<const float4*>(p.theta + off));
              th[u][1] = ld_noise4(reinterpret_cast<const float4*>(p.theta + off + 4));
              e16[u] = trow16 ? ld_noise4u(reinterpret_cast<const uint4*>(trow16 + off)) : make_uint4(0u, 0u, 0u, 0u);
            } else {
              th[u][0] = ld_noise4(reinterpret_cast<const float4*>(p.theta + off));
              th[u][1] = ld_noise4(reinterpret_cast<const float4*>(p.theta + off + 4));
              ep[u][0] = ld_noise4(reinterpret_cast<const float4*>(trow + off));
              ep[u][1] = ld_noise4(reinterpret_cast<const float4*>(trow + off + 4));
            }
          }
        }
        // ... then wait for the ring slot
        if (!waited) {
          mbar_wait(smem_u32(bar_empty + stage), phase ^ 1);
          waited = true;
        }
#pragma unroll
        for (int u = 0; u < kBatch; ++u) {
          const int it = it0 + u * kPT + ptid;
          if (it < n_items) {
            const float sg = ssig;
            uint32_t w[4];
            if constexpr (S16) {
              // W = theta16 + (s*sigma)_bf16 * eps16: exact product-sum, one rounding to bf16
              const uint32_t sg2 = pack_bf16(sg, sg);
              const uint32_t tw[4] = {t16[u].x, t16[u].y, t16[u].z, t16[u].w};
              const uint32_t ew[4] = {e16[u].x, e16[u].y, e16[u].z, e16[u].w};
#pragma unroll
              for (int c = 0; c < 4; ++c) asm("fma.rn.bf16x2 %0, %1, %2, %3;" : "=r"(w[c]) : "r"(sg2), "r"(ew[c]), "r"(tw[c]));
            } else if constexpr (F16) {
              const float2 e0 = unpack_f16(e16[u].x), e1 = unpack_f16(e16[u].y);
              const float2 e2 = unpack_f16(e16[u].z), e3 = unpack_f16(e16[u].w);
              w[0] = pack_f16(fmaf(sg, e0.x, th[u][0].x), fmaf(sg, e0.y, th[u][0].y));
              w[1] = pack_f16(fmaf(sg, e1.x, th[u][0].z), fmaf(sg, e1.y, th[u][0].w));
              w[2] = pack_f16(fmaf(sg, e2.x, th[u][1].x), fmaf(sg, e2.y, th[u][1].y));
              w[3] = pack_f16(fmaf(sg, e3.x, th[u][1].z), fmaf(sg, e3.y, th[u][1].w));
            } else {
              w[0] = pack_bf16(fmaf(sg, ep[u][0].x, th[u][0].x), fmaf(sg, ep[u][0].y, th[u][0].y));
              w[1] = pack_bf16(fmaf(sg, ep[u][0].z, th[u][0].z), fmaf(sg, ep[u][0].w, th[u][0].w));
              w[2] = pack_bf16(fmaf(sg, ep[u][1].x, th[u][1].x), fmaf(sg, ep[u][1].y, th[u][1].y));
              w[3] = pack_bf16(fmaf(sg, ep[u][1].z, th[u][1].z), fmaf(sg, ep[u][1].w, th[u][1].w));
            }
            st_shared_v4(sbase + sw128_offset(it >> 3, it & 7), w[0], w[1], w[2], w[3]);
          }
        }
      }
      if (!waited) mbar_wait(smem_u32(bar_empty + stage), phase ^ 1);
      fence_proxy_async();
      __syncwarp();
      if (lane == 0) mbar_arrive(smem_u32(bar_full + stage));
      for (int sk = 0; sk < kProdGroups && has; ++sk) has = advance();
      kst += kProdGroups;
    }
  }
}

size_t tc_smem_bytes() {
  return 1024 + 2 * (size_t)kHBytes + (size_t)kStages * kStageBytes + kMaxW * sizeof(float) +
         2 * kStages * sizeof(uint64_t) + 4 * sizeof(float);
}

template <int MODE>
int launch_tc(estk_ctx* ctx, const EvalTCParams& p, cudaStream_t stream) {
  const size_t smem = tc_smem_bytes();
  ESTK_CUDA(cudaFuncSetAttribute(eval_mlp_tc_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int grid = ctx->sm_count < p.n_tasks ? ctx->sm_count : p.n_tasks;
  eval_mlp_tc_kernel<MODE><<<grid, kThreadsTC, smem, stream>>>(p);
  ESTK_CUDA(cudaGetLastError());
  return ESTK_OK;
}

int tc_supported(const estk_mlp_desc& d, int B, const char** why, int mode) {
  if (mode == kModeF16 && d.n_layers >= 1 && 2 * d.dims[0] > kMaxW) {
    *why = "fp16 mode splits the observations into hi + lo halves: input width <= 256"; return 0;
  }
  if (d.n_layers < 1 || d.n_layers > ESTK_MAX_LAYERS) { *why = "n_layers"; return 0; }
  if (d.activation != 0) { *why = "activation"; return 0; }
  for (int l = 0; l < d.n_layers; ++l) {
    if (d.dims[l] % 64 || d.dims[l] > kMaxW || d.dims[l] < 64) { *why = "layer input width must be a multiple of 64 in [64,512]"; return 0; }
    const int N = d.dims[l + 1];
    if (N % 32 || N > kMaxW || N < 32) { *why = "layer output width must be a multiple of 32 in [32,512]"; return 0; }
  }
  if (B % 256) { *why = "batch must be a multiple of 256"; return 0; }
  return 1;
}

int run_tc(estk_ctx* ctx, EvalTCParams& p, cudaStream_t stream, const char* who) {
  const char* why = "";
  if (!tc_supported(p.desc, p.B, &why, p.mode)) {
    estk_set_error("%s: shape not supported by the tensor-core path (%s)", who, why);
    return ESTK_ERR_UNSUPPORTED;
  }
  ESTK_CHECK_ARG(p.pairs >= 1 && p.pairs <= ESTK_MAX_POPULATION / 2, "%s: pairs=%d", who, p.pairs);
  p.chunks = p.B / kRows;
  ESTK_CHECK_ARG(p.chunks <= 2 * kEvalMaxChunks, "%s: batch too large", who);
  p.n_centre = p.centre_out ? p.chunks : 0;
  ESTK_CHECK_ARG(!p.centre_out || p.pairs * 2 < ESTK_MAX_POPULATION, "%s: population too large to fold the centre task", who);
  p.n_tasks = p.n_centre + p.pairs * p.n_signs * p.chunks;
  p.partial = ctx->eval_partial;
  p.counters = ctx->counters;
  if (p.mode == kModeF16) return launch_tc<kModeF16>(ctx, p, stream);
  if (p.mode == kModeBF16S) return launch_tc<kModeBF16S>(ctx, p, stream);
  return launch_tc<kModeBF16>(ctx, p, stream);
}

}  // namespace

extern "C" int estk_eval_mlp_bf16(estk_ctx* ctx, const estk_mlp_desc* desc, const float* theta,
                                  const float* table, const int64_t* offsets, const int32_t* order,
                                  int32_t pairs, float sigma, const float* obs, const float* target,
                                  int32_t B, float* returns_plus, float* returns_minus, float* bc_plus,
                                  float* bc_minus, int32_t bc_obs, int32_t bc_dim, float* centre_return_out,
                                  void* stream) {
  ESTK_CHECK_ARG(ctx && desc && theta && table && offsets && obs && target && returns_plus && returns_minus,
                 "estk_eval_mlp_bf16: null argument");
  ESTK_CHECK_ARG((bc_plus == nullptr) == (bc_minus == nullptr), "estk_eval_mlp_bf16: bc_plus/bc_minus must both be set or both null");
  ESTK_CHECK_ARG(ESTK_ALIGNED16(theta) && ESTK_ALIGNED16(table) && ESTK_ALIGNED16(obs) && ESTK_ALIGNED16(target),
                 "estk_eval_mlp_bf16: theta/table/obs/target must be 16-byte aligned");
  EvalTCParams p = {};
  p.desc = *desc; p.theta = theta; p.table = table; p.offsets = offsets; p.order = order;
  p.pairs = pairs; p.sigma = sigma; p.obs = obs; p.target = target; p.B = B;
  p.ret_plus = returns_plus; p.ret_minus = returns_minus;
  p.bc_plus = bc_plus; p.bc_minus = bc_minus; p.bc_obs = bc_obs; p.bc_dim = bc_dim;
  p.n_signs = 2; p.centre_out = centre_return_out; p.mode = kModeBF16;
  return run_tc(ctx, p, (cudaStream_t)stream, "estk_eval_mlp_bf16");
}

extern "C" int estk_eval_mlp_center_bf16(estk_ctx* ctx, const estk_mlp_desc* desc, const float* theta,
                                         const float* obs, const float* target, int32_t B,
                                         float* return_out, float* bc_out, int32_t bc_obs,
                                         int32_t bc_dim, void* stream) {
  ESTK_CHECK_ARG(ctx && desc && theta && obs && target && return_out, "estk_eval_mlp_center_bf16: null argument");
  EvalTCParams p = {};
  p.desc = *desc; p.theta = theta; p.table = theta; p.offsets = nullptr; p.order = nullptr;
  p.pairs = 1; p.sigma = 0.f; p.obs = obs; p.target = target; p.B = B;
  p.ret_plus = return_out; p.ret_minus = nullptr;
  p.bc_plus = bc_out; p.bc_minus = nullptr; p.bc_obs = bc_obs; p.bc_dim = bc_dim;
  p.n_signs = 1; p.mode = kModeBF16;
  return run_tc(ctx, p, (cudaStream_t)stream, "estk_eval_mlp_center_bf16");
}

__global__ void __launch_bounds__(256) shadow_bf16_kernel(const float4* __restrict__ src, uint2* __restrict__ dst, int64_t n4) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 v = src[i];
    uint2 o;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(o.x) : "f"(v.y), "f"(v.x));
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(o.y) : "f"(v.w), "f"(v.z));
    dst[i] = o;
  }
}

extern "C" int estk_shadow_bf16(estk_ctx* ctx, const float* src, uint16_t* dst, int64_t n, void* stream) {
  ESTK_CHECK_ARG(ctx && src && dst && n > 0 && (n % 4) == 0, "estk_shadow_bf16: null argument or n not a multiple of 4");
  ESTK_CHECK_ARG(ESTK_ALIGNED16(src) && ((uintptr_t)dst & 7u) == 0, "estk_shadow_bf16: unaligned buffers");
  int blocks = (int)((n / 4 + 255) / 256);
  if (blocks > ctx->sm_count * 16) blocks = ctx->sm_count * 16;
  shadow_bf16_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4*>(src),
                                                             reinterpret_cast<uint2*>(dst), n / 4);
  ESTK_CUDA(cudaGetLastError());
  return ESTK_OK;
}

extern "C" int estk_eval_mlp_bf16s(estk_ctx* ctx, const estk_mlp_desc* desc, const float* theta,
                                   const uint16_t* theta16, const float* table, const uint16_t* table16,
                                   const int64_t* offsets, const int32_t* order, int32_t pairs, float sigma,
                                   const float* obs, const float* target, int32_t B, float* returns_plus,
                                   float* returns_minus, float* bc_plus, float* bc_minus, int32_t bc_obs,
                                   int32_t bc_dim, float* centre_return_out, void* stream) {
  ESTK_CHECK_ARG(ctx && desc && theta && theta16 && table && table16 && offsets && obs && target &&
                 returns_plus && returns_minus, "estk_eval_mlp_bf16s: null argument");
  ESTK_CHECK_ARG((bc_plus == nullptr) == (bc_minus == nullptr), "estk_eval_mlp_bf16s: bc_plus/bc_minus must both be set or both null");
  ESTK_CHECK_ARG(ESTK_ALIGNED16(theta) && ESTK_ALIGNED16(table) && ESTK_ALIGNED16(obs) && ESTK_ALIGNED16(target) &&
                 ESTK_ALIGNED16(theta16) && ESTK_ALIGNED16(table16),
                 "estk_eval_mlp_bf16s: buffers must be 16-byte aligned");
  EvalTCParams p = {};
  p.desc = *desc; p.theta = theta; p.table = table; p.theta16 = theta16; p.table16 = table16;
  p.offsets = offsets; p.order = order;
  p.pairs = pairs; p.sigma = sigma; p.obs = obs; p.target = target; p.B = B;
  p.ret_plus = returns_plus; p.ret_minus = returns_minus;
  p.bc_plus = bc_plus; p.bc_minus = bc_minus; p.bc_obs = bc_obs; p.bc_dim = bc_dim;
  p.n_signs = 2; p.centre_out = centre_return_out; p.mode = kModeBF16S;
  return run_tc(ctx, p, (cudaStream_t)stream, "estk_eval_mlp_bf16s");
}

extern "C" int estk_eval_mlp_center_bf16s(estk_ctx* ctx, const estk_mlp_desc* desc, const float* theta,
                                          const uint16_t* theta16, const float* obs, const float* target,
                                          int32_t B, float* return_out, float* bc_out, int32_t bc_obs,
                                          int32_t bc_dim, void* stream) {
  ESTK_CHECK_ARG(ctx && desc && theta && theta16 && obs && target && return_out, "estk_eval_mlp_center_bf16s: null argument");
  EvalTCParams p = {};
  p.desc = *desc; p.theta = theta; p.table = theta; p.theta16 = theta16; p.table16 = theta16;
  p.offsets = nullptr; p.order = nullptr;
  p.pairs = 1; p.sigma = 0.f; p.obs = obs; p.target = target; p.B = B;
  p.ret_plus = return_out; p.ret_minus = nullptr;
  p.bc_plus = bc_out; p.bc_minus = nullptr; p.bc_obs = bc_obs; p.bc_dim = bc_dim;
  p.n_signs = 1; p.mode = kModeBF16S;
  return run_tc(ctx, p, (cudaStream_t)stream, "estk_eval_mlp_center_bf16s");
}

// ---- fp16 operands from fp32 theta + the exact 16-bit noise table (the default tensor-core mode).
__global__ void __launch_bounds__(256) shadow_f16_kernel(const float4* __restrict__ src, uint2* __restrict__ dst, int64_t n4,
                                                         unsigned long long* __restrict__ inexact) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  unsigned int bad = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 v = src[i];
    const __half2 a = __floats2half2_rn(v.x, v.y), b = __floats2half2_rn(v.z, v.w);
    const float2 fa = __half22float2(a), fb = __half22float2(b);
    bad += (fa.x != v.x) + (fa.y != v.y) + (fb.x != v.z) + (fb.y != v.w);
    uint2 o;
    o.x = *reinterpret_cast<const uint32_t*>(&a);
    o.y = *reinterpret_cast<const uint32_t*>(&b);
    dst[i] = o;
  }
  if (inexact && bad) atomicAdd(inexact, (unsigned long long)bad);
}

extern "C" int estk_shadow_f16(estk_ctx* ctx, const float* src, uint16_t* dst, int64_t n, uint64_t* inexact_count,
                               void* stream) {
  ESTK_CHECK_ARG(ctx && src && dst && n > 0 && (n % 4) == 0, "estk_shadow_f16: null argument or n not a multiple of 4");
  ESTK_CHECK_ARG(ESTK_ALIGNED16(src) && ((uintptr_t)dst & 7u) == 0, "estk_shadow_f16: unaligned buffers");
  int blocks = (int)((n / 4 + 255) / 256);
  if (blocks > ctx->sm_count * 16) blocks = ctx->sm_count * 16;
  shadow_f16_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4*>(src),
                                                            reinterpret_cast<uint2*>(dst), n / 4,
                                                            reinterpret_cast<unsigned long long*>(inexact_count));
  ESTK_CUDA(cudaGetLastError());
  return ESTK_OK;
}

extern "C" int estk_eval_mlp_f16(estk_ctx* ctx, const estk_mlp_desc* desc, const float* theta, const float* table,
                                 const uint16_t* table16, const int64_t* offsets, const int32_t* order, int32_t pairs,
                                 float sigma, const float* obs, const float* target, int32_t B, float* returns_plus,
                                 float* returns_minus, float* bc_plus, float* bc_minus, int32_t bc_obs,
                                 int32_t bc_dim, float* centre_return_out, void* stream) {
  ESTK_CHECK_ARG(ctx && desc && theta && table && table16 && offsets && obs && target && returns_plus && returns_minus,
                 "estk_eval_mlp_f16: null argument");
  ESTK_CHECK_ARG((bc_plus == nullptr) == (bc_minus == nullptr), "estk_eval_mlp_f16: bc_plus/bc_minus must both be set or both null");
  ESTK_CHECK_ARG(ESTK_ALIGNED16(theta) && ESTK_ALIGNED16(table) && ESTK_ALIGNED16(obs) && ESTK_ALIGNED16(target) &&
                 ESTK_ALIGNED16(table16), "estk_eval_mlp_f16: buffers must be 16-byte aligned");
  EvalTCParams p = {};
  p.desc = *desc; p.theta = theta; p.table = table; p.table16 = table16;
  p.offsets = offsets; p.order = order;
  p.pairs = pairs; p.sigma = sigma; p.obs = obs; p.target = target; p.B = B;
  p.ret_plus = returns_plus; p.ret_minus = returns_minus;
  p.bc_plus = bc_plus; p.bc_minus = bc_minus; p.bc_obs = bc_obs; p.bc_dim = bc_dim;
  p.n_signs = 2; p.centre_out = centre_return_out; p.mode = kModeF16;
  return run_tc(ctx, p, (cudaStream_t)stream, "estk_eval_mlp_f16");
}

extern "C" int estk_eval_mlp_center_f16(estk_ctx* ctx, const estk_mlp_desc* desc, const float* theta,
                                        const float* obs, const float* target, int32_t B, float* return_out,
                                        float* bc_out, int32_t bc_obs, int32_t bc_dim, void* stream) {
  ESTK_CHECK_ARG(ctx && desc && theta && obs && target && return_out, "estk_eval_mlp_center_f16: null argument");
  ESTK_CHECK_ARG(ESTK_ALIGNED16(theta) && ESTK_ALIGNED16(obs) && ESTK_ALIGNED16(target),
                 "estk_eval_mlp_center_f16: buffers must be 16-byte aligned");
  EvalTCParams p = {};
  p.desc = *desc; p.theta = theta; p.table = theta; p.offsets = nullptr; p.order = nullptr;
  p.pairs = 1; p.sigma = 0.f; p.obs = obs; p.target = target; p.B = B;
  p.ret_plus = return_out; p.ret_minus = nullptr;
  p.bc_plus = bc_out; p.bc_minus = nullptr; p.bc_obs = bc_obs; p.bc_dim = bc_dim;
  p.n_signs = 1; p.mode = kModeF16;
  return run_tc(ctx, p, (cudaStream_t)stream, "estk_eval_mlp_center_f16");
}

extern "C" int estk_eval_mlp_f16_supported(const estk_mlp_desc* desc, int32_t B) {
  const char* why = "";
  return desc ? tc_supported(*desc, B, &why, kModeF16) : 0;
}

extern "C" int estk_eval_mlp_bf16_supported(const estk_mlp_desc* desc, int32_t B) {
  const char* why = "";
  return desc ? tc_supported(*desc, B, &why, kModeBF16) : 0;
}
