// estk_eval_conv.cu -- population evaluate for the conv + VirtualBatchNorm policy
// of the reference's Atari example (fp32 CUDA cores, correctness-first).
//
// Replaces, per member theta +- sigma*eps (reference file:line, /root/reference):
//   Policy.forward            examples/atari.py:25-37
//     xref = relu(bn1(conv1(xref)));  xref = relu(bn2(conv2(xref)))     # stats pass
//     x = relu(bn1(conv1(x)));  x = relu(bn2(conv2(x)));  x = fc2(relu(fc1(x.view(-1,2592))))
//   VirtualBatchNorm.forward  estorch/modules.py:48-58  first call: per-(C,H,W) mean and
//                             UNBIASED variance over the reference batch (:51-52),
//                             normalize (:42-46): (x-mean)/sqrt(var+eps)*gamma_c+beta_c
//   ES._calculate_returns     estorch/estorch.py:195-202  (synthetic agent: -mean((out-y)^2))
// In the reference the reference-batch pass is repeated on every forward call; the
// weights are fixed within a rollout, so once per member is the same function.
//
// Architecture (fixed by the example): conv1 4->16 k8 s4 (84x84 -> 20x20), VBN(16),
// conv2 16->32 k4 s2 (-> 9x9), VBN(32), fc1 2592->256, fc2 256->A.  Parameter order =
// registration order (SURVEY App. A.10): conv1.w 4096, conv1.b 16, bn1.w 16, bn1.b 16,
// conv2.w 8192, conv2.b 32, bn2.w 32, bn2.b 32, fc1.w 663552, fc1.b 256, fc2.w 256A, fc2.b A.
//
// One persistent CTA per member (grid = #SMs): small weights perturbed into shared
// memory; layer-1 reference activations and the flattened conv features of the
// observation batch go through a per-CTA global scratch slab (L2 resident).
#include "estk_common.cuh"

namespace {

constexpr int kT = 256;
constexpr int C1 = 16, H1 = 20, W1 = 20, P1 = C1 * H1 * W1;   // 6400
constexpr int C2 = 32, H2 = 9, W2 = 9, P2 = C2 * H2 * W2;     // 2592
constexpr int IMG = 4 * 84 * 84;
constexpr int FC1 = 256;
constexpr int TB = 32;    // images per fc tile
constexpr int KT = 32;    // k-tile of fc1

struct ConvParams {
  const float* theta;
  const float* table;
  const int64_t* offsets;  // null => centre
  const int32_t* order;
  int pairs;
  float sigma;
  int A, R, B;
  const float* xref;
  const float* obs;
  const float* target;
  float* ret_plus;
  float* ret_minus;
  float* scratch;          // per CTA: R*P1 + B*P2 floats
  int64_t scratch_per_cta;
  int members;
};

struct Offs { int64_t c1w, c1b, g1, b1, c2w, c2b, g2, b2, f1w, f1b, f2w, f2b; };

__device__ __forceinline__ Offs layout(int A) {
  Offs o;
  o.c1w = 0; o.c1b = 4096; o.g1 = 4112; o.b1 = 4128; o.c2w = 4144; o.c2b = 12336; o.g2 = 12368; o.b2 = 12400;
  o.f1w = 12432; o.f1b = o.f1w + (int64_t)FC1 * P2; o.f2w = o.f1b + FC1; o.f2b = o.f2w + (int64_t)A * FC1;
  return o;
}

__global__ void __launch_bounds__(kT, 1) eval_conv_vbn_kernel(const ConvParams p) {
  extern __shared__ __align__(16) float sm[];
  float* sW1 = sm;                    // [16][256]
  float* sW2 = sW1 + C1 * 256;        // [32][256]
  float* sSmall = sW2 + C2 * 256;     // conv1.b 16, conv2.b 32, bn1.b 16, bn2.b 32  (96 of 128)
  float* sA1 = sSmall + 128;          // [6400] scale of VBN1 per position
  float* sM1 = sA1 + P1;              // [6400] mean
  float* sA2 = sM1 + P1;              // [2592]
  float* sM2 = sA2 + P2;              // [2592]
  float* sX1 = sM2 + P2;              // [6400] normalised layer-1 activations of one image
  // fc phase aliases sX1.. : Wt [KT][FC1+1], Xt [TB][KT], Hs [TB][FC1]
  float* sWt = sX1;
  float* sXt = sWt + KT * (FC1 + 1);
  float* sHs = sA1;                   // stats are dead by then: [TB][FC1] = 8192 floats <= 2*P1
  __shared__ float s_red[kT / 32];

  const int tid = threadIdx.x;
  const Offs L = layout(p.A);
  const bool centre = (p.offsets == nullptr);
  float* R1 = p.scratch + (int64_t)blockIdx.x * p.scratch_per_cta;   // [R][P1]
  float* XS = R1 + (int64_t)p.R * P1;                                  // [B][P2]

  for (int member = blockIdx.x; member < p.members; member += gridDim.x) {
    const int pairs = p.pairs;
    const bool minus = (!centre) && member >= pairs;
    const int slot = centre ? 0 : (minus ? member - pairs : member);
    const int j = (!centre && p.order) ? p.order[slot] : slot;
    const float* trow = centre ? p.theta : p.table + p.offsets[j];
    const float sg = centre ? 0.f : (minus ? -p.sigma : p.sigma);
    auto par = [&](int64_t idx) -> float {   // perturbed parameter, same two roundings as estorch.py:189-192
      return __fadd_rn(__ldg(p.theta + idx), __fmul_rn(sg, ld_noise1(trow + idx)));
    };
    __syncthreads();
    for (int i = tid; i < C1 * 256; i += kT) sW1[i] = par(L.c1w + i);
    for (int i = tid; i < C2 * 256; i += kT) sW2[i] = par(L.c2w + i);
    if (tid < 16) sSmall[tid] = par(L.c1b + tid);
    if (tid < 32) sSmall[16 + tid] = par(L.c2b + tid);
    if (tid < 16) sSmall[48 + tid] = par(L.b1 + tid);
    if (tid < 32) sSmall[64 + tid] = par(L.b2 + tid);
    __syncthreads();

    // conv1 of one image for this thread's spatial positions -> out[q][co]
    auto conv1_image = [&](const float* img, float (&out)[2][C1]) {
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int hw = tid + q * kT;
#pragma unroll
        for (int co = 0; co < C1; ++co) out[q][co] = sSmall[co];
        if (hw >= H1 * W1) continue;
        const int oh = hw / W1, ow = hw % W1;
        for (int ci = 0; ci < 4; ++ci) {
          for (int kh = 0; kh < 8; ++kh) {
            const float* src = img + (size_t)ci * 84 * 84 + (size_t)(oh * 4 + kh) * 84 + ow * 4;
            const float4 a = __ldg(reinterpret_cast<const float4*>(src));
            const float4 b = __ldg(reinterpret_cast<const float4*>(src + 4));
            const float x[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
            const int wofs = ci * 64 + kh * 8;
#pragma unroll
            for (int co = 0; co < C1; ++co) {
              const float* w = sW1 + co * 256 + wofs;
#pragma unroll
              for (int kw = 0; kw < 8; ++kw) out[q][co] = fmaf(x[kw], w[kw], out[q][co]);
            }
          }
        }
      }
    };

    // ---------------- phase B: reference batch through conv1, per-position statistics
    // Welford's update in frame order (welford_add): a sum of squares minus sum * mean cancels
    // catastrophically where the mean is large and the variance small, e.g. 0..255 pixels that never change.
    {
      float mean[2][C1], m2[2][C1];
#pragma unroll
      for (int q = 0; q < 2; ++q)
#pragma unroll
        for (int co = 0; co < C1; ++co) { mean[q][co] = 0.f; m2[q][co] = 0.f; }
      for (int r = 0; r < p.R; ++r) {
        float out[2][C1];
        conv1_image(p.xref + (size_t)r * IMG, out);
        const float inv = 1.f / (float)(r + 1);
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const int hw = tid + q * kT;
          if (hw >= H1 * W1) continue;
#pragma unroll
          for (int co = 0; co < C1; ++co) {
            const float y = out[q][co];
            R1[(size_t)r * P1 + co * (H1 * W1) + hw] = y;
            welford_add(y, inv, mean[q][co], m2[q][co]);
          }
        }
      }
      const float invR1 = 1.f / (float)(p.R - 1);
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int hw = tid + q * kT;
        if (hw >= H1 * W1) continue;
#pragma unroll
        for (int co = 0; co < C1; ++co) {
          const float var = m2[q][co] * invR1;   // unbiased (modules.py:52)
          const float a = par(L.g1 + co) / sqrtf(var + 1e-5f);
          sA1[co * (H1 * W1) + hw] = a;
          sM1[co * (H1 * W1) + hw] = mean[q][co];
        }
      }
    }
    __syncthreads();

    // conv2 of the image currently in sX1 for this thread's outputs o = tid + 256*i
    auto conv2_image = [&](float (&out)[11]) {
#pragma unroll
      for (int i = 0; i < 11; ++i) {
        const int o = tid + i * kT;
        out[i] = 0.f;
        if (o >= P2) continue;
        const int co = o / (H2 * W2), pos = o % (H2 * W2), oh = pos / W2, ow = pos % W2;
        float acc = sSmall[16 + co];
        const float* w = sW2 + co * 256;
        for (int ci = 0; ci < C1; ++ci) {
          const float* x = sX1 + ci * (H1 * W1) + (oh * 2) * W1 + ow * 2;
#pragma unroll
          for (int kh = 0; kh < 4; ++kh)
#pragma unroll
            for (int kw = 0; kw < 4; ++kw) acc = fmaf(x[kh * W1 + kw], w[ci * 16 + kh * 4 + kw], acc);
        }
        out[i] = acc;
      }
    };

    // ---------------- phase C: reference batch through VBN1/ReLU/conv2, statistics of layer 2
    {
      float mean[11], m2[11];
#pragma unroll
      for (int i = 0; i < 11; ++i) { mean[i] = 0.f; m2[i] = 0.f; }
      for (int r = 0; r < p.R; ++r) {
        __syncthreads();
        for (int i = tid; i < P1; i += kT)
          sX1[i] = fmaxf(fmaf(R1[(size_t)r * P1 + i] - sM1[i], sA1[i], sSmall[48 + i / (H1 * W1)]), 0.f);
        __syncthreads();
        float out[11];
        conv2_image(out);
        const float inv = 1.f / (float)(r + 1);
#pragma unroll
        for (int i = 0; i < 11; ++i) welford_add(out[i], inv, mean[i], m2[i]);
      }
      const float invR1 = 1.f / (float)(p.R - 1);
#pragma unroll
      for (int i = 0; i < 11; ++i) {
        const int o = tid + i * kT;
        if (o >= P2) continue;
        const int co = o / (H2 * W2);
        const float a = par(L.g2 + co) / sqrtf(m2[i] * invR1 + 1e-5f);
        sA2[o] = a;
        sM2[o] = mean[i];
      }
    }
    __syncthreads();

    // ---------------- phase D: observation batch -> flattened conv features XS[b][2592]
    for (int b = 0; b < p.B; ++b) {
      float out1[2][C1];
      conv1_image(p.obs + (size_t)b * IMG, out1);
      __syncthreads();   // previous image's conv2 finished reading sX1
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int hw = tid + q * kT;
        if (hw >= H1 * W1) continue;
#pragma unroll
        for (int co = 0; co < C1; ++co) {
          const int i = co * (H1 * W1) + hw;
          sX1[i] = fmaxf(fmaf(out1[q][co] - sM1[i], sA1[i], sSmall[48 + co]), 0.f);
        }
      }
      __syncthreads();
      float out2[11];
      conv2_image(out2);
#pragma unroll
      for (int i = 0; i < 11; ++i) {
        const int o = tid + i * kT;
        if (o < P2) XS[(size_t)b * P2 + o] = fmaxf(fmaf(out2[i] - sM2[o], sA2[o], sSmall[64 + o / (H2 * W2)]), 0.f);
      }
    }
    __syncthreads();

    // ---------------- phase E: fc1 (thread = output neuron), ReLU, fc2, squared error
    float loss = 0.f;
    for (int b0 = 0; b0 < p.B; b0 += TB) {
      const int nb = min(TB, p.B - b0);
      float acc[TB];
#pragma unroll
      for (int i = 0; i < TB; ++i) acc[i] = 0.f;
      for (int k0 = 0; k0 < P2; k0 += KT) {
        __syncthreads();
        for (int e = tid; e < FC1 * KT; e += kT) {      // weight tile, coalesced along k
          const int k = e % KT, jn = e / KT;
          sWt[k * (FC1 + 1) + jn] = par(L.f1w + (int64_t)jn * P2 + k0 + k);
        }
        for (int e = tid; e < TB * KT; e += kT) {
          const int k = e % KT, bi = e / KT;
          sXt[bi * KT + k] = (bi < nb) ? XS[(size_t)(b0 + bi) * P2 + k0 + k] : 0.f;
        }
        __syncthreads();
#pragma unroll 4
        for (int k = 0; k < KT; ++k) {
          const float w = sWt[k * (FC1 + 1) + tid];
#pragma unroll
          for (int bi = 0; bi < TB; ++bi) acc[bi] = fmaf(w, sXt[bi * KT + k], acc[bi]);
        }
      }
      const float bias = par(L.f1b + tid);
      __syncthreads();
#pragma unroll
      for (int bi = 0; bi < TB; ++bi) sHs[bi * FC1 + tid] = fmaxf(acc[bi] + bias, 0.f);
      __syncthreads();
      for (int e = tid; e < nb * p.A; e += kT) {
        const int bi = e / p.A, a = e % p.A;
        float y = par(L.f2b + a);
        for (int k = 0; k < FC1; ++k) y = fmaf(sHs[bi * FC1 + k], par(L.f2w + (int64_t)a * FC1 + k), y);
        const float d = y - __ldg(p.target + (size_t)(b0 + bi) * p.A + a);
        loss = fmaf(d, d, loss);
      }
    }
    loss = warp_sum_f(loss);
    if ((tid & 31) == 0) s_red[tid >> 5] = loss;
    __syncthreads();
    if (tid == 0) {
      float s = 0.f;
      for (int w = 0; w < kT / 32; ++w) s += s_red[w];
      const float r = -(s / ((float)p.B * (float)p.A));
      if (centre) p.ret_plus[0] = r;
      else if (minus) p.ret_minus[j] = r;
      else p.ret_plus[j] = r;
    }
    __syncthreads();
  }
}

size_t conv_smem_bytes() {
  const size_t fc_tile = (size_t)KT * (FC1 + 1) + (size_t)TB * KT;     // aliases the sX1 region in phase E
  const size_t tail = fc_tile > (size_t)P1 ? fc_tile : (size_t)P1;
  return sizeof(float) * ((size_t)C1 * 256 + (size_t)C2 * 256 + 128 + 2 * (size_t)P1 + 2 * (size_t)P2 + tail);
}

}  // namespace

extern "C" int64_t estk_eval_conv_vbn_scratch_bytes(estk_ctx* ctx, int32_t precision, int32_t ref_batch, int32_t B) {
  if (!ctx || ref_batch < 2 || B < 1) return -1;
  if (precision == ESTK_PREC_F16) return (int64_t)ctx->sm_count * eval_conv_tc_scratch_per_cta(ref_batch, B);
  if (precision != ESTK_PREC_FP32) return -1;
  return (int64_t)ctx->sm_count * ((int64_t)ref_batch * P1 + (int64_t)B * P2) * (int64_t)sizeof(float);
}

extern "C" int estk_eval_conv_vbn(estk_ctx* ctx, int32_t precision, int32_t n_actions, const float* theta,
                                  const float* table, const uint16_t* table16,
                                  const int64_t* offsets, const int32_t* order, int32_t pairs, float sigma,
                                  const float* xref, int32_t ref_batch, const float* obs, const float* target,
                                  int32_t B, float* returns_plus, float* returns_minus, void* scratch,
                                  int64_t scratch_bytes, void* stream) {
  const bool f16 = precision == ESTK_PREC_F16;
  const EvalConvCall c = {precision, n_actions, ref_batch, B, theta, table, table16, offsets, order, pairs, sigma,
                          xref, obs, target, returns_plus, returns_minus, scratch, scratch_bytes};
  if (((n_actions >> 16) & 0xff) == (ESTK_ACTIONS >> 16)) return eval_conv_actions(ctx, c, (cudaStream_t)stream);
  ESTK_CHECK_ARG(ctx && theta && xref && obs && target && returns_plus && scratch, "estk_eval_conv_vbn: null argument");
  ESTK_CHECK_ARG(offsets == nullptr || (table && (table16 || !f16) && returns_minus),
                 "estk_eval_conv_vbn: table%s/returns_minus required with offsets", f16 ? "/table16" : "");
  ESTK_CHECK_ARG(n_actions >= 1 && n_actions <= 64, "estk_eval_conv_vbn: n_actions=%d", n_actions);
  ESTK_CHECK_ARG(ref_batch >= 2 && B >= 1, "estk_eval_conv_vbn: ref_batch must be >= 2 (unbiased variance), B >= 1");
  ESTK_CHECK_ARG(pairs >= 1 && pairs <= ESTK_MAX_POPULATION / 2, "estk_eval_conv_vbn: pairs=%d", pairs);
  ESTK_CHECK_ARG(ESTK_ALIGNED16(xref) && ESTK_ALIGNED16(obs), "estk_eval_conv_vbn: images must be 16-byte aligned");
  ESTK_CHECK_ARG(!f16 || (ESTK_ALIGNED16(theta) && ESTK_ALIGNED16(scratch) && (table16 == nullptr || ESTK_ALIGNED16(table16))),
                 "estk_eval_conv_vbn: f16 needs theta, table16 and scratch 16-byte aligned");
  if (!f16 && precision != ESTK_PREC_FP32) {
    estk_set_error("estk_eval_conv_vbn: precision %d is not supported (ESTK_PREC_FP32 or ESTK_PREC_F16)", precision);
    return ESTK_ERR_UNSUPPORTED;
  }
  const int64_t need = estk_eval_conv_vbn_scratch_bytes(ctx, precision, ref_batch, B);
  ESTK_CHECK_ARG(scratch_bytes >= need, "estk_eval_conv_vbn: scratch %lld < %lld bytes", (long long)scratch_bytes, (long long)need);
  if (f16) return eval_conv_tc(ctx, c, (cudaStream_t)stream);
  ConvParams p = {};
  p.theta = theta; p.table = table; p.offsets = offsets; p.order = order; p.pairs = pairs; p.sigma = sigma;
  p.A = n_actions; p.R = ref_batch; p.B = B; p.xref = xref; p.obs = obs; p.target = target;
  p.ret_plus = returns_plus; p.ret_minus = returns_minus;
  p.scratch = reinterpret_cast<float*>(scratch);
  p.scratch_per_cta = (int64_t)ref_batch * P1 + (int64_t)B * P2;
  p.members = offsets ? 2 * pairs : 1;
  const size_t smem = conv_smem_bytes();
  ESTK_CUDA(cudaFuncSetAttribute(eval_conv_vbn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int grid = ctx->sm_count;
  if (grid > p.members) grid = p.members;
  eval_conv_vbn_kernel<<<grid, kT, smem, (cudaStream_t)stream>>>(p);
  ESTK_CUDA(cudaGetLastError());
  return ESTK_OK;
}
