// estk_act_conv.cu -- estk_eval_conv_vbn with n_actions | ESTK_ACTIONS (fp32): the VirtualBatchNorm
// statistics of every perturbed Atari policy once per generation, then every member's outputs on that
// member's own frames, the per-step operation of an environment population.
//
// Replaces (reference file:line):
//   Policy.forward           examples/atari.py:25-37: the reference batch xref runs through conv1/VBN1/
//                            conv2/VBN2 on EVERY call to get the VBN statistics.  They depend only on the
//                            member's weights and xref, so here they are computed once per member
//                            (conv_stats_kernel) and each environment step reuses them (conv_act_kernel).
//   VirtualBatchNorm.forward estorch/modules.py:48-58 (mean / unbiased variance over the reference batch)
//
// conv_stats_kernel: phases B-C of eval_conv_vbn_kernel (estk_eval_conv.cu) with the same arithmetic in
// the same order -- one persistent CTA per member, the R raw conv1 outputs in a per-CTA slab of the
// context workspace -- writing the VBN scale a = gamma / sqrtf(var + 1e-5f) and the mean (Welford's update) to
// stats[member][ESTK_CONV_VBN_STATS_FLOATS] instead of shared memory.
//
// conv_act_kernel: one CTA per antithetic pair x chunk of NB frames per member.  The pair's noise is read
// once and serves both signs: conv1 / conv2 weights are formed as W+ = theta + sigma*t and
// W- = theta - sigma*t in shared memory (2 x 48 KB); each sign's frames go through conv1, VBN1 (that
// member's stats, coalesced loads), ReLU, conv2, VBN2, ReLU into features [2][NB][2592] (shared memory
// for NB <= 4, a workspace slab for NB = 8); fc1 is tiled over k (each W+/W- tile from one noise read,
// aliasing the dead conv weights); fc2 last.  Per element the arithmetic of eval_conv_vbn_kernel: fmaf
// chains from the bias in (ci, kh, kw) order, fmaxf(fmaf(y - mean, a, beta), 0), fc1 one chain from 0 in
// ascending k then + bias and ReLU, fc2 one chain from the bias -- so a member's outputs are the bits
// of the y its fp32 evaluate computes.  No atomics: the same bits from run to run.
//
// Occupancy: a CTA holds 145-207 KB of shared memory (1 per SM) and there are pairs x chunks of them;
// at the reference's P = 100, B = 1 that is 50 CTAs on 132 SMs.  The k-split of fc1 across CTAs that
// would fill the rest needs a combine pass; DESIGN.md section 4.7 has the measured cost of not doing it.
#include "estk_common.cuh"

namespace {

constexpr int kT = 256;
constexpr int C1 = 16, H1 = 20, W1 = 20, P1 = C1 * H1 * W1;   // 6400
constexpr int C2 = 32, H2 = 9, W2 = 9, P2 = C2 * H2 * W2;     // 2592
constexpr int IMG = 4 * 84 * 84;
constexpr int FC1 = 256;
constexpr int KT = 32;                                         // k-tile of fc1 (2592 = 81 tiles)
constexpr int FC2_AT = 32;                                     // fc2 outputs per formed weight tile
constexpr int kStats = 2 * P1 + 2 * P2;
static_assert(kStats == ESTK_CONV_VBN_STATS_FLOATS, "stats layout: a1, mean1 [6400], a2, mean2 [2592]");

// parameter offsets, registration order of examples/atari.py:17-23
constexpr int64_t oC1W = 0, oC1B = 4096, oG1 = 4112, oB1 = 4128, oC2W = 4144, oC2B = 12336, oG2 = 12368,
                  oB2 = 12400, oF1W = 12432, oF1B = oF1W + (int64_t)FC1 * P2, oF2W = oF1B + FC1;

struct StatsParams {
  const float* theta;
  const float* table;
  const uint16_t* table16;
  const int64_t* offsets;   // null => centre
  const int32_t* order;
  int pairs;
  float sigma;
  int R;
  const float* xref;
  float* stats;             // [members][kStats]
  float* slab;              // per CTA [R][P1]
  int members;
};

__global__ void __launch_bounds__(kT, 1) conv_stats_kernel(const StatsParams p) {
  extern __shared__ __align__(16) float sm[];
  float* sW1 = sm;                    // [16][256]
  float* sW2 = sW1 + C1 * 256;        // [32][256]
  float* sSmall = sW2 + C2 * 256;     // conv1.b 16, conv2.b 32, bn1.b 16  (64)
  float* sA1 = sSmall + 64;           // [6400]
  float* sM1 = sA1 + P1;              // [6400]
  float* sX1 = sM1 + P1;              // [6400] normalised layer-1 activations of one reference frame

  const int tid = threadIdx.x;
  const bool centre = (p.offsets == nullptr);
  float* R1 = p.slab + (int64_t)blockIdx.x * p.R * P1;   // [R][P1]

  for (int member = blockIdx.x; member < p.members; member += gridDim.x) {
    const int pairs = p.pairs;
    const bool minus = (!centre) && member >= pairs;
    const int slot = centre ? 0 : (minus ? member - pairs : member);
    const int j = (!centre && p.order) ? p.order[slot] : slot;
    const NoiseRow nz = noise_row(p.theta, p.table, p.table16, p.offsets, j);
    const float sg = centre ? 0.f : (minus ? -p.sigma : p.sigma);
    float* const st = p.stats + (int64_t)(minus ? pairs + j : j) * kStats;
    auto par = [&](int64_t idx) -> float {   // perturbed parameter, the evaluate's two roundings
      return __fadd_rn(__ldg(p.theta + idx), __fmul_rn(sg, nz(idx)));
    };
    __syncthreads();
    for (int i = tid; i < C1 * 256; i += kT) sW1[i] = par(oC1W + i);
    for (int i = tid; i < C2 * 256; i += kT) sW2[i] = par(oC2W + i);
    if (tid < 16) sSmall[tid] = par(oC1B + tid);
    if (tid < 32) sSmall[16 + tid] = par(oC2B + tid);
    if (tid < 16) sSmall[48 + tid] = par(oB1 + tid);
    __syncthreads();

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

    // ---------------- reference batch through conv1, per-position statistics of layer 1
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
          const float a = par(oG1 + co) / sqrtf(var + 1e-5f);
          const int i = co * (H1 * W1) + hw;
          sA1[i] = a;
          sM1[i] = mean[q][co];
          st[i] = a;
          st[P1 + i] = mean[q][co];
        }
      }
    }
    __syncthreads();

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

    // ---------------- reference batch through VBN1 / ReLU / conv2, statistics of layer 2
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
        const float a = par(oG2 + co) / sqrtf(m2[i] * invR1 + 1e-5f);
        st[2 * P1 + o] = a;
        st[2 * P1 + P2 + o] = mean[i];
      }
    }
  }
}

size_t stats_smem_bytes() { return sizeof(float) * ((size_t)C1 * 256 + (size_t)C2 * 256 + 64 + 3 * (size_t)P1); }

struct ActParams {
  const float* theta;
  const float* table;
  const uint16_t* table16;
  const int64_t* offsets;   // null => centre (theta, one member)
  const int32_t* order;
  int pairs;
  float sigma;
  int A, B, chunks;
  const float* obs;         // population [2*pairs][B][4][84][84], centre [B][4][84][84]
  const float* stats;       // [members][kStats]
  float* out_plus;          // [pairs][B][A] (centre [B][A])
  float* out_minus;         // [pairs][B][A]
  float* slab;              // SLAB: per CTA [2][NB][P2]
};

// shared memory: conv weights of both signs, biases, one layer-1 frame, then the features unless SLAB
constexpr int kActW = 2 * C1 * 256 + 2 * C2 * 256;   // 24576 floats; fc1 / fc2 tiles alias it later
constexpr int kActHead = kActW + 224 + P1;
static_assert(2 * KT * (FC1 + 1) + 2 * 8 * FC1 <= kActW, "fc1 tiles + hidden rows fit in the conv-weight region");
static_assert(2 * FC2_AT * FC1 + 2 * 8 * FC1 <= kActW, "fc2 tiles + hidden rows fit in the conv-weight region");

template <int NB, bool SLAB>
__global__ void __launch_bounds__(kT, 1) conv_act_kernel(const ActParams p) {
  extern __shared__ __align__(16) float sm[];
  float* const sW1 = sm;                   // [2][16][256]  (+, -)
  float* const sW2 = sW1 + 2 * C1 * 256;   // [2][32][256]
  float* const sB = sm + kActW;            // conv1.b [2][16], conv2.b [2][32], bn1.b [2][16], bn2.b [2][32]
  float* const sX1 = sB + 224;             // [6400]
  float* const sWtp = sm;                  // fc1: [KT][FC1+1] W+, then W-  (aliases sW1 / sW2)
  float* const sWtm = sWtp + KT * (FC1 + 1);
  float* const sH = sm + 2 * KT * (FC1 + 1);    // [2][NB][FC1] hidden rows (+ rows, then - rows)
  float* const sV = sm;                    // fc2: [2][FC2_AT][FC1] weights of both signs
  float* const F = SLAB ? p.slab + (size_t)blockIdx.x * 2 * NB * P2 : sm + kActHead;   // [2][NB][P2]

  const int tid = threadIdx.x;
  const bool centre = (p.offsets == nullptr);
  const float sigma = centre ? 0.f : p.sigma;
  const int A = p.A;
  const int64_t oF2B = oF2W + (int64_t)A * FC1;
  const int items = p.pairs * p.chunks;

  for (int item = blockIdx.x; item < items; item += gridDim.x) {
    const int slot = item / p.chunks, chunk = item % p.chunks;
    const int j = (!centre && p.order) ? p.order[slot] : slot;
    const NoiseRow nz = noise_row(p.theta, p.table, p.table16, p.offsets, j);
    const int b0 = chunk * NB, nb = min(NB, p.B - b0);
    const int signs = centre ? 1 : 2;

    __syncthreads();   // the previous item's readers of shared memory are done
    for (int i = tid; i < C1 * 256; i += kT) estk_form_pm(p.theta, nz, sigma, oC1W + i, sW1[i], sW1[C1 * 256 + i]);
    for (int i = tid; i < C2 * 256; i += kT) estk_form_pm(p.theta, nz, sigma, oC2W + i, sW2[i], sW2[C2 * 256 + i]);
    if (tid < 16) estk_form_pm(p.theta, nz, sigma, oC1B + tid, sB[tid], sB[16 + tid]);
    if (tid < 32) estk_form_pm(p.theta, nz, sigma, oC2B + tid, sB[32 + tid], sB[64 + tid]);
    if (tid < 16) estk_form_pm(p.theta, nz, sigma, oB1 + tid, sB[96 + tid], sB[112 + tid]);
    if (tid < 32) estk_form_pm(p.theta, nz, sigma, oB2 + tid, sB[128 + tid], sB[160 + tid]);
    __syncthreads();

    // ---------------- each sign's frames: conv1, VBN1, ReLU, conv2, VBN2, ReLU -> F[s][b]
    for (int s = 0; s < signs; ++s) {
      const int64_t member = s ? (int64_t)p.pairs + j : j;
      const float* const st = p.stats + member * kStats;
      const float* const W1s = sW1 + s * C1 * 256;
      const float* const W2s = sW2 + s * C2 * 256;
      const float* const b1s = sB + s * 16;
      const float* const b2s = sB + 32 + s * 32;
      const float* const be1s = sB + 96 + s * 16;
      const float* const be2s = sB + 128 + s * 32;
      for (int bl = 0; bl < nb; ++bl) {
        const float* const img = p.obs + ((size_t)member * p.B + b0 + bl) * IMG;
        float out1[2][C1];
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const int hw = tid + q * kT;
#pragma unroll
          for (int co = 0; co < C1; ++co) out1[q][co] = b1s[co];
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
                const float* w = W1s + co * 256 + wofs;
#pragma unroll
                for (int kw = 0; kw < 8; ++kw) out1[q][co] = fmaf(x[kw], w[kw], out1[q][co]);
              }
            }
          }
        }
        __syncthreads();   // the previous frame's conv2 finished reading sX1
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const int hw = tid + q * kT;
          if (hw >= H1 * W1) continue;
#pragma unroll
          for (int co = 0; co < C1; ++co) {
            const int i = co * (H1 * W1) + hw;
            sX1[i] = fmaxf(fmaf(out1[q][co] - __ldg(st + P1 + i), __ldg(st + i), be1s[co]), 0.f);
          }
        }
        __syncthreads();
        float* const Fr = F + (size_t)(s * NB + bl) * P2;
#pragma unroll
        for (int i = 0; i < 11; ++i) {
          const int o = tid + i * kT;
          if (o >= P2) continue;
          const int co = o / (H2 * W2), pos = o % (H2 * W2), oh = pos / W2, ow = pos % W2;
          float acc = b2s[co];
          const float* w = W2s + co * 256;
          for (int ci = 0; ci < C1; ++ci) {
            const float* x = sX1 + ci * (H1 * W1) + (oh * 2) * W1 + ow * 2;
#pragma unroll
            for (int kh = 0; kh < 4; ++kh)
#pragma unroll
              for (int kw = 0; kw < 4; ++kw) acc = fmaf(x[kh * W1 + kw], w[ci * 16 + kh * 4 + kw], acc);
          }
          Fr[o] = fmaxf(fmaf(acc - __ldg(st + 2 * P1 + P2 + o), __ldg(st + 2 * P1 + o), be2s[co]), 0.f);
        }
      }
    }

    // ---------------- fc1: thread = output neuron, one chain per row from 0 in ascending k
    float accp[NB], accm[NB];
#pragma unroll
    for (int i = 0; i < NB; ++i) { accp[i] = 0.f; accm[i] = 0.f; }
    const float* const Fp = F;
    const float* const Fm = F + (size_t)NB * P2;
    for (int k0 = 0; k0 < P2; k0 += KT) {
      __syncthreads();   // features written / the previous tile consumed
      for (int e = tid; e < FC1 * KT; e += kT) {      // one noise read per weight, both signs; coalesced along k
        const int k = e % KT, jn = e / KT;
        estk_form_pm(p.theta, nz, sigma, oF1W + (int64_t)jn * P2 + k0 + k, sWtp[k * (FC1 + 1) + jn],
                     sWtm[k * (FC1 + 1) + jn]);
      }
      __syncthreads();
#pragma unroll 4
      for (int k = 0; k < KT; ++k) {
        const float wp = sWtp[k * (FC1 + 1) + tid], wm = sWtm[k * (FC1 + 1) + tid];
#pragma unroll
        for (int i = 0; i < NB; ++i) {
          accp[i] = fmaf(wp, Fp[(size_t)i * P2 + k0 + k], accp[i]);
          accm[i] = fmaf(wm, Fm[(size_t)i * P2 + k0 + k], accm[i]);
        }
      }
    }
    {
      float bp, bm;
      estk_form_pm(p.theta, nz, sigma, oF1B + tid, bp, bm);
#pragma unroll
      for (int i = 0; i < NB; ++i) {
        sH[i * FC1 + tid] = fmaxf(accp[i] + bp, 0.f);
        sH[(NB + i) * FC1 + tid] = fmaxf(accm[i] + bm, 0.f);
      }
    }

    // ---------------- fc2: one chain per (row, action) from the bias, weights formed FC2_AT actions at a time
    for (int a0 = 0; a0 < A; a0 += FC2_AT) {
      const int na = min(FC2_AT, A - a0);
      __syncthreads();   // fc1 tiles / the previous fc2 tile consumed, sH written
      for (int e = tid; e < na * FC1; e += kT)
        estk_form_pm(p.theta, nz, sigma, oF2W + (int64_t)a0 * FC1 + e, sV[e], sV[FC2_AT * FC1 + e]);
      __syncthreads();
      for (int e = tid; e < signs * nb * na; e += kT) {
        const int a = e % na, r = e / na, s = r / nb, bl = r % nb;
        float bp, bm;
        estk_form_pm(p.theta, nz, sigma, oF2B + a0 + a, bp, bm);
        float y = s ? bm : bp;
        const float* const h = sH + (s * NB + bl) * FC1;
        const float* const w = sV + s * FC2_AT * FC1 + a * FC1;
        for (int k = 0; k < FC1; ++k) y = fmaf(h[k], w[k], y);
        float* const out = s ? p.out_minus : p.out_plus;
        out[((size_t)j * p.B + b0 + bl) * A + a0 + a] = y;
      }
    }
  }
}

size_t act_smem_bytes(int nb, bool slab) {
  return sizeof(float) * ((size_t)kActHead + (slab ? 0 : (size_t)2 * nb * P2));
}

template <int NB>
int launch_act(estk_ctx* ctx, ActParams& p, cudaStream_t stream) {
  constexpr bool SLAB = NB == 8;
  auto kern = conv_act_kernel<NB, SLAB>;
  const size_t smem = act_smem_bytes(NB, SLAB);
  ESTK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int64_t items = (int64_t)p.pairs * p.chunks;
  int grid = (int)std::min<int64_t>(items, INT_MAX);
  if (SLAB) {   // persistent: the slab the caller reserved holds sm_count CTAs' features
    grid = (int)std::min<int64_t>(items, ctx->sm_count);
    p.slab = ctx->eval_slab;
  }
  kern<<<grid, kT, smem, stream>>>(p);
  ESTK_CUDA(cudaGetLastError());
  return ESTK_OK;
}

}  // namespace

int eval_conv_actions(estk_ctx* ctx, const EvalConvCall& c, cudaStream_t stream) {
  const char* who = "estk_eval_conv_vbn[ESTK_ACTIONS]";
  if (c.precision != ESTK_PREC_FP32) {
    estk_set_error("%s: actions are computed with ESTK_PREC_FP32 only (precision %d)", who, c.precision);
    return ESTK_ERR_UNSUPPORTED;
  }
  const int A = c.A & 0xff;
  const bool centre = c.offsets == nullptr;
  ESTK_CHECK_ARG((c.A & ~0xff) == ESTK_ACTIONS && A >= 1 && A <= 64,
                 "%s: n_actions=0x%x (bits 0-7 the action count 1..64, bits 8-15 zero, bits 16-23 ESTK_ACTIONS)",
                 who, (unsigned)c.A);
  ESTK_CHECK_ARG(c.xref || c.obs,
                 "%s: xref and obs are both NULL (a call runs the stats phase, the act phase or both)", who);
  ESTK_CHECK_ARG(ctx && c.theta && c.scratch && (centre || c.table || c.table16),
                 "%s: null argument (theta, scratch, and for a population table or table16)", who);
  ESTK_CHECK_ARG(!c.obs || (c.ret_plus && (centre || c.ret_minus)),
                 "%s: the act phase needs returns_plus (and returns_minus for a population)", who);
  ESTK_CHECK_ARG(centre || (c.pairs >= 1 && c.pairs <= ESTK_MAX_POPULATION / 2), "%s: pairs=%d", who, c.pairs);
  ESTK_CHECK_ARG(!c.xref || (c.R >= 2 && ESTK_ALIGNED16(c.xref)),
                 "%s: the stats phase needs ref_batch >= 2 (unbiased variance) and a 16-byte aligned xref", who);
  ESTK_CHECK_ARG(!c.obs || (c.B >= 1 && ESTK_ALIGNED16(c.obs)),
                 "%s: the act phase needs B >= 1 and 16-byte aligned obs", who);
  ESTK_CHECK_ARG(ESTK_ALIGNED16(c.scratch), "%s: scratch must be 16-byte aligned", who);
  const int members = centre ? 1 : 2 * c.pairs;
  const int64_t need = (int64_t)members * ESTK_CONV_VBN_STATS_FLOATS * (int64_t)sizeof(float);
  ESTK_CHECK_ARG(c.scratch_bytes >= need,
                 "%s: scratch %lld < %lld bytes (members * ESTK_CONV_VBN_STATS_FLOATS * 4)", who,
                 (long long)c.scratch_bytes, (long long)need);

  const int B = c.B, nb = c.obs ? estk_chunk_rows(B) : 1;
  const int stats_grid = std::min(ctx->sm_count, members);
  const int64_t chunks = c.obs ? (B + nb - 1) / nb : 1;
  const int act_grid = (int)std::min<int64_t>((centre ? 1 : c.pairs) * chunks, ctx->sm_count);
  int64_t slab = 0;
  if (c.xref) slab = (int64_t)stats_grid * c.R * P1;
  if (c.obs && nb == 8) slab = std::max<int64_t>(slab, (int64_t)act_grid * 2 * 8 * P2);
  if (slab) {
    const int rc = estk_ctx_reserve(ctx, 0, 0, stream, who, slab);
    if (rc) return rc;
  }
  float* const stats = reinterpret_cast<float*>(c.scratch);
  if (c.xref) {
    StatsParams s = {};
    s.theta = c.theta; s.offsets = c.offsets; s.R = c.R; s.xref = c.xref; s.stats = stats; s.slab = ctx->eval_slab;
    s.members = members;
    if (centre) {
      s.pairs = 1;
    } else {
      s.table = c.table; s.table16 = c.table16; s.order = c.order; s.pairs = c.pairs; s.sigma = c.sigma;
    }
    const size_t smem = stats_smem_bytes();
    ESTK_CUDA(cudaFuncSetAttribute(conv_stats_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    conv_stats_kernel<<<stats_grid, kT, smem, stream>>>(s);
    ESTK_CUDA(cudaGetLastError());
  }
  if (!c.obs) return ESTK_OK;
  ActParams a = {};
  a.theta = c.theta; a.offsets = c.offsets; a.A = A; a.B = B; a.chunks = (int)chunks; a.obs = c.obs; a.stats = stats;
  a.out_plus = c.ret_plus;
  if (centre) {
    a.pairs = 1;
  } else {
    a.table = c.table; a.table16 = c.table16; a.order = c.order; a.pairs = c.pairs; a.sigma = c.sigma;
    a.out_minus = c.ret_minus;
  }
  return estk_dispatch(EstkChunkRows{}, nb, [&](auto NB) { return launch_act<NB>(ctx, a, stream); });
}
