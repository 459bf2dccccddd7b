// estk_eval_conv_tc.cu -- tensor-core population evaluate ("f16") for the conv +
// VirtualBatchNorm policy of the reference's Atari example.
//
// Same function as estk_eval_conv.cu (examples/atari.py:25-37, estorch/modules.py:42-58,
// estorch.py:195-202), same parameter layout, same output placement.  The three GEMMs
// (conv1 as an implicit GEMM, conv2 as an implicit GEMM, fc1) run on the tensor cores with
// mma.sync.m16n8k16 (fp16 operands, fp32 accumulation); VBN statistics, normalisation,
// fc2 and the loss stay fp32 on the CUDA cores.
//
// Arithmetic (DESIGN §4.5).  Every GEMM operand v -- formed weight W = theta + s*sigma*eps
// (fp32, eps read from the exact fp16 table copy), network input, normalised activation --
// is split into two fp16 values
//     v_hi = rn_f16(v),   v_lo = rn_f16((v - v_hi) * 2^12)
// and each product is taken as  a_hi*b_hi + 2^-12 * (a_hi*b_lo + a_lo*b_hi)  with the two
// sums in separate fp32 accumulators.  That carries 22 significant bits per operand: with
// one fp16 rounding per weight this policy's returns move by 1e-4..2e-4 (max-norm relative)
// from the fp32 forward, because every VBN layer renormalises the rounding error back to
// unit scale; with the split they stay within the fp32 parity bar.  The 2^12 scale keeps
// v_lo out of the fp16 subnormal range for every |v| >= 2^-14.
//
// Work decomposition: one persistent 256-thread CTA per member (grid = #SMs).
//   B  reference frames -> conv1 (25 m16 position tiles x 16 channels per frame);
//      raw outputs go to a per-CTA global slab, shifted sums for mean / unbiased variance
//      accumulate in shared memory (each (c,h,w) entry is owned by one thread: no atomics)
//   C  reference frames: slab -> VBN1 -> ReLU -> split -> conv2 (6 m16 tiles x 32) -> stats
//   D  observations: conv1 -> VBN1 -> ReLU -> conv2 -> VBN2 -> ReLU -> split features (slab)
//   E  fc1 transposed (D[256 x 32 obs] = W X^T, W formed straight into A fragments),
//      bias + ReLU, fc2 + squared error in fp32, fixed-order loss combine.
#include "estk_common.cuh"
#include <cuda_fp16.h>

namespace {

constexpr int kT = 256;                       // 8 warps
constexpr int C1 = 16, H1 = 20, W1 = 20, HW1 = H1 * W1, P1 = C1 * HW1;   // 6400
constexpr int C2 = 32, H2 = 9, W2 = 9, HW2 = H2 * W2, P2 = C2 * HW2;     // 2592
constexpr int IMG = 4 * 84 * 84, CH = 84 * 84;
constexpr int FC1 = 256;
constexpr int NB = 32;                        // observations per fc1 tile (4 n8 fragments)
constexpr int KPAD = 264;                     // row pitch (halves) of the conv weight tiles: conflict-free B loads
constexpr float kLo = 4096.f, kLoInv = 1.f / 4096.f;

struct ConvTcParams {
  const float* theta;
  const __half* table16;
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
  unsigned char* scratch;  // per CTA: R1 [R][P1] fp32, then XS hi / lo [B][P2] fp16 each
  int64_t scratch_per_cta;
  int members;
};

constexpr int64_t kC1w = 0, kC1b = 4096, kG1 = 4112, kB1 = 4128, kC2w = 4144, kC2b = 12336, kG2 = 12368,
                  kB2 = 12400, kF1w = 12432, kF1b = kF1w + (int64_t)FC1 * P2, kF2w = kF1b + FC1;

// ---------------------------------------------------------------- split operands, mma
__device__ __forceinline__ void split2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  const __half h0 = __float2half_rn(x0), h1 = __float2half_rn(x1);
  const __half l0 = __float2half_rn((x0 - __half2float(h0)) * kLo);
  const __half l1 = __float2half_rn((x1 - __half2float(h1)) * kLo);
  hi = (uint32_t)__half_as_ushort(h0) | ((uint32_t)__half_as_ushort(h1) << 16);
  lo = (uint32_t)__half_as_ushort(l0) | ((uint32_t)__half_as_ushort(l1) << 16);
}
__device__ __forceinline__ void split1(float x, __half& hi, __half& lo) {
  hi = __float2half_rn(x);
  lo = __float2half_rn((x - __half2float(hi)) * kLo);
}

// d += a * b, m16n8k16, row.col, fp16 operands, fp32 accumulators
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
               "{%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// split product: main += a_hi b_hi, corr += a_hi b_lo + a_lo b_hi
__device__ __forceinline__ void mma3(float (&m)[4], float (&c)[4], const uint32_t (&ah)[4], const uint32_t (&al)[4],
                                     uint32_t bh0, uint32_t bh1, uint32_t bl0, uint32_t bl1) {
  mma16816(m, ah, bh0, bh1);
  mma16816(c, ah, bl0, bl1);
  mma16816(c, al, bh0, bh1);
}
__device__ __forceinline__ uint32_t lds32(const __half* p) { return *reinterpret_cast<const uint32_t*>(p); }

struct Smem {
  __half w1h[C1 * KPAD], w1l[C1 * KPAD];     // conv1 weights [co][k], k = ci*64 + kh*8 + kw
  __half w2h[C2 * KPAD], w2l[C2 * KPAD];     // conv2 weights [co][k], k = ci*16 + kh*4 + kw
  float s1[P1], q1[P1];                      // VBN1: shifted sums, then scale a / shift c
  float s2[P2], q2[P2], y2[P2];              // VBN2: shifted sums + shift, then a / c
  struct { __half h[CH], l[CH]; } img;       // one input channel, split
  union {
    float y1[P1];                            // VBN1 shift (first reference frame), phase B only
    struct { __half h[P1], l[P1]; } x1;      // one frame's normalised layer-1 map [c][h][w], split
  } u;
  float small[128];                          // conv1.b 16, conv2.b 32
  float red[kT / 32];
};
// the fc phase reuses s1 / q1 for the hidden activations [NB][FC1]
static_assert(2 * P1 >= NB * FC1, "fc1 activations alias the VBN1 statistics");

__global__ void __launch_bounds__(kT, 1) eval_conv_vbn_tc_kernel(const ConvTcParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Smem& S = *reinterpret_cast<Smem*>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const bool centre = (p.offsets == nullptr);
  float* R1 = reinterpret_cast<float*>(p.scratch + (int64_t)blockIdx.x * p.scratch_per_cta);   // [R][P1]
  __half* XSh = reinterpret_cast<__half*>(R1 + (int64_t)p.R * P1);                           // [B][P2]
  __half* XSl = XSh + (int64_t)p.B * P2;

  for (int member = blockIdx.x; member < p.members; member += gridDim.x) {
    const bool minus = (!centre) && member >= p.pairs;
    const int slot = centre ? 0 : (minus ? member - p.pairs : member);
    const int j = (!centre && p.order) ? p.order[slot] : slot;
    const __half* trow = centre ? nullptr : p.table16 + p.offsets[j];
    const float sg = centre ? 0.f : (minus ? -p.sigma : p.sigma);
    // perturbed parameter, the two roundings of estorch.py:189-192 (exact fp16 -> fp32 noise)
    auto par = [&](int64_t idx) -> float {
      const float e = centre ? 0.f : __half2float(trow[idx]);
      return __fadd_rn(__ldg(p.theta + idx), __fmul_rn(sg, e));
    };
    __syncthreads();   // previous member's fc phase is done with the shared memory
    for (int i = tid; i < C1 * 256; i += kT) {
      __half h, l;
      split1(par(kC1w + i), h, l);
      S.w1h[(i >> 8) * KPAD + (i & 255)] = h;
      S.w1l[(i >> 8) * KPAD + (i & 255)] = l;
    }
    for (int i = tid; i < C2 * 256; i += kT) {
      __half h, l;
      split1(par(kC2w + i), h, l);
      S.w2h[(i >> 8) * KPAD + (i & 255)] = h;
      S.w2l[(i >> 8) * KPAD + (i & 255)] = l;
    }
    if (tid < 16) S.small[tid] = par(kC1b + tid);
    if (tid < 32) S.small[16 + tid] = par(kC2b + tid);

    // ---- conv1 of one frame: warp w owns position tiles w, w+8, w+16 (and 24 for warp 0);
    //      epi(tile, nb, acc) receives acc[4] = outputs (pos g / g+8, channels nb*8+2t, +1), bias added
    auto conv1_frame = [&](const float* img, auto&& epi) {
      float am[4][2][4], ac[4][2][4];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int nb = 0; nb < 2; ++nb)
#pragma unroll
          for (int e = 0; e < 4; ++e) { am[i][nb][e] = 0.f; ac[i][nb][e] = 0.f; }
      const int ntiles = warp == 0 ? 4 : 3;
      for (int ci = 0; ci < 4; ++ci) {
        __syncthreads();   // previous channel (or the previous frame's readers) done with u.img
        const float4* src = reinterpret_cast<const float4*>(img + (size_t)ci * CH);
        for (int i = tid; i < CH / 4; i += kT) {
          const float4 v = __ldg(src + i);
          uint32_t h0, l0, h1, l1;
          split2(v.x, v.y, h0, l0);
          split2(v.z, v.w, h1, l1);
          *reinterpret_cast<uint2*>(S.img.h + 4 * i) = make_uint2(h0, h1);
          *reinterpret_cast<uint2*>(S.img.l + 4 * i) = make_uint2(l0, l1);
        }
        __syncthreads();
#pragma unroll
        for (int s = 0; s < 4; ++s) {   // k-step: kh = 2s (a0/a1) and 2s+1 (a2/a3), kw = 2t, 2t+1
          const int kb = ci * 64 + s * 16 + 2 * t;
          uint32_t bh[2][2], bl[2][2];
#pragma unroll
          for (int nb = 0; nb < 2; ++nb) {
            const int r = (nb * 8 + g) * KPAD + kb;
            bh[nb][0] = lds32(S.w1h + r); bh[nb][1] = lds32(S.w1h + r + 8);
            bl[nb][0] = lds32(S.w1l + r); bl[nb][1] = lds32(S.w1l + r + 8);
          }
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            if (i < ntiles) {
              const int pt = warp + 8 * i;
              const int p0 = pt * 16 + g, p1 = p0 + 8;
              const int o0 = ((p0 / W1) * 4 + 2 * s) * 84 + (p0 % W1) * 4 + 2 * t;
              const int o1 = ((p1 / W1) * 4 + 2 * s) * 84 + (p1 % W1) * 4 + 2 * t;
              const uint32_t ah[4] = {lds32(S.img.h + o0), lds32(S.img.h + o1), lds32(S.img.h + o0 + 84),
                                      lds32(S.img.h + o1 + 84)};
              const uint32_t al[4] = {lds32(S.img.l + o0), lds32(S.img.l + o1), lds32(S.img.l + o0 + 84),
                                      lds32(S.img.l + o1 + 84)};
#pragma unroll
              for (int nb = 0; nb < 2; ++nb) mma3(am[i][nb], ac[i][nb], ah, al, bh[nb][0], bh[nb][1], bl[nb][0], bl[nb][1]);
            }
          }
        }
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (i < ntiles) {
#pragma unroll
          for (int nb = 0; nb < 2; ++nb) {
            const float b0 = S.small[nb * 8 + 2 * t], b1 = S.small[nb * 8 + 2 * t + 1];
            float y[4];
            y[0] = fmaf(ac[i][nb][0], kLoInv, am[i][nb][0]) + b0;
            y[1] = fmaf(ac[i][nb][1], kLoInv, am[i][nb][1]) + b1;
            y[2] = fmaf(ac[i][nb][2], kLoInv, am[i][nb][2]) + b0;
            y[3] = fmaf(ac[i][nb][3], kLoInv, am[i][nb][3]) + b1;
            epi(warp + 8 * i, nb, y);
          }
        }
      }
    };

    // ---- conv2 of the map in x1h/x1l: 24 units (m16 tile mt = u % 6, channel block nb = u / 6),
    //      warp w owns units w, w+8, w+16; epi(mt, nb, y) as for conv1 (rows = positions, >= 81 ignored)
    auto conv2_frame = [&](auto&& epi) {
      float am[3][4], ac[3][4];
      int pa[3], pb[3];
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        const int u = warp + 8 * i, mt = u % 6;
        const int p0 = min(mt * 16 + g, HW2 - 1), p1 = min(mt * 16 + g + 8, HW2 - 1);
        pa[i] = (p0 / W2) * 2 * W1 + (p0 % W2) * 2;
        pb[i] = (p1 / W2) * 2 * W1 + (p1 % W2) * 2;
#pragma unroll
        for (int e = 0; e < 4; ++e) { am[i][e] = 0.f; ac[i][e] = 0.f; }
      }
      const int kofs = (t >> 1) * W1 + (t & 1) * 2;   // a0: kh = t/2, kw = 2(t%2); a2: kh + 2
#pragma unroll 2
      for (int ci = 0; ci < C1; ++ci) {
        const __half* xh = S.u.x1.h + ci * HW1 + kofs;
        const __half* xl = S.u.x1.l + ci * HW1 + kofs;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          const int nb = (warp + 8 * i) / 6;
          const int r = (nb * 8 + g) * KPAD + ci * 16 + 2 * t;
          const uint32_t ah[4] = {lds32(xh + pa[i]), lds32(xh + pb[i]), lds32(xh + pa[i] + 2 * W1), lds32(xh + pb[i] + 2 * W1)};
          const uint32_t al[4] = {lds32(xl + pa[i]), lds32(xl + pb[i]), lds32(xl + pa[i] + 2 * W1), lds32(xl + pb[i] + 2 * W1)};
          mma3(am[i], ac[i], ah, al, lds32(S.w2h + r), lds32(S.w2h + r + 8), lds32(S.w2l + r), lds32(S.w2l + r + 8));
        }
      }
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        const int u = warp + 8 * i, mt = u % 6, nb = u / 6;
        const float b0 = S.small[16 + nb * 8 + 2 * t], b1 = S.small[16 + nb * 8 + 2 * t + 1];
        float y[4];
        y[0] = fmaf(ac[i][0], kLoInv, am[i][0]) + b0;
        y[1] = fmaf(ac[i][1], kLoInv, am[i][1]) + b1;
        y[2] = fmaf(ac[i][2], kLoInv, am[i][2]) + b0;
        y[3] = fmaf(ac[i][3], kLoInv, am[i][3]) + b1;
        epi(mt, nb, y);
      }
    };
    // element e of an epilogue fragment -> (position row, channel)
    auto frag_pos = [&](int tile, int e) { return tile * 16 + g + ((e >> 1) << 3); };
    auto frag_ch = [&](int nb, int e) { return nb * 8 + 2 * t + (e & 1); };

    // ---------------- phase B: reference frames through conv1, VBN1 statistics
    // shifted sums around the first frame's value: mean = y0 + s/R, var = (q - s*s/R)/(R-1)
    for (int r = 0; r < p.R; ++r) {
      float* out = R1 + (size_t)r * P1;
      conv1_frame(p.xref + (size_t)r * IMG, [&](int pt, int nb, const float (&y)[4]) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int i = frag_ch(nb, e) * HW1 + frag_pos(pt, e);
          out[i] = y[e];
          if (r == 0) { S.u.y1[i] = y[e]; S.s1[i] = 0.f; S.q1[i] = 0.f; }
          else {
            const float d = y[e] - S.u.y1[i];
            S.s1[i] += d;
            S.q1[i] = fmaf(d, d, S.q1[i]);
          }
        }
      });
    }
    __syncthreads();
    {
      const float invR = 1.f / (float)p.R, invR1 = 1.f / (float)(p.R - 1);
      for (int i = tid; i < P1; i += kT) {
        const int co = i / HW1;
        const float s = S.s1[i];
        const float mean = S.u.y1[i] + s * invR;
        const float var = fmaxf((S.q1[i] - s * (s * invR)) * invR1, 0.f);   // unbiased (modules.py:52)
        const float a = par(kG1 + co) / sqrtf(var + 1e-5f);
        S.s1[i] = a;
        S.q1[i] = par(kB1 + co) - mean * a;
      }
    }

    // ---------------- phase C: reference frames through VBN1/ReLU/conv2, VBN2 statistics
    for (int r = 0; r < p.R; ++r) {
      __syncthreads();   // previous frame's conv2 done with x1 (and phase B's y1 reads done)
      const float* src = R1 + (size_t)r * P1;
      for (int i = tid; i < P1; i += kT) {
        __half h, l;
        split1(fmaxf(fmaf(src[i], S.s1[i], S.q1[i]), 0.f), h, l);
        S.u.x1.h[i] = h;
        S.u.x1.l[i] = l;
      }
      __syncthreads();
      conv2_frame([&](int mt, int nb, const float (&y)[4]) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int pos = frag_pos(mt, e);
          if (pos >= HW2) continue;
          const int i = frag_ch(nb, e) * HW2 + pos;
          if (r == 0) { S.y2[i] = y[e]; S.s2[i] = 0.f; S.q2[i] = 0.f; }
          else {
            const float d = y[e] - S.y2[i];
            S.s2[i] += d;
            S.q2[i] = fmaf(d, d, S.q2[i]);
          }
        }
      });
    }
    __syncthreads();
    {
      const float invR = 1.f / (float)p.R, invR1 = 1.f / (float)(p.R - 1);
      for (int i = tid; i < P2; i += kT) {
        const int co = i / HW2;
        const float s = S.s2[i];
        const float mean = S.y2[i] + s * invR;
        const float var = fmaxf((S.q2[i] - s * (s * invR)) * invR1, 0.f);
        const float a = par(kG2 + co) / sqrtf(var + 1e-5f);
        S.s2[i] = a;
        S.q2[i] = par(kB2 + co) - mean * a;
      }
    }
    // (the first conv1_frame below begins with a barrier that publishes s2 / q2)

    // ---------------- phase D: observations -> split conv features XS[b][2592]
    for (int b = 0; b < p.B; ++b) {
      conv1_frame(p.obs + (size_t)b * IMG, [&](int pt, int nb, const float (&y)[4]) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int i = frag_ch(nb, e) * HW1 + frag_pos(pt, e);
          __half h, l;
          split1(fmaxf(fmaf(y[e], S.s1[i], S.q1[i]), 0.f), h, l);
          S.u.x1.h[i] = h;
          S.u.x1.l[i] = l;
        }
      });
      __syncthreads();
      __half* fh = XSh + (size_t)b * P2;
      __half* fl = XSl + (size_t)b * P2;
      conv2_frame([&](int mt, int nb, const float (&y)[4]) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int pos = frag_pos(mt, e);
          if (pos >= HW2) continue;
          const int i = frag_ch(nb, e) * HW2 + pos;
          __half h, l;
          split1(fmaxf(fmaf(y[e], S.s2[i], S.q2[i]), 0.f), h, l);
          fh[i] = h;
          fl[i] = l;
        }
      });
    }
    __syncthreads();   // features of every observation are in the slab (CTA-scope visibility)

    // ---------------- phase E: fc1 on the tensor cores, bias + ReLU, fc2 + squared error in fp32
    // D[256 x NB] = W X^T; warp w owns neurons [32w, 32w+32) (two m16 tiles)
    float* sH = S.s1;   // [NB][FC1]
    float loss = 0.f;
    for (int b0 = 0; b0 < p.B; b0 += NB) {
      const int nbv = min(NB, p.B - b0);
      float am[2][4][4], ac[2][4][4];
#pragma unroll
      for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int n = 0; n < 4; ++n)
#pragma unroll
          for (int e = 0; e < 4; ++e) { am[m][n][e] = 0.f; ac[m][n][e] = 0.f; }
      // B-operand rows (observations), clamped: padded columns are computed and never read
      const __half* xr_h[4];
      const __half* xr_l[4];
#pragma unroll
      for (int n = 0; n < 4; ++n) {
        const int ob = b0 + min(n * 8 + g, nbv - 1);
        xr_h[n] = XSh + (size_t)ob * P2 + 2 * t;
        xr_l[n] = XSl + (size_t)ob * P2 + 2 * t;
      }
      // A-operand rows (neurons): element (row, k) of tile m at W[32w + 16m + row][k]
      int64_t wrow[2][2];
#pragma unroll
      for (int m = 0; m < 2; ++m) {
        wrow[m][0] = kF1w + (int64_t)(32 * warp + 16 * m + g) * P2 + 2 * t;
        wrow[m][1] = wrow[m][0] + 8 * (int64_t)P2;
      }
#pragma unroll 2
      for (int k0 = 0; k0 < P2; k0 += 16) {
        uint32_t ah[2][4], al[2][4];
#pragma unroll
        for (int m = 0; m < 2; ++m) {
#pragma unroll
          for (int q = 0; q < 4; ++q) {   // q: a0 (row g, k), a1 (row g+8, k), a2 (row g, k+8), a3 (row g+8, k+8)
            const int64_t idx = wrow[m][q & 1] + k0 + (q >> 1) * 8;
            const float2 th = __ldg(reinterpret_cast<const float2*>(p.theta + idx));
            float2 e = make_float2(0.f, 0.f);
            if (!centre) e = __half22float2(*reinterpret_cast<const __half2*>(trow + idx));
            split2(__fadd_rn(th.x, __fmul_rn(sg, e.x)), __fadd_rn(th.y, __fmul_rn(sg, e.y)), ah[m][q], al[m][q]);
          }
        }
#pragma unroll
        for (int n = 0; n < 4; ++n) {
          const uint32_t bh0 = lds32(xr_h[n] + k0), bh1 = lds32(xr_h[n] + k0 + 8);
          const uint32_t bl0 = lds32(xr_l[n] + k0), bl1 = lds32(xr_l[n] + k0 + 8);
#pragma unroll
          for (int m = 0; m < 2; ++m) mma3(am[m][n], ac[m][n], ah[m], al[m], bh0, bh1, bl0, bl1);
        }
      }
      __syncthreads();   // previous chunk's fc2 done with sH
#pragma unroll
      for (int m = 0; m < 2; ++m) {
        const int n0 = 32 * warp + 16 * m + g;
        const float bias0 = par(kF1b + n0), bias1 = par(kF1b + n0 + 8);
#pragma unroll
        for (int n = 0; n < 4; ++n) {
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int ob = n * 8 + 2 * t + (e & 1);
            const int neuron = n0 + ((e >> 1) << 3);
            const float h = fmaf(ac[m][n][e], kLoInv, am[m][n][e]) + ((e >> 1) ? bias1 : bias0);
            sH[ob * FC1 + neuron] = fmaxf(h, 0.f);
          }
        }
      }
      __syncthreads();
      for (int e = tid; e < nbv * p.A; e += kT) {
        const int bi = e / p.A, a = e % p.A;
        float y = par(kF2w + (int64_t)FC1 * p.A + a);   // fc2.b follows fc2.w
        for (int k = 0; k < FC1; ++k) y = fmaf(sH[bi * FC1 + k], par(kF2w + (int64_t)a * FC1 + k), y);
        const float d = y - __ldg(p.target + (size_t)(b0 + bi) * p.A + a);
        loss = fmaf(d, d, loss);
      }
    }
    loss = warp_sum_f(loss);
    if (lane == 0) S.red[warp] = loss;
    __syncthreads();
    if (tid == 0) {
      float s = 0.f;
      for (int w = 0; w < kT / 32; ++w) s += S.red[w];
      const float r = -(s / ((float)p.B * (float)p.A));
      if (centre) p.ret_plus[0] = r;
      else if (minus) p.ret_minus[j] = r;
      else p.ret_plus[j] = r;
    }
  }
}

}  // namespace

int64_t eval_conv_tc_scratch_per_cta(int R, int B) {
  return (int64_t)R * P1 * (int64_t)sizeof(float) + 2 * (int64_t)B * P2 * (int64_t)sizeof(__half);
}

// estk_eval_conv_vbn with ESTK_PREC_F16 (estk_eval_conv.cu has checked the arguments)
int eval_conv_tc(estk_ctx* ctx, const EvalConvCall& c, cudaStream_t stream) {
  ConvTcParams p = {};
  p.theta = c.theta; p.table16 = reinterpret_cast<const __half*>(c.table16); p.offsets = c.offsets; p.order = c.order;
  p.pairs = c.pairs; p.sigma = c.sigma;
  p.A = c.A; p.R = c.R; p.B = c.B; p.xref = c.xref; p.obs = c.obs; p.target = c.target;
  p.ret_plus = c.ret_plus; p.ret_minus = c.ret_minus;
  p.scratch = reinterpret_cast<unsigned char*>(c.scratch);
  p.scratch_per_cta = eval_conv_tc_scratch_per_cta(c.R, c.B);
  p.members = c.offsets ? 2 * c.pairs : 1;
  const size_t smem = sizeof(Smem);
  ESTK_CUDA(cudaFuncSetAttribute(eval_conv_vbn_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int grid = ctx->sm_count;
  if (grid > p.members) grid = p.members;
  eval_conv_vbn_tc_kernel<<<grid, kT, smem, stream>>>(p);
  ESTK_CUDA(cudaGetLastError());
  return ESTK_OK;
}
