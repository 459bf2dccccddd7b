// estk_eval_cnn_tf32.cu -- estk_eval_cnn_tf32 (include/estk_eval_cnn_tf32.h): the fixed-batch evaluate of a
// convolutional policy (Conv2d stack, flatten, Linear head) for every perturbed member, each layer an implicit
// GEMM on TF32 tensor cores (mma.sync m16n8k8, fp32 accumulation).
//
// One work item = one antithetic pair x one chunk of BC images; a persistent grid of 256-thread CTAs loops over
// the items.  Layer l of a sign is the GEMM Y[m][n] = sum_k X[m][k] * W[n][k] with m = (image, output position)
// over the chunk's BC * Ho * Wo rows, n the output channel and k the tap (ci, kh, kw); a Linear is the same GEMM
// with one position and its flattened input as the taps.  The CTA walks the layer in tiles of kBM rows x kBN
// outputs; for each tile it walks K in k-tiles of kBK taps from 0: every thread gathers its rows' inputs for
// the tile (im2col addressing, padding taps and the K, M and N tails as zeros, rounded with cvt.rna.tf32) into
// shared memory, and the tile's weights of both signs are formed there from one read of theta and the noise
// row (estk_form_pm, then rounded the same way).  Each warp owns 16 rows x 32 outputs of both signs: per k-step
// of 8 taps one A fragment per sign against four B fragments per sign.  So every output of every member is
// accumulated over the same k-walk (k-tiles, then k-steps, ascending), whatever its row, its sign, the chunk or
// the schedule: a member's bits are the centre form's on its materialised row.  The epilogue adds the fp32
// bias (formed, not rounded), applies estk_hidden_act (or identity / tanhf after the last layer) and stores the
// fp32 activation, [sign][image][c][h][w], in the CTA's slab of the context workspace; the next layer rounds it
// as it gathers.  Layer 0 reads the images from obs, one gather for both signs.
//
// After the last layer one thread per (sign, image) scores the row with estk_row_loss (the accuracy with
// estk_argmax_fold, as the fp32 kernel does), writes the behaviour characteristic and the per-image value to
// the context workspace, and the item of a pair that arrives last sums the values in image order
// (ESTK_PAIR_FINISH).  The chunk BC only sets the work split: the bits do not depend on it.
#include "estk_common.cuh"
#include "estk_eval_cnn_tf32.h"

namespace {

constexpr int kThreads = 256;     // 8 warps, 16 rows each
constexpr int kBM = 128;          // rows of one sign per tile
constexpr int kBN = 32;           // outputs per tile: four n8 fragments per warp
constexpr int kBK = 32;           // taps per k-tile: four k-steps of 8
constexpr int kLd = kBK + 4;      // shared row stride in words: conflict-free fragment reads
constexpr int kMaxBC = 128;
constexpr int64_t kSlabBudgetFloats = (int64_t)1 << 28;   // 1 GB of slab for the whole grid (at least one CTA's)
constexpr int64_t kSlabCtaFloats = (int64_t)1 << 21;      // BC halves until a CTA's slab is within 8 MB
constexpr int kMaxAct = 1 << 26;                          // the largest layer output served: one CTA within 1 GB
constexpr size_t kSmem = sizeof(uint32_t) * 2 * (kBM + kBN) * kLd   // A and W tiles of both signs
                         + sizeof(int64_t) * kBM + sizeof(int) * 2 * kBM + sizeof(float) * 2 * kBN;

struct Tf32Params {
  EstkCnnLayer layer[ESTK_MAX_LAYERS];
  int n_layers, out, maxact;
  const float* theta;
  const float* table;
  const int64_t* offsets;    // null => centre (theta, sigma ignored, the + sign only)
  const int32_t* order;
  int pairs;
  float sigma;
  const float* obs;          // [B][c][h][w]
  const float* target;       // [B][out]
  int B, BC, chunks;
  float* ret_plus;
  float* ret_minus;
  float* bc_plus;
  float* bc_minus;
  int bc_obs, bc_dim;
  float* partial;            // [pairs][2][B] per-image loss values
  unsigned int* counters;    // [pairs], zero on entry, zero on exit
  float* slab;               // [gridDim.x][2 buffers][2 signs][BC][maxact]
};

// rna_tf32(v): round to nearest, ties away from zero, to TF32 (the low 13 bits of the result are zero)
__device__ __forceinline__ uint32_t rna_tf32(float v) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
  return r;
}

__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
               "{%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

template <int HID, int HEAD>
__global__ void __launch_bounds__(kThreads, 1) eval_cnn_tf32_kernel(const Tf32Params p) {
  extern __shared__ __align__(16) uint32_t sm[];
  uint32_t* const As = sm;                                              // [2][kBM][kLd] inputs, + then -
  uint32_t* const Ws = As + 2 * kBM * kLd;                              // [2][kBN][kLd] weights, + then -
  int64_t* const rbase = reinterpret_cast<int64_t*>(Ws + 2 * kBN * kLd);   // [kBM] row's input offset at tap 0
  int* const rih = reinterpret_cast<int*>(rbase + kBM);                 // [kBM] top row of the receptive field
  int* const riw = rih + kBM;                                           // [kBM] its left column
  float* const bias = reinterpret_cast<float*>(riw + kBM);              // [2][kBN]

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t4 = lane & 3;
  const bool centre = p.offsets == nullptr;
  const float sigma = centre ? 0.f : p.sigma;
  const int nsign = centre ? 1 : 2;
  const int L = p.n_layers, BC = p.BC;
  const int64_t act = (int64_t)BC * p.maxact;   // one sign's activations in one buffer
  float* const slab = p.slab + (size_t)blockIdx.x * 4 * act;

  for (int64_t item = blockIdx.x; item < (int64_t)p.pairs * p.chunks; item += gridDim.x) {
    const int slot = (int)(item / p.chunks), chunk = (int)(item % p.chunks);
    const int j = p.order ? p.order[slot] : slot;
    const NoiseRow nz = noise_row(p.theta, p.table, nullptr, p.offsets, j);
    const int b0 = chunk * BC, nb = min(BC, p.B - b0);

    for (int l = 0; l < L; ++l) {
      const EstkCnnLayer ly = p.layer[l];
      const bool last = l == L - 1;
      const int64_t ximg = l == 0 ? (int64_t)ly.cin * ly.hin * ly.win : p.maxact;   // input floats per image
      const float* const X = l == 0 ? p.obs + b0 * ximg : slab + ((l - 1) & 1) * 2 * act;
      const bool xsplit = l > 0 && nsign == 2;   // the - member has inputs of its own (layer 0: the same images)
      float* const Y = slab + (l & 1) * 2 * act;
      const int P = ly.ho * ly.wo, M = nb * P, kk = ly.k * ly.k;
      for (int n0 = 0; n0 < ly.cout; n0 += kBN) {
        for (int m0 = 0; m0 < M; m0 += kBM) {
          __syncthreads();   // the previous tile's row table, bias and fragments consumed
          if (tid < kBM) {
            const int m = m0 + tid;
            if (m < M) {
              const int b = m / P, pos = m - b * P, oh = pos / ly.wo, ow = pos - oh * ly.wo;
              const int ih0 = oh * ly.s - ly.pad, iw0 = ow * ly.s - ly.pad;
              rih[tid] = ih0;
              riw[tid] = iw0;
              rbase[tid] = b * ximg + (int64_t)ih0 * ly.win + iw0;
            } else {   // a row past the chunk reads zeros
              rih[tid] = INT_MIN / 2;
              riw[tid] = 0;
              rbase[tid] = 0;
            }
          } else if (tid < kBM + 2 * kBN) {
            const int e = tid - kBM, n = n0 + e % kBN;
            float wp = 0.f, wm = 0.f;
            if (n < ly.cout) estk_form_pm(p.theta, nz, sigma, ly.wbase + (int64_t)ly.cout * ly.K + n, wp, wm);
            bias[e] = e < kBN ? wp : wm;
          }
          float acc[2][4][4] = {};
          for (int k0 = 0; k0 < ly.K; k0 += kBK) {
            // this lane's tap of the k-tile: the column it gathers
            const int kx = k0 + lane;
            int toff = 0, kh = INT_MIN / 2, kw = 0;
            if (kx < ly.K) {
              const int ci = kx / kk, rem = kx - ci * kk;
              kh = rem / ly.k;
              kw = rem - kh * ly.k;
              toff = (ci * ly.hin + kh) * ly.win + kw;
            }
            __syncthreads();   // the previous k-tile's fragments read; the row table and the layer input written
#pragma unroll 4
            for (int i = 0; i < kBM / 8; ++i) {
              const int r = warp + 8 * i;
              const bool ok = (unsigned)(rih[r] + kh) < (unsigned)ly.hin && (unsigned)(riw[r] + kw) < (unsigned)ly.win;
              const float* const xp = X + rbase[r] + toff;
              As[r * kLd + lane] = rna_tf32(ok ? xp[0] : 0.f);
              if (xsplit) As[(kBM + r) * kLd + lane] = rna_tf32(ok ? xp[act] : 0.f);
            }
#pragma unroll
            for (int e = tid; e < kBN * kBK; e += kThreads) {
              const int n = e / kBK, kc = e % kBK, on = n0 + n, kt = k0 + kc;
              float wp = 0.f, wm = 0.f;
              if (on < ly.cout && kt < ly.K) estk_form_pm(p.theta, nz, sigma, ly.wbase + (int64_t)on * ly.K + kt, wp, wm);
              Ws[n * kLd + kc] = rna_tf32(wp);
              Ws[(kBN + n) * kLd + kc] = rna_tf32(wm);
            }
            __syncthreads();
            if (m0 + 16 * warp < M) {
#pragma unroll
              for (int ks = 0; ks < kBK; ks += 8) {
#pragma unroll
                for (int s = 0; s < 2; ++s) {
                  if (s >= nsign) break;
                  const uint32_t* const A = As + ((s && xsplit ? kBM : 0) + 16 * warp) * kLd + ks + t4;
                  const uint32_t a[4] = {A[g * kLd], A[(g + 8) * kLd], A[g * kLd + 4], A[(g + 8) * kLd + 4]};
#pragma unroll
                  for (int f = 0; f < 4; ++f) {
                    if (n0 + 8 * f >= ly.cout) break;
                    const uint32_t* const w = Ws + (s * kBN + 8 * f + g) * kLd + ks + t4;
                    mma_tf32(acc[s][f], a, w[0], w[4]);
                  }
                }
              }
            }
          }
          // epilogue: + bias, the activation, the fp32 value to the layer's output [sign][image][n][position]
          if (m0 + 16 * warp < M) {
#pragma unroll
            for (int s = 0; s < 2; ++s) {
              if (s >= nsign) break;
#pragma unroll
              for (int f = 0; f < 4; ++f)
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                  const int m = m0 + 16 * warp + g + (q >> 1) * 8, nl = 8 * f + 2 * t4 + (q & 1), n = n0 + nl;
                  if (m < M && n < ly.cout) {
                    float y = acc[s][f][q] + bias[s * kBN + nl];
                    if (!last) y = estk_hidden_act<HID, true>(y);
                    else if (HEAD == kHeadTanh) y = tanhf(y);
                    const int b = m / P, pos = m - b * P;
                    Y[s * act + (int64_t)b * p.maxact + (int64_t)n * P + pos] = y;
                  }
                }
            }
          }
        }
      }
    }

    // ---- one thread per (sign, image) scores the row in column order; the outputs are the last layer's
    __syncthreads();
    const float* const Yo = slab + ((L - 1) & 1) * 2 * act;
    for (int r = tid; r < 2 * nb; r += kThreads) {
      const int s = r / nb, bl = r - s * nb, b = b0 + bl;
      if (s >= nsign) {   // the centre form has no - member: its partials are zeros (the finish reads, then drops them)
        p.partial[((size_t)slot * 2 + 1) * p.B + b] = 0.f;
        __threadfence();
        continue;
      }
      const float* const yr = Yo + s * act + (int64_t)bl * p.maxact;
      const float* const tg = p.target + (size_t)b * p.out;
      float v;
      if constexpr (HEAD == kHeadAccuracy) {   // 1 where the first argmaxes of logits and target agree
        float ym = -INFINITY, tm = -INFINITY;
        int yi = INT_MAX, ti = INT_MAX;
        for (int o = 0; o < p.out; ++o) {
          estk_argmax_fold(ym, yi, yr[o], o);
          estk_argmax_fold(tm, ti, __ldg(tg + o), o);
        }
        v = yi == ti ? 1.f : 0.f;
      } else {
        v = estk_row_loss<HEAD>([&](int c) { return yr[c]; }, tg, p.out);
      }
      float* const bc = s ? p.bc_minus : p.bc_plus;
      if (bc && b < p.bc_obs)
        for (int o = 0; o < p.out; ++o) {
          const int64_t e = (int64_t)b * p.out + o;
          if (e < p.bc_dim) bc[(size_t)j * p.bc_dim + e] = yr[o];
        }
      p.partial[((size_t)slot * 2 + s) * p.B + b] = v;
      __threadfence();
    }
    __syncthreads();
    if (tid == 0 && estk_pair_arrive(p.counters + slot, p.chunks))
      ESTK_PAIR_FINISH(p.partial + (size_t)slot * 2 * p.B, p.B,
                       HEAD == kHeadAccuracy ? -(float)p.B
                                             : (float)((int64_t)p.B * (HEAD == kHeadXent ? 1 : p.out)),
                       p.ret_plus, p.ret_minus, j, p.counters + slot);
  }
}

template <int HID, int HEAD>
int launch_tf32(estk_ctx* ctx, Tf32Params& p, cudaStream_t stream, const char* who) {
  SlabLaunch l = {};
  l.slab = true;
  l.items = (int64_t)p.pairs * p.chunks;
  l.smem_shared = l.smem_slab = kSmem;
  l.slab_per_cta = 4 * (int64_t)p.BC * p.maxact;
  l.members = p.pairs;
  l.eval_floats = (int64_t)p.pairs * 2 * p.B;
  l.slab_cap = kSlabBudgetFloats;
  return estk_launch_eval(ctx, eval_cnn_tf32_kernel<HID, HEAD>, eval_cnn_tf32_kernel<HID, HEAD>, p, l, kThreads,
                          stream, who, [&] {
                            p.partial = ctx->eval_partial;
                            p.counters = estk_member_counters(ctx);
                          });
}

// The code checks of the fp32 route (ESTK_ACTIONS and the cells refused as ESTK_ERR_INVALID here), then the
// layers; ESTK_ERR_INVALID (with the reason) or ESTK_OK
int tf32_parse(const estk_mlp_desc& d, int B, EstkCnnShape& s, const char* who) {
  if (const int rc = eval_cnn_code_check(d.activation, ESTK_ERR_INVALID, who)) return rc;
  if (const int rc = eval_cnn_batch_check(d.activation, B, who)) return rc;
  return eval_cnn_parse(d, (d.activation >> 24) & 0xff, s, who);
}

bool tf32_serves(const EstkCnnShape& s) { return s.maxact <= kMaxAct; }

}  // namespace

extern "C" int estk_eval_cnn_tf32(estk_ctx* ctx, const estk_mlp_desc* desc, const float* theta, const float* table,
                                  const int64_t* offsets, const int32_t* order, int32_t pairs, float sigma,
                                  const float* obs, const float* target, int32_t B, float* ret_plus,
                                  float* ret_minus, float* bc_plus, float* bc_minus, int32_t bc_obs, int32_t bc_dim,
                                  void* stream) {
  const char* who = "estk_eval_cnn_tf32";
  ESTK_CHECK_ARG(desc, "%s: null desc", who);
  const bool centre = offsets == nullptr;
  // the record of the fp32 route, with its centre conventions (pairs 1, sigma 0, no table, order or - outputs)
  EvalMlpCall c = {};
  c.desc = *desc;
  c.precision = ESTK_PREC_FP32;
  c.theta = theta; c.obs = obs; c.target = target; c.B = B;
  c.ret_plus = ret_plus; c.bc_plus = bc_plus; c.bc_obs = bc_obs; c.bc_dim = bc_dim;
  c.pairs = 1;
  if (!centre) {
    c.table = table; c.offsets = offsets; c.order = order; c.pairs = pairs; c.sigma = sigma;
    c.ret_minus = ret_minus; c.bc_minus = bc_minus;
  }
  if (const int rc = eval_returns_check(ctx, c, who)) return rc;
  EstkCnnShape s = {};
  if (const int rc = tf32_parse(c.desc, B, s, who)) return rc;
  if (!tf32_serves(s)) {
    estk_set_error("%s: a layer output of %d floats per image exceeds the %d the kernel serves", who, s.maxact,
                   kMaxAct);
    return ESTK_ERR_UNSUPPORTED;
  }

  Tf32Params p = {};
  std::copy(s.layer, s.layer + ESTK_MAX_LAYERS, p.layer);
  p.n_layers = s.n_layers; p.out = s.out; p.maxact = s.maxact;
  p.theta = c.theta; p.table = c.table; p.offsets = c.offsets; p.order = c.order; p.pairs = c.pairs;
  p.sigma = c.sigma; p.obs = c.obs; p.target = c.target; p.B = c.B;
  p.ret_plus = c.ret_plus; p.ret_minus = c.ret_minus;
  p.bc_plus = c.bc_plus; p.bc_minus = c.bc_minus; p.bc_obs = c.bc_obs; p.bc_dim = c.bc_dim;
  // images per work item: at most B and kMaxBC, halved until a CTA's slab is within kSlabCtaFloats
  int bc = kMaxBC;
  while (bc > 1 && (bc / 2 >= B || 4 * (int64_t)bc * s.maxact > kSlabCtaFloats)) bc /= 2;
  p.BC = bc;
  p.chunks = (B + bc - 1) / bc;
  const int low = c.desc.activation & 0xffffff;
  return estk_dispatch(EstkHiddenKinds{}, low & 0xff, [&](auto HID) {
    return estk_dispatch(EstkValues<kHeadIdentity, kHeadXent, kHeadAccuracy, kHeadTanh>{}, estk_head(low),
                         [&](auto HEAD) { return launch_tf32<HID, HEAD>(ctx, p, (cudaStream_t)stream, who); });
  });
}

extern "C" int estk_eval_cnn_tf32_supported(const estk_mlp_desc* desc, int32_t B) {
  EstkCnnShape s = {};
  return desc && B >= 1 && tf32_parse(*desc, B, s, "estk_eval_cnn_tf32_supported") == ESTK_OK && tf32_serves(s);
}
