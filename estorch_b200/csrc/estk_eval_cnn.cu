// estk_eval_cnn.cu -- estk_eval_mlp with n_conv != 0 in bits 24-31 of the activation code, fp32: the
// fixed-batch evaluate of a convolutional policy (Conv2d stack, flatten, Linear head) for every perturbed
// member.  The device-agent evaluate of a small CNN: image classification with ESTK_LOSS_XENT, or regression
// of frames onto targets with the squared error.
//
// A Linear layer is the 1x1 convolution of its input flattened to [K][1][1] (torch's parameter layout
// [out][in] is [out][in][1][1]), so one layer routine serves both: layer l maps [Cin][Hin][Win] to
// [Cout][Ho][Wo], and every output element is one fmaf chain from 0 over the taps in ascending (ci, kh, kw)
// order -- taps in the zero padding are skipped -- then + bias, then the hidden activation (or, for the last
// layer, the output activation).  Activations are kept k-major, [C*H*W][ROWS], so the last conv's output is
// already the first Linear's input in torch's flatten order.
//
// One work item = one antithetic pair x one chunk of BC images, 256 threads, as in eval_rnn_seq_kernel
// (estk_eval_rnn_seq.cu): the pair's noise row is read once for both signs, and every weight tile (OG output
// channels x KT taps) is formed in shared memory as W+ = theta + sigma*t and W- = theta - sigma*t.  A thread
// takes output elements (row, channel, position) in turn; when the layer's taps span several k-chunks the
// partial chain is kept in the output buffer between chunks (the same fp32 value, so the same bits).  After
// the last layer one thread per row scores its image in column order; the per-image values go to the
// context workspace and the item of a pair that arrives last sums them in image order (include/estk.h
// states the order: the bits do not depend on BC, the schedule or `order`; no float atomics).
//
// The two activation buffers ([2][max layer output][ROWS]) stay in shared memory when they fit the budget
// below; otherwise they live in a per-CTA slab of the context workspace and a persistent grid loops over the
// work items (the same code, global instead of shared addresses).  Layer 0 reads the images from `obs`.
//
// estk_act_cnn (include/estk_act_cnn.h) runs the same kernel with kHeadAct in HEAD: layer 0 reads each member's
// own images, the epilogue writes the last layer's outputs instead of scoring them, and there are no partials
// and no arrival counters.  The layer walk is shared, so a member's outputs are the bits the evaluate writes to
// its behaviour characteristic for the same images.
#include "estk_common.cuh"
#include "estk_act_cnn.h"

namespace {

constexpr int kThreads = 256;
constexpr int kTile = 2048;                  // weights per sign in one tile (OG x KT)
constexpr int kMaxKT = 256;                  // taps per tile
constexpr size_t kSmemBudget = 220 * 1024;   // up to the 227 KB a CTA may hold
constexpr size_t kSmemPreferred = 110 * 1024;  // two CTAs per SM
constexpr int64_t kSlabBudgetFloats = (int64_t)1 << 28;  // 1 GB of slab for the whole grid (at least one CTA's)

struct CnnLayer {
  int cin, hin, win, cout, k, s, pad, ho, wo;
  int K;            // cin * k * k: taps per output
  int64_t wbase;    // weight [cout][K], then bias [cout]
};

struct CnnParams {
  CnnLayer layer[ESTK_MAX_LAYERS];
  int n_layers, in_size, out, maxact;   // maxact: the largest layer output C*H*W
  const float* theta;
  const float* table;
  const int64_t* offsets;    // null => centre (theta, sigma ignored)
  const int32_t* order;
  int pairs;
  float sigma;
  const float* obs;          // [B][c][h][w]
  const float* target;       // [B][out]
  int B, BC, chunks;
  float* ret_plus;
  float* ret_minus;
  float* bc_plus;            // [pairs][bc_dim]: policy(obs[:bc_obs]).flatten()[:bc_dim]
  float* bc_minus;
  int bc_obs, bc_dim;
  float* partial;            // [pairs][2][B] per-image loss values
  unsigned int* counters;    // [pairs], zero on entry, zero on exit
  float* slab;               // SLAB: [gridDim.x][2][maxact][ROWS]
  // the act variant: obs is [2*pairs][B][c][h][w] (block j the + member of local pair j, pairs + j its mirror)
  // or, for the centre, [B][c][h][w]; the outputs are [pairs][B][out] per sign (after every field above, so
  // the evaluate kernels read their parameters at the same offsets)
  float* out_plus;
  float* out_minus;
};

// OG x KT of a layer's weight tile
__host__ __device__ inline int cnn_kt(int K) { return K < kMaxKT ? K : kMaxKT; }
__host__ __device__ inline int cnn_og(int K, int cout) {
  const int og = kTile / cnn_kt(K);
  return og < cout ? og : cout;
}

template <int HID, int HEAD, bool SLAB>
__global__ void __launch_bounds__(kThreads) eval_cnn_kernel(const CnnParams p) {
  constexpr bool ACT = (HEAD & kHeadAct) != 0;
  constexpr int OUT_HEAD = HEAD & ~kHeadAct;
  extern __shared__ __align__(16) float smem[];
  const int ROWS = 2 * p.BC, BC = p.BC;
  float* const Wp = smem;                          // [OG][KT]
  float* const Wm = Wp + kTile;                    // [OG][KT]
  int* const toff = reinterpret_cast<int*>(Wm + kTile);   // [KT] input offset of tap t: (ci*Hin + kh)*Win + kw
  int* const tkhw = toff + kMaxKT;                         // [KT] kh << 8 | kw
  const size_t act = (size_t)p.maxact * ROWS;
  float* const buf0 = SLAB ? p.slab + (size_t)blockIdx.x * 2 * act : reinterpret_cast<float*>(tkhw + kMaxKT);
  float* const buf1 = buf0 + act;

  const int tid = threadIdx.x;
  const bool centre = (p.offsets == nullptr);
  const float sigma = centre ? 0.f : p.sigma;
  const int L = p.n_layers;

  unsigned int slot = blockIdx.x / (unsigned)p.chunks, chunk = blockIdx.x % (unsigned)p.chunks;
  for (; slot < (unsigned)p.pairs; chunk += gridDim.x, slot += chunk / p.chunks, chunk %= p.chunks) {
    const int j = p.order ? p.order[slot] : (int)slot;
    const NoiseRow nz{centre ? p.theta : p.table + p.offsets[j], nullptr};   // the fp32 table only
    const int b0 = chunk * BC;
    const int nb = min(BC, p.B - b0);                // images of this chunk (rows past it read zeros)

    for (int l = 0; l < L; ++l) {
      const CnnLayer ly = p.layer[l];
      const bool last = l == L - 1;
      const float* const X = (l & 1) ? buf0 : buf1;  // layer l-1's output (layer 0 reads obs)
      float* const Y = (l & 1) ? buf1 : buf0;
      const int KT = cnn_kt(ly.K), OG = cnn_og(ly.K, ly.cout), kk = ly.k * ly.k;
      const unsigned P = (unsigned)ly.ho * ly.wo, HWin = (unsigned)ly.hin * ly.win;
      for (int oc0 = 0; oc0 < ly.cout; oc0 += OG) {
        const int og_n = min(OG, ly.cout - oc0);
        const unsigned elems = (unsigned)ROWS * og_n * P;
        for (int k0 = 0; k0 < ly.K; k0 += KT) {
          const int kt = min(KT, ly.K - k0);
          const bool first = k0 == 0, fin = k0 + kt == ly.K;
          __syncthreads();   // the previous tile consumed; the previous layer's (or item's) buffers written
          for (int e = tid; e < og_n * kt; e += kThreads) {
            const int og = e / kt, t = e % kt;
            const int64_t idx = ly.wbase + (int64_t)(oc0 + og) * ly.K + k0 + t;
            const float th = __ldg(p.theta + idx);
            const float ep = __fmul_rn(sigma, nz(idx));
            Wp[og * kt + t] = __fadd_rn(th, ep);
            Wm[og * kt + t] = __fsub_rn(th, ep);
          }
          for (int t = tid; t < kt; t += kThreads) {
            const int kidx = k0 + t, ci = kidx / kk, rem = kidx % kk, kh = rem / ly.k, kw = rem % ly.k;
            toff[t] = (ci * ly.hin + kh) * ly.win + kw;
            tkhw[t] = kh << 8 | kw;
          }
          __syncthreads();
          for (unsigned e = tid; e < elems; e += kThreads) {
            const int r = (int)(e % ROWS);
            const unsigned rest = e / ROWS;
            const int pos = (int)(rest % P), og = (int)(rest / P);
            const int oh = pos / ly.wo, ow = pos % ly.wo;
            const int ih0 = oh * ly.s - ly.pad, iw0 = ow * ly.s - ly.pad;
            const bool minus = r >= BC;
            const int b = r - (minus ? BC : 0);
            const float* const Ws = (minus ? Wm : Wp) + og * kt;
            float* const yp = Y + ((size_t)(oc0 + og) * P + pos) * ROWS + r;
            float acc = first ? 0.f : *yp;
            if (l == 0) {
              // the act variant's centre has no - members: its - rows read nothing and are never written out
              if (b < nb && !(ACT && centre && minus)) {
                size_t img = b0 + b;
                if constexpr (ACT) img += (size_t)(minus ? p.pairs + j : j) * p.B;   // the member's own images
                const float* const xb = p.obs + img * HWin * ly.cin + (ih0 * ly.win + iw0);
#pragma unroll 4
                for (int t = 0; t < kt; ++t) {
                  const int kh = tkhw[t] >> 8, kw = tkhw[t] & 0xff;
                  if ((unsigned)(ih0 + kh) < (unsigned)ly.hin && (unsigned)(iw0 + kw) < (unsigned)ly.win)
                    acc = fmaf(__ldg(xb + toff[t]), Ws[t], acc);
                }
              }
            } else {
              const float* const xr = X + (ptrdiff_t)(ih0 * ly.win + iw0) * ROWS + r;
#pragma unroll 4
              for (int t = 0; t < kt; ++t) {
                const int kh = tkhw[t] >> 8, kw = tkhw[t] & 0xff;
                if ((unsigned)(ih0 + kh) < (unsigned)ly.hin && (unsigned)(iw0 + kw) < (unsigned)ly.win)
                  acc = fmaf(xr[(ptrdiff_t)toff[t] * ROWS], Ws[t], acc);
              }
            }
            if (fin) {
              const int64_t bidx = ly.wbase + (int64_t)ly.cout * ly.K + oc0 + og;
              float y = acc + estk_form_sign(p.theta, nz, sigma, bidx, minus);
              if (!last) y = estk_hidden_act<HID, true>(y);   // SiLU without the div.rn call: the same bits
              else if (OUT_HEAD == kHeadTanh) y = tanhf(y);
              acc = y;
            }
            *yp = acc;
          }
        }
      }
    }

    // ---- thread r < ROWS scores image r in column order; the outputs are in the last layer's buffer
    __syncthreads();
    const float* const Yo = ((L - 1) & 1) ? buf1 : buf0;
    if constexpr (ACT) {   // thread r < ROWS writes image r's outputs themselves to out[j][b] of its sign
      const int bl = tid % BC;
      const bool minus = tid >= BC;
      if (tid < ROWS && bl < nb && !(centre && minus)) {
        float* const y = (minus ? p.out_minus : p.out_plus) + ((size_t)j * p.B + b0 + bl) * p.out;
        for (int o = 0; o < p.out; ++o) y[o] = Yo[(size_t)o * ROWS + tid];
      }
      continue;
    }
    const int r = tid, bl = tid % BC, b = b0 + bl;
    if (tid < ROWS && bl < nb) {
      const bool minus = r >= BC;
      const float* const tg = p.target + (size_t)b * p.out;
      float s = 0.f;   // the kernel's own lines, not estk_row_loss: the inlined helper changes its SASS
      if constexpr (HEAD == kHeadXent) {
        float m = -INFINITY;
        for (int o = 0; o < p.out; ++o) m = fmaxf(m, Yo[(size_t)o * ROWS + r]);
        float se = 0.f, st = 0.f, sty = 0.f;
        for (int o = 0; o < p.out; ++o) {
          const float y = Yo[(size_t)o * ROWS + r], tv = __ldg(tg + o);
          se += expf(y - m);
          st += tv;
          sty = fmaf(tv, y, sty);
        }
        s = fmaf(m + logf(se), st, -sty);
      } else if constexpr (HEAD == kHeadAccuracy) {   // 1 where the first argmaxes of logits and target agree
        float ym = -INFINITY, tm = -INFINITY;
        int yi = INT_MAX, ti = INT_MAX;
        for (int o = 0; o < p.out; ++o) {
          estk_argmax_fold(ym, yi, Yo[(size_t)o * ROWS + r], o);
          estk_argmax_fold(tm, ti, __ldg(tg + o), o);
        }
        s = yi == ti ? 1.f : 0.f;
      } else {
        for (int o = 0; o < p.out; ++o) {
          const float d = Yo[(size_t)o * ROWS + r] - __ldg(tg + o);
          s = fmaf(d, d, s);
        }
      }
      float* const bc = minus ? p.bc_minus : p.bc_plus;
      if (bc && !(centre && minus) && b < p.bc_obs)
        for (int o = 0; o < p.out; ++o) {
          const int64_t e = (int64_t)b * p.out + o;
          if (e < p.bc_dim) bc[(size_t)j * p.bc_dim + e] = Yo[(size_t)o * ROWS + r];
        }
      p.partial[((size_t)slot * 2 + (minus ? 1 : 0)) * p.B + b] = s;
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

size_t fixed_smem() { return sizeof(float) * 2 * kTile + sizeof(int) * 2 * kMaxKT; }

template <int HID, int HEAD>
int launch_cnn(estk_ctx* ctx, CnnParams& p, cudaStream_t stream, const char* who) {
  constexpr bool ACT = (HEAD & kHeadAct) != 0;
  // the largest chunk of images whose activations fit in shared memory, preferring two CTAs per SM
  int bc = 0;
  size_t smem_all = 0;
  for (size_t budget : {kSmemPreferred, kSmemBudget}) {
    for (int cand : {16, 4, 1}) {
      const size_t s = fixed_smem() + sizeof(float) * 2 * (size_t)p.maxact * 2 * cand;
      if (s <= budget && (cand == 1 || p.B > cand / 4)) { bc = cand; smem_all = s; break; }
    }
    if (bc) break;
  }
  SlabLaunch l = {};
  l.slab = bc == 0;
  if (l.slab) bc = 1;
  p.BC = bc;
  p.chunks = (p.B + bc - 1) / bc;
  l.items = (int64_t)p.pairs * p.chunks;
  l.smem_shared = smem_all;
  l.smem_slab = fixed_smem();
  l.slab_per_cta = (int64_t)2 * p.maxact * 2 * bc;
  // the act variant keeps no partials and no counters: it reserves on the slab path only
  l.members = ACT ? 0 : p.pairs;
  l.eval_floats = ACT ? 0 : (int64_t)p.pairs * 2 * p.B;
  // the persistent loop serves any grid, so a large image costs the memory of a few CTAs' buffers, not of
  // every resident CTA's
  l.slab_cap = kSlabBudgetFloats;
  return estk_launch_eval(ctx, eval_cnn_kernel<HID, HEAD, false>, eval_cnn_kernel<HID, HEAD, true>, p, l, kThreads,
                          stream, who, [&] {
                            if (ACT) return;
                            p.partial = ctx->eval_partial;
                            p.counters = estk_member_counters(ctx);
                          });
}

// The kernel of hidden kind code & 0xff and head `head` (estk_head, or kHeadAct | the output of an act call)
int launch_code(estk_ctx* ctx, CnnParams& p, int code, int head, cudaStream_t stream, const char* who) {
  return estk_dispatch(EstkHiddenKinds{}, code & 0xff, [&](auto HID) {
    return estk_dispatch(EstkCnnHeads{}, head, [&](auto HEAD) { return launch_cnn<HID, HEAD>(ctx, p, stream, who); });
  });
}

// The layers of a packed descriptor (include/estk.h, convolutional evaluate) into p.layer, p.n_layers, p.in_size,
// p.out and p.maxact; n_conv (1..7) is bits 24-31 of d.activation, checked by the caller.  Every malformed
// field is ESTK_ERR_INVALID.
int cnn_parse(const estk_mlp_desc& d, int n_conv, CnnParams& p, const char* who) {
  ESTK_CHECK_ARG(d.n_layers > n_conv && d.n_layers <= ESTK_MAX_LAYERS,
                 "%s: n_layers=%d must exceed n_conv=%d (at least one Linear) and be at most %d", who, d.n_layers,
                 n_conv, ESTK_MAX_LAYERS);
  const uint32_t in = (uint32_t)d.dims[0];
  int c = in & 1023, h = (in >> 10) & 1023, w = (in >> 20) & 1023;
  ESTK_CHECK_ARG((in >> 30) == 0 && c >= 1 && h >= 1 && w >= 1,
                 "%s: dims[0]=0x%x is not ESTK_CNN_INPUT(c, h, w) with c, h, w in 1..1023", who, in);
  p.in_size = c * h * w;
  int64_t wbase = 0, maxact = 0;
  const int64_t kIdxLimit = (int64_t)1 << 30;   // 32-bit element indexing: ROWS (<= 32) x layer size < 2^35 / 32
  for (int l = 0; l < d.n_layers; ++l) {
    CnnLayer& ly = p.layer[l];
    ly.cin = c; ly.hin = h; ly.win = w;
    if (l < n_conv) {
      const uint32_t f = (uint32_t)d.dims[l + 1];
      ly.cout = f & 4095; ly.k = (f >> 12) & 63; ly.s = (f >> 18) & 63; ly.pad = (f >> 24) & 63;
      ESTK_CHECK_ARG((f >> 30) == 0 && ly.cout >= 1 && ly.k >= 1 && ly.s >= 1 && ly.pad < ly.k,
                     "%s: dims[%d]=0x%x is not ESTK_CNN_CONV(out_c 1..4095, k 1..63, stride 1..63, pad < k)", who,
                     l + 1, f);
      ESTK_CHECK_ARG(h + 2 * ly.pad >= ly.k && w + 2 * ly.pad >= ly.k,
                     "%s: conv %d (k=%d, pad=%d) is larger than its %dx%d input", who, l, ly.k, ly.pad, h, w);
      ly.ho = (h + 2 * ly.pad - ly.k) / ly.s + 1;
      ly.wo = (w + 2 * ly.pad - ly.k) / ly.s + 1;
    } else {   // a Linear: the 1x1 convolution of the flattened input
      ESTK_CHECK_ARG(d.dims[l + 1] >= 1, "%s: dims[%d]=%d", who, l + 1, d.dims[l + 1]);
      ly.cin = c * h * w; ly.hin = ly.win = 1;
      ly.cout = d.dims[l + 1]; ly.k = ly.s = 1; ly.pad = 0; ly.ho = ly.wo = 1;
    }
    const int64_t K = (int64_t)ly.cin * ly.k * ly.k, outsz = (int64_t)ly.cout * ly.ho * ly.wo;
    ESTK_CHECK_ARG(K < kIdxLimit && outsz < kIdxLimit && (int64_t)ly.cin * ly.hin * ly.win < kIdxLimit,
                   "%s: layer %d has more than 2^30 inputs, taps or outputs per image", who, l);
    ly.K = (int)K;
    ly.wbase = wbase;
    wbase += (int64_t)ly.cout * K + ly.cout;
    maxact = std::max(maxact, outsz);
    c = ly.cout; h = ly.ho; w = ly.wo;
  }
  p.n_layers = d.n_layers;
  p.out = c;
  p.maxact = (int)maxact;
  return ESTK_OK;
}

}  // namespace

int eval_cnn_parse(const estk_mlp_desc& d, int n_conv, EstkCnnShape& s, const char* who) {
  CnnParams p = {};
  if (const int rc = cnn_parse(d, n_conv, p, who)) return rc;
  for (int l = 0; l < p.n_layers; ++l) {
    const CnnLayer& a = p.layer[l];
    s.layer[l] = EstkCnnLayer{a.cin, a.hin, a.win, a.cout, a.k, a.s, a.pad, a.ho, a.wo, a.K, a.wbase};
  }
  s.n_layers = p.n_layers; s.in_size = p.in_size; s.out = p.out; s.maxact = p.maxact;
  return ESTK_OK;
}

int eval_cnn_code_check(int code, int route_rc, const char* who) {
  const int n_conv = (code >> 24) & 0xff, low = code & 0xffffff;
  ESTK_CHECK_ARG(n_conv >= 1 && n_conv <= 7, "%s: n_conv=%d (bits 24-31 of activation 0x%x) is outside 1..7", who,
                 n_conv, code);
  if (estk_eval_route(low) != kRouteDense) {
    estk_set_error("%s: ESTK_ACTIONS and the recurrent cells are not supported with a conv stack (code 0x%x)", who,
                   code);
    return route_rc;
  }
  ESTK_CHECK_ARG(estk_act_valid(low), "%s: activation=0x%x: bits 0-23 are not a defined hidden | output | loss "
                 "combination", who, code);
  return ESTK_OK;
}

int eval_cnn_batch_check(int code, int B, const char* who) {
  ESTK_CHECK_ARG(!estk_loss_accuracy(code & 0xffffff) || B <= kAccuracyMaxB,
                 "%s: B=%d: the accuracy's count is exact in fp32 for B < 2^24 only", who, B);
  return ESTK_OK;
}

int eval_cnn(estk_ctx* ctx, const EvalMlpCall& call, cudaStream_t stream) {
  const char* who = "estk_eval_mlp[convolutional]";
  if (const int rc = eval_returns_supported(call, who)) return rc;
  const estk_mlp_desc& d = call.desc;
  const int code = d.activation, n_conv = (code >> 24) & 0xff, low = code & 0xffffff;
  if (const int rc = eval_cnn_code_check(code, ESTK_ERR_UNSUPPORTED, who)) return rc;
  if (const int rc = eval_returns_check(ctx, call, who)) return rc;
  if (const int rc = eval_cnn_batch_check(code, call.B, who)) return rc;

  CnnParams p = {};
  if (const int rc = cnn_parse(d, n_conv, p, who)) return rc;
  p.theta = call.theta; p.table = call.table; p.offsets = call.offsets; p.order = call.order;
  p.pairs = call.pairs; p.sigma = call.sigma; p.obs = call.obs; p.target = call.target; p.B = call.B;
  p.ret_plus = call.ret_plus; p.ret_minus = call.ret_minus;
  p.bc_plus = call.bc_plus; p.bc_minus = call.bc_minus; p.bc_obs = call.bc_obs; p.bc_dim = call.bc_dim;
  return launch_code(ctx, p, low, estk_head(low), stream, who);
}

extern "C" int estk_act_cnn(estk_ctx* ctx, const estk_mlp_desc* desc, const float* theta, const float* table,
                            const int64_t* offsets, const int32_t* order, int32_t pairs, float sigma,
                            const float* obs, int32_t B, float* out_plus, float* out_minus, void* stream) {
  const char* who = "estk_act_cnn";
  const bool centre = offsets == nullptr;
  ESTK_CHECK_ARG(ctx && desc && theta && obs && out_plus, "%s: null context, desc, theta, obs or out_plus", who);
  ESTK_CHECK_ARG(centre || (table && out_minus), "%s: a population needs table and out_minus", who);
  ESTK_CHECK_ARG(B >= 1, "%s: B=%d must be positive", who, B);
  ESTK_CHECK_ARG(centre || (pairs >= 1 && pairs <= ESTK_MAX_POPULATION / 2), "%s: pairs=%d is outside 1..%d", who,
                 pairs, ESTK_MAX_POPULATION / 2);
  const estk_mlp_desc& d = *desc;
  const int code = d.activation, n_conv = (code >> 24) & 0xff, low = code & 0xffffff, hid = low & 0xff;
  ESTK_CHECK_ARG(n_conv >= 1 && n_conv <= 7, "%s: n_conv=%d (bits 24-31 of activation 0x%x) is outside 1..7", who,
                 n_conv, code);
  ESTK_CHECK_ARG((low & ~0xff) == ESTK_ACTIONS || (low & ~0xff) == (ESTK_ACTIONS | ESTK_ACT_OUT_TANH),
                 "%s: activation=0x%x: bits 8-23 must be ESTK_ACTIONS, optionally with ESTK_ACT_OUT_TANH", who, code);
  ESTK_CHECK_ARG(estk_in(EstkHiddenKinds{}, hid), "%s: activation=0x%x: bits 0-7 are not a hidden kind", who, code);

  CnnParams p = {};
  if (const int rc = cnn_parse(d, n_conv, p, who)) return rc;
  p.theta = theta; p.obs = obs; p.B = B; p.out_plus = out_plus;
  if (centre) {
    p.pairs = 1;
  } else {
    p.table = table; p.offsets = offsets; p.order = order; p.pairs = pairs; p.sigma = sigma; p.out_minus = out_minus;
  }
  const int head = kHeadAct | ((low & ESTK_ACT_OUT_TANH) ? kHeadTanh : kHeadIdentity);
  return launch_code(ctx, p, low, head, (cudaStream_t)stream, who);
}
