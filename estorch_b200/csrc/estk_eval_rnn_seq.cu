// estk_eval_rnn_seq.cu -- estk_eval_mlp with a recurrent cell code (ESTK_CELL_GRU / ESTK_CELL_LSTM) and a
// return (the squared error, or ESTK_LOSS_XENT), fp32: the sequence evaluate.  Every perturbed recurrent
// policy runs over a fixed batch of B sequences of T steps from a zero state, and its return scores all
// B*T steps -- the device-agent evaluate of a policy with memory (delayed recall, sequence classification,
// time-series regression).
//
// One work item = one antithetic pair x one chunk of BC sequences, as in act_rnn_kernel (estk_act_rnn.cu):
// the pair's noise row is read once for both signs, and every weight tile is formed in shared memory as
// W+ = theta + sigma*t and W- = theta - sigma*t.  The 2*BC rows (sign-major) keep their state (h, and c for
// LSTM) on chip across all T steps; each step stages x_t, then runs the step of act_rnn_kernel element by
// element -- the gate chains, the cell update, the head -- so a member's outputs are the bits that T chained
// ESTK_ACTIONS launches produce when each is fed the previous one's state.  The weight tiles are formed again
// at every step (the "streamed" form: it serves every shape).  After the head, one thread per row scores the
// step; the per-sequence sums go to the context workspace, and the item that arrives last sums them in
// sequence order (include/estk.h states the order: the bits do not depend on BC or the schedule; no float
// atomics).
//
// The activations ([width][ROWS], k-major: x_t|h, the gate buffer, c, the head's outputs) stay in shared
// memory when they fit the budget below; otherwise they live in a per-CTA slab of the context workspace and
// a persistent grid loops over the work items (the same code, global instead of shared addresses).
//
// Algorithmic bytes per launch = 4*n*pairs (noise rows) + 4*n (theta) + 4*B*T*(in+out) (observations and
// targets) + 4*P (returns); the weights are re-formed T times per work item from L1 / L2.
#include "estk_common.cuh"
#include <algorithm>
#include <climits>

namespace {

constexpr int kThreads = 256;
constexpr int KT = 32;                       // k-chunk of the weight tile
// activations + tiles in shared memory, up to the 227 KB a CTA may hold; above it the activations stream
// through the slab (DESIGN §9 has this budget against 96 KB at H = 128 - 256)
constexpr size_t kSmemBudget = 220 * 1024;
constexpr int kHeadIdentity = 0, kHeadTanh = 1, kHeadXent = 2;

// row groups per CTA: 2 (one per sign) for a single row per sign, else 4
__host__ __device__ constexpr int seq_groups(int bc) { return bc == 1 ? 2 : 4; }
__host__ __device__ constexpr int seq_ot(int bc) { return kThreads / seq_groups(bc); }   // outputs per tile
__host__ __device__ constexpr int seq_gates(int cell) { return cell == ESTK_CELL_GRU ? 3 : 4; }

// floats of one work item's activations per row: x_t|h, the gate buffer (GRU: + b_n), c (LSTM), the head's outputs
__host__ __device__ inline int seq_act_width(int cell, int in, int H, int out) {
  return in + H + seq_gates(cell) * H + H + out;
}

struct SeqParams {
  int in, H, out, T;
  const float* theta;
  const float* table;
  const int64_t* offsets;    // null => centre (theta, sigma ignored, no - member)
  const int32_t* order;
  int pairs;
  float sigma;
  const float* obs;          // [B][T][in]
  const float* target;       // [B][T][out]
  int B, chunks;
  float* ret_plus;
  float* ret_minus;
  float* bc_plus;            // [pairs][bc_dim]: y of the first bc_obs sequences, (b, t, c) order
  float* bc_minus;
  int bc_obs, bc_dim;
  float* partial;            // [pairs][2][B] per-sequence loss sums
  unsigned int* counters;    // [pairs], zero on entry, zero on exit
  float* slab;               // SLAB: [gridDim.x][act_floats / ROWS][ROWS]
};

template <int BC, int CELL, int HEAD, bool SLAB>
__global__ void __launch_bounds__(kThreads, SLAB ? 1 : 2) eval_rnn_seq_kernel(const SeqParams p) {
  constexpr bool GRU = CELL == ESTK_CELL_GRU;
  constexpr int NG = seq_gates(CELL);
  constexpr int ROWS = 2 * BC;
  constexpr int RG = seq_groups(BC), OT = seq_ot(BC), OTP = OT + 1;  // +1: conflict-free tile stores
  constexpr int RSTEP = RG / 2;                                      // row groups per sign
  constexpr int NB = (BC + RSTEP - 1) / RSTEP;                       // rows per thread
  extern __shared__ __align__(16) float smem[];
  const int in = p.in, H = p.H, out = p.out, T = p.T, GH = NG * H, KX = in + H;
  float* const Wp = smem;                     // [KT][OTP]
  float* const Wm = Wp + KT * OTP;            // [KT][OTP]
  float* const X = SLAB ? p.slab + (size_t)blockIdx.x * seq_act_width(CELL, in, H, out) * ROWS : Wm + KT * OTP;
  float* const Gt = X + (size_t)KX * ROWS;                          // [GH (+H for GRU's b_n)][ROWS]
  float* const Cs = Gt + (size_t)(GH + (GRU ? H : 0)) * ROWS;       // LSTM: [H][ROWS]
  float* const Y = Cs + (size_t)(GRU ? 0 : H) * ROWS;               // [out][ROWS]

  const int tid = threadIdx.x;
  const int c = tid % OT, q = tid / OT;
  const bool minus = (q & 1) != 0;
  const int bsub = q >> 1;                    // this thread's rows: b = bsub + RSTEP*i, row = minus*BC + b
  const float* const Wsel = minus ? Wm : Wp;
  const bool centre = (p.offsets == nullptr);
  const float sigma = centre ? 0.f : p.sigma;
  // parameter layout (torch's): W_ih [GH][in], W_hh [GH][H], b_ih [GH], b_hh [GH], W_head [out][H], b_head [out]
  const int64_t w_hh = (int64_t)GH * in, b_ih = w_hh + (int64_t)GH * H, b_hh = b_ih + GH;
  const int64_t w_head = b_hh + GH, b_head = w_head + (int64_t)out * H;

  // work items (slot, chunk), slot-major, strided by the grid; 32-bit index arithmetic
  unsigned int slot = blockIdx.x / (unsigned)p.chunks, chunk = blockIdx.x % (unsigned)p.chunks;
  for (; slot < (unsigned)p.pairs; chunk += gridDim.x, slot += chunk / p.chunks, chunk %= p.chunks) {
    const int j = p.order ? p.order[slot] : (int)slot;
    const float* const trow = centre ? p.theta : p.table + p.offsets[j];
    const int b0 = chunk * BC;
    // W+ / W- of parameter idx: theta +- (sigma*t), two roundings
    auto wpm = [&](int64_t idx, float& wp, float& wm) {
      const float th = __ldg(p.theta + idx);
      const float ep = __fmul_rn(sigma, ld_noise1(trow + idx));
      wp = __fadd_rn(th, ep);
      wm = __fsub_rn(th, ep);
    };
    // acc[i] = fmaf chain over k < K of Xs[k][row_i] * W[o0+c][k], W = this sign's weights at wbase ([nout][K])
    auto chain = [&](float (&acc)[NB], const float* Xs, int K, int64_t wbase, int o0, int nout) {
      for (int k0 = 0; k0 < K; k0 += KT) {
        __syncthreads();  // previous tile consumed (and Xs written)
        for (int e = tid; e < OT * KT; e += kThreads) {
          const int k = e % KT, o = e / KT;
          float wp = 0.f, wm = 0.f;
          if (o0 + o < nout && k0 + k < K) wpm(wbase + (int64_t)(o0 + o) * K + k0 + k, wp, wm);
          Wp[k * OTP + o] = wp;
          Wm[k * OTP + o] = wm;
        }
        __syncthreads();
        const int kmax = min(KT, K - k0);
#pragma unroll 4
        for (int k = 0; k < kmax; ++k) {
          const float w = Wsel[k * OTP + c];
          const float* xk = Xs + (size_t)(k0 + k) * ROWS + (minus ? BC : 0) + bsub;
#pragma unroll
          for (int i = 0; i < NB; ++i)
            if (bsub + RSTEP * i < BC) acc[i] = fmaf(xk[RSTEP * i], w, acc[i]);
        }
      }
    };

    __syncthreads();   // the previous item's readers of X / Gt / Cs / Y are done
    for (int idx = tid; idx < H * ROWS; idx += kThreads) {     // the zero state
      X[(size_t)in * ROWS + idx] = 0.f;
      if (!GRU) Cs[idx] = 0.f;
    }
    float rloss = 0.f;     // thread tid < ROWS: its row's loss, summed over the steps in t order

    for (int t = 0; t < T; ++t) {
      // ---- stage x_t for both signs: X[k][s*BC + b] = obs[b0+b][t][k], k < in (the last barrier of the
      //      previous step separates these writes from that step's readers of X's first `in` rows)
      for (int idx = tid; idx < BC * in; idx += kThreads) {
        const int b = idx / in, k = idx % in;
        const float x = b0 + b < p.B ? __ldg(p.obs + ((size_t)(b0 + b) * T + t) * in + k) : 0.f;
        X[k * ROWS + b] = x;
        X[k * ROWS + BC + b] = x;
      }

      // ---- 1. gate pre-activations (act_rnn_kernel's)
      for (int o0 = 0; o0 < GH; o0 += OT) {
        float ai[NB], ah[NB];
#pragma unroll
        for (int i = 0; i < NB; ++i) ai[i] = ah[i] = 0.f;
        chain(ai, X, in, 0, o0, GH);
        chain(ah, X + (size_t)in * ROWS, H, w_hh, o0, GH);
        const int o = o0 + c;
        if (o < GH) {
          float bp, bm, hp, hm;
          wpm(b_ih + o, bp, bm);
          wpm(b_hh + o, hp, hm);
          const float bi = minus ? bm : bp, bh = minus ? hm : hp;
#pragma unroll
          for (int i = 0; i < NB; ++i) {
            const int bl = bsub + RSTEP * i;
            if (bl >= BC) continue;
            const int r = (minus ? BC : 0) + bl;
            const float a = ai[i] + bi, b = ah[i] + bh;
            if (GRU && o >= 2 * H) {
              Gt[(size_t)o * ROWS + r] = a;
              Gt[(size_t)(o + H) * ROWS + r] = b;      // b_n at rows GH .. GH + H
            } else {
              Gt[(size_t)o * ROWS + r] = a + b;
            }
          }
        }
      }
      __syncthreads();

      // ---- 2. the cell update, elementwise: h' replaces h in X (and c' replaces c)
      for (int idx = tid; idx < ROWS * H; idx += kThreads) {
        const int r = idx % ROWS, u = idx / ROWS;
        float* const hp = X + (size_t)(in + u) * ROWS + r;
        const float h = *hp;
        float hn;
        if constexpr (GRU) {
          const float rg = estk_sigmoid_rn(Gt[(size_t)u * ROWS + r]);
          const float z = estk_sigmoid_rn(Gt[(size_t)(H + u) * ROWS + r]);
          const float n = tanhf(fmaf(rg, Gt[(size_t)(GH + u) * ROWS + r], Gt[(size_t)(2 * H + u) * ROWS + r]));
          hn = fmaf(z, h - n, n);
        } else {
          const float ig = estk_sigmoid_rn(Gt[(size_t)u * ROWS + r]);
          const float fg = estk_sigmoid_rn(Gt[(size_t)(H + u) * ROWS + r]);
          const float gg = tanhf(Gt[(size_t)(2 * H + u) * ROWS + r]);
          const float og = estk_sigmoid_rn(Gt[(size_t)(3 * H + u) * ROWS + r]);
          const float cn = fmaf(fg, Cs[(size_t)u * ROWS + r], ig * gg);
          Cs[(size_t)u * ROWS + r] = cn;
          hn = og * tanhf(cn);
        }
        *hp = hn;
      }

      // ---- 3. the head on h' (chain's first __syncthreads orders it after the h' writes)
      for (int o0 = 0; o0 < out; o0 += OT) {
        float acc[NB];
#pragma unroll
        for (int i = 0; i < NB; ++i) acc[i] = 0.f;
        chain(acc, X + (size_t)in * ROWS, H, w_head, o0, out);
        const int o = o0 + c;
        if (o < out) {
          float bp, bm;
          wpm(b_head + o, bp, bm);
          const float bias = minus ? bm : bp;
          float* const bc = minus ? p.bc_minus : p.bc_plus;
#pragma unroll
          for (int i = 0; i < NB; ++i) {
            const int bl = bsub + RSTEP * i;
            if (bl >= BC) continue;
            float y = acc[i] + bias;
            if constexpr (HEAD == kHeadTanh) y = tanhf(y);
            Y[(size_t)o * ROWS + (minus ? BC : 0) + bl] = y;
            const int b = b0 + bl;
            const int64_t e = ((int64_t)b * T + t) * out + o;
            if (bc && !(centre && minus) && b < p.B && b < p.bc_obs && e < p.bc_dim) bc[(size_t)j * p.bc_dim + e] = y;
          }
        }
      }
      __syncthreads();

      // ---- 4. thread r < ROWS scores step t of row r in column order
      const int b = b0 + tid % BC;
      if (tid < ROWS && b < p.B) {
        const float* const tg = p.target + ((size_t)b * T + t) * out;
        float s;
        if constexpr (HEAD == kHeadXent) {
          float m = -INFINITY;
          for (int o = 0; o < out; ++o) m = fmaxf(m, Y[(size_t)o * ROWS + tid]);
          float se = 0.f, st = 0.f, sty = 0.f;
          for (int o = 0; o < out; ++o) {
            const float y = Y[(size_t)o * ROWS + tid], tv = __ldg(tg + o);
            se += expf(y - m);
            st += tv;
            sty = fmaf(tv, y, sty);
          }
          s = fmaf(m + logf(se), st, -sty);
        } else {
          s = 0.f;
          for (int o = 0; o < out; ++o) {
            const float d = Y[(size_t)o * ROWS + tid] - __ldg(tg + o);
            s = fmaf(d, d, s);
          }
        }
        rloss += s;
      }
      // the next step's first writes (x_t) are ordered after this step's readers of X by the barriers above;
      // Y and Gt are next written only after the next step's first chain barrier
    }

    // ---- per-sequence sums to the workspace; the last item of the pair sums them in sequence order
    const int bl = tid % BC, bb = b0 + bl;
    if (tid < ROWS && bb < p.B) {
      p.partial[((size_t)slot * 2 + tid / BC) * p.B + bb] = rloss;
      __threadfence();
    }
    __syncthreads();
    if (tid == 0) {
      const unsigned int arrived = atomicAdd(p.counters + slot, 1u);
      if (arrived == (unsigned int)p.chunks - 1) {
        __threadfence();
        const float* const part = p.partial + (size_t)slot * 2 * p.B;
        float sp = 0.f, sm = 0.f;
        for (int s = 0; s < p.B; ++s) { sp += __ldcg(part + s); sm += __ldcg(part + p.B + s); }
        const int64_t cnt = (int64_t)p.B * T * (HEAD == kHeadXent ? 1 : out);
        const float denom = (float)cnt;
        p.ret_plus[j] = -(sp / denom);
        if (p.ret_minus) p.ret_minus[j] = -(sm / denom);
        p.counters[slot] = 0u;  // ready for the next launch
      }
    }
  }
}

size_t tile_bytes(int bc) { return sizeof(float) * 2 * KT * (seq_ot(bc) + 1); }

template <int BC, int CELL, int HEAD>
int launch_seq(estk_ctx* ctx, SeqParams& p, cudaStream_t stream, const char* who) {
  p.chunks = (p.B + BC - 1) / BC;
  const int64_t items = (int64_t)p.pairs * p.chunks;
  const int64_t act_floats = (int64_t)seq_act_width(CELL, p.in, p.H, p.out) * 2 * BC;
  const size_t smem_all = tile_bytes(BC) + sizeof(float) * (size_t)act_floats;
  const bool slab = smem_all > kSmemBudget;
  auto kern = slab ? eval_rnn_seq_kernel<BC, CELL, HEAD, true> : eval_rnn_seq_kernel<BC, CELL, HEAD, false>;
  const size_t smem = slab ? tile_bytes(BC) : smem_all;
  ESTK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int grid = (int)std::min<int64_t>(items, INT_MAX);
  if (slab) {
    int per_sm = 0;
    ESTK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kThreads, smem));
    grid = (int)std::min<int64_t>(items, (int64_t)ctx->sm_count * std::max(per_sm, 1));
  }
  const int rc = estk_ctx_reserve(ctx, p.pairs, (int64_t)p.pairs * 2 * p.B, stream, who,
                                  slab ? (int64_t)grid * act_floats : 0);
  if (rc) return rc;
  p.partial = ctx->eval_partial;
  p.counters = estk_member_counters(ctx);
  p.slab = slab ? ctx->eval_slab : nullptr;
  kern<<<grid, kThreads, smem, stream>>>(p);
  ESTK_CUDA(cudaGetLastError());
  return ESTK_OK;
}

template <int BC>
int launch_bc(estk_ctx* ctx, SeqParams& p, int code, cudaStream_t stream, const char* who) {
  const int head = (code & ESTK_LOSS_XENT) ? kHeadXent : (code & ESTK_ACT_OUT_TANH) ? kHeadTanh : kHeadIdentity;
  if ((code & 0xff) == ESTK_CELL_GRU) {
    if (head == kHeadXent) return launch_seq<BC, ESTK_CELL_GRU, kHeadXent>(ctx, p, stream, who);
    if (head == kHeadTanh) return launch_seq<BC, ESTK_CELL_GRU, kHeadTanh>(ctx, p, stream, who);
    return launch_seq<BC, ESTK_CELL_GRU, kHeadIdentity>(ctx, p, stream, who);
  }
  if (head == kHeadXent) return launch_seq<BC, ESTK_CELL_LSTM, kHeadXent>(ctx, p, stream, who);
  if (head == kHeadTanh) return launch_seq<BC, ESTK_CELL_LSTM, kHeadTanh>(ctx, p, stream, who);
  return launch_seq<BC, ESTK_CELL_LSTM, kHeadIdentity>(ctx, p, stream, who);
}

}  // namespace

int eval_rnn_sequence(estk_ctx* ctx, const estk_mlp_desc* desc, int precision, const float* theta,
                      const float* table, const int64_t* offsets, const int32_t* order, int pairs, float sigma,
                      const float* obs, const float* target, int B, float* returns_plus, float* returns_minus,
                      float* bc_plus, float* bc_minus, int bc_obs, int bc_dim, const float* centre_return_out,
                      cudaStream_t stream) {
  const char* who = "estk_eval_mlp[recurrent cell, sequence]";
  const bool centre = offsets == nullptr;
  ESTK_CHECK_ARG(precision == ESTK_PREC_FP32 || precision == ESTK_PREC_F16 || precision == ESTK_PREC_BF16 ||
                 precision == ESTK_PREC_BF16S || precision == ESTK_PREC_F16_ANY, "%s: unknown precision %d", who,
                 precision);
  if (precision != ESTK_PREC_FP32) {
    estk_set_error("%s: the sequence evaluate is computed with ESTK_PREC_FP32 only (precision %d)", who, precision);
    return ESTK_ERR_UNSUPPORTED;
  }
  if (centre_return_out) {
    estk_set_error("%s: centre_return_out (folded centre rollout) needs a tensor-core precision", who);
    return ESTK_ERR_UNSUPPORTED;
  }
  ESTK_CHECK_ARG(ctx && theta && obs && target && returns_plus && (centre || (table && returns_minus)),
                 "%s: null argument (theta, obs, target, returns_plus, and for a population table and "
                 "returns_minus)", who);
  ESTK_CHECK_ARG(centre || (bc_plus == nullptr) == (bc_minus == nullptr),
                 "%s: bc_plus/bc_minus must both be set or both null", who);
  ESTK_CHECK_ARG(!bc_plus || (bc_obs > 0 && bc_dim > 0), "%s: bc_obs/bc_dim must be positive with bc outputs", who);
  const estk_mlp_desc& d = *desc;
  ESTK_CHECK_ARG(d.n_layers == 2, "%s: a recurrent cell is n_layers = 2, dims = (in, H, out, T) (n_layers=%d)", who,
                 d.n_layers);
  for (int l = 0; l <= 2; ++l) ESTK_CHECK_ARG(d.dims[l] >= 1, "%s: dims[%d]=%d", who, l, d.dims[l]);
  ESTK_CHECK_ARG(d.dims[3] >= 1, "%s: dims[3] = T, the number of steps, must be positive (T=%d)", who, d.dims[3]);
  // the parameter count and every row width fit comfortably in 32 bits for the widths accepted here
  ESTK_CHECK_ARG(d.dims[0] <= (1 << 16) && d.dims[1] <= (1 << 13) && d.dims[2] <= (1 << 16),
                 "%s: dims (%d, %d, %d) exceed (65536, 8192, 65536)", who, d.dims[0], d.dims[1], d.dims[2]);
  ESTK_CHECK_ARG(B >= 1, "%s: B must be positive", who);
  ESTK_CHECK_ARG(centre || (pairs >= 1 && pairs <= ESTK_MAX_POPULATION / 2), "%s: pairs=%d", who, pairs);
  SeqParams p = {};
  p.in = d.dims[0]; p.H = d.dims[1]; p.out = d.dims[2]; p.T = d.dims[3];
  p.theta = theta; p.offsets = offsets; p.obs = obs; p.target = target; p.B = B;
  p.ret_plus = returns_plus; p.bc_plus = bc_plus; p.bc_obs = bc_obs; p.bc_dim = bc_dim;
  if (centre) {
    p.pairs = 1;
  } else {
    p.table = table; p.order = order; p.pairs = pairs; p.sigma = sigma;
    p.ret_minus = returns_minus; p.bc_minus = bc_minus;
  }
  // chunk of sequences per work item: the bits do not depend on it (the returns are summed per sequence)
  if (B == 1) return launch_bc<1>(ctx, p, d.activation, stream, who);
  if (B <= 4) return launch_bc<4>(ctx, p, d.activation, stream, who);
  return launch_bc<16>(ctx, p, d.activation, stream, who);
}
