// estk_act_rnn.cu -- estk_eval_mlp with a recurrent cell code (ESTK_CELL_GRU / ESTK_CELL_LSTM) and
// ESTK_ACTIONS (fp32): one step of every perturbed recurrent policy on that member's own observation and
// state, the per-step operation of an environment population whose policy has memory.
//
// The policy is one torch.nn.GRUCell / nn.LSTMCell (in -> H) and one Linear head (H -> out) [+ Tanh]; the
// step is the function [x | state] -> [y | state'], so observations and outputs carry the state:
// obs rows are in + S wide, output rows out + S, with S = H (GRU: h) or 2H (LSTM: h then c).
//
// One CTA = one antithetic pair x one chunk of BC observations per member, as eval_mlp_act_kernel
// (estk_eval_mlp_act.cu): the pair's noise row is read once for both signs, and every weight tile is
// formed in shared memory as W+ = theta + sigma*t and W- = theta - sigma*t.  Thread = one output column x
// NB rows of one sign.  Per step:
//   1. gates: per gate row g < G*H two fmaf chains from 0 in ascending k -- x against W_ih[g] and h against
//      W_hh[g] -- each + its own bias; the pre-activation a + b goes to the gate buffer (GRU's n gate keeps
//      a and b apart: n = tanhf(fmaf(r, b_n, a_n)));
//   2. the cell update, elementwise: h' (and c') into the head's input and the output row;
//   3. the head: the fp32 act kernel's layer on h' (+ bias, tanhf for ESTK_ACT_OUT_TANH).
// include/estk.h states the arithmetic.  No float atomics: the bits do not depend on the schedule.
//
// The activations ([width][ROWS], k-major: x|h, the gate buffer, h') stay in shared memory when they fit
// in the budget below; otherwise they live in a per-CTA slab of the context workspace and a persistent
// grid loops over the work items (the same code, global instead of shared addresses).
//
// Algorithmic bytes per launch = 4*n*pairs (noise rows; 2*n*pairs from table16) + 4*n (theta)
// + 4*P*B*(in+out+2S) (observations, state and outputs).
#include "estk_common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int KT = 32;                       // k-chunk of the weight tile
constexpr size_t kSmemBudget = 96 * 1024;    // activations + tiles; above it the activations stream

// row groups per CTA: 2 (one per sign) for a single row per sign, else 4
__host__ __device__ constexpr int rnn_groups(int bc) { return bc == 1 ? 2 : 4; }
__host__ __device__ constexpr int rnn_ot(int bc) { return kThreads / rnn_groups(bc); }   // outputs per tile
__host__ __device__ constexpr int cell_gates(int cell) { return cell == ESTK_CELL_GRU ? 3 : 4; }

struct RnnParams {
  int in, H, out;
  const float* theta;
  const float* table;
  const uint16_t* table16;   // non-null: read instead of table (its exact fp16 copy)
  const int64_t* offsets;    // null => centre (theta, sigma ignored, no - member)
  const int32_t* order;
  int pairs;
  float sigma;
  const float* obs;          // population [2*pairs][B][in+S], centre [B][in+S]
  int B, chunks;
  float* bc_plus;            // population [pairs][bc_dim], rows [B][out+S]
  float* bc_minus;
  int bc_obs, bc_dim;
  float* slab;               // SLAB: [gridDim.x][act_floats / ROWS][ROWS]
};

// floats of one work item's activations per row: x|h, the gate buffer (GRU: + b_n), h'
__host__ __device__ inline int rnn_act_width(int cell, int in, int H) {
  return in + H + cell_gates(cell) * H + (cell == ESTK_CELL_GRU ? H : 0) + H;
}

template <int BC, int CELL, bool OUT_TANH, bool SLAB>
__global__ void __launch_bounds__(kThreads, 3) act_rnn_kernel(const RnnParams p) {
  constexpr bool GRU = CELL == ESTK_CELL_GRU;
  constexpr int NG = cell_gates(CELL);
  constexpr int ROWS = 2 * BC;
  constexpr int RG = rnn_groups(BC), OT = rnn_ot(BC), OTP = OT + 1;  // +1: conflict-free tile stores
  constexpr int RSTEP = RG / 2;                                      // row groups per sign
  constexpr int NB = (BC + RSTEP - 1) / RSTEP;                       // rows per thread
  extern __shared__ __align__(16) float smem[];
  const int in = p.in, H = p.H, out = p.out, GH = NG * H;
  const int S = GRU ? H : 2 * H, KX = in + H, XW = in + S, YW = out + S;
  float* const Wp = smem;                     // [KT][OTP]
  float* const Wm = Wp + KT * OTP;            // [KT][OTP]
  float* const X = SLAB ? p.slab + (size_t)blockIdx.x * rnn_act_width(CELL, in, H) * ROWS : Wm + KT * OTP;
  float* const Gt = X + (size_t)KX * ROWS;                          // [GH (+H for GRU's b_n)][ROWS]
  float* const Hn = Gt + (size_t)(GH + (GRU ? H : 0)) * ROWS;       // [H][ROWS]

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
    const int64_t toff = centre ? 0 : p.offsets[j];
    const NoiseRow nz{centre ? p.theta : p.table + toff, (centre || !p.table16) ? nullptr : p.table16 + toff};
    const int b0 = chunk * BC;
    // acc[i] = fmaf chain over k < K of Xs[k][row_i] * W[o0+c][k], W = this sign's weights at wbase ([nout][K])
    auto chain = [&](float (&acc)[NB], const float* Xs, int K, int64_t wbase, int o0, int nout) {
      for (int k0 = 0; k0 < K; k0 += KT) {
        __syncthreads();  // previous tile consumed (and Xs written)
        for (int e = tid; e < OT * KT; e += kThreads) {
          const int k = e % KT, o = e / KT;
          float wp = 0.f, wm = 0.f;
          if (o0 + o < nout && k0 + k < K)
            estk_form_pm(p.theta, nz, sigma, wbase + (int64_t)(o0 + o) * K + k0 + k, wp, wm);
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
    auto member_of = [&](int s) -> int64_t { return s ? (int64_t)p.pairs + j : j; };

    __syncthreads();   // the previous item's readers of X / Gt / Hn are done
    // ---- stage each member's own x | h: X[k][s*BC + b] = obs[member_s][b0+b][k], k < in + H
    for (int idx = tid; idx < ROWS * KX; idx += kThreads) {
      const int r = idx / KX, k = idx % KX;
      const int s = r / BC, b = r % BC;
      const bool ok = b0 + b < p.B && !(centre && s);
      X[k * ROWS + r] = ok ? __ldg(p.obs + ((size_t)member_of(s) * p.B + b0 + b) * XW + k) : 0.f;
    }

    // ---- 1. gate pre-activations
    for (int o0 = 0; o0 < GH; o0 += OT) {
      float ai[NB], ah[NB];
#pragma unroll
      for (int i = 0; i < NB; ++i) ai[i] = ah[i] = 0.f;
      chain(ai, X, in, 0, o0, GH);
      chain(ah, X + (size_t)in * ROWS, H, w_hh, o0, GH);
      const int o = o0 + c;
      if (o < GH) {
        float bp, bm, hp, hm;
        estk_form_pm(p.theta, nz, sigma, b_ih + o, bp, bm);
        estk_form_pm(p.theta, nz, sigma, b_hh + o, hp, hm);
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

    // ---- 2. the cell update, elementwise: h' -> Hn and the output row (LSTM: c' too)
    for (int idx = tid; idx < ROWS * H; idx += kThreads) {
      const int r = idx % ROWS, u = idx / ROWS;
      const int s = r / BC, b = r % BC;
      const float h = X[(size_t)(in + u) * ROWS + r];
      float hn, cn = 0.f;
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
        const bool ok = b0 + b < p.B && !(centre && s);
        const float cc = ok ? __ldg(p.obs + ((size_t)member_of(s) * p.B + b0 + b) * XW + in + H + u) : 0.f;
        cn = fmaf(fg, cc, ig * gg);
        hn = og * tanhf(cn);
      }
      Hn[(size_t)u * ROWS + r] = hn;
      const int bb = b0 + b;
      if (!(centre && s) && bb < p.B && bb < p.bc_obs) {
        float* const bc = (s ? p.bc_minus : p.bc_plus) + (size_t)j * p.bc_dim;
        const int64_t e = (int64_t)bb * YW + out + u;
        if (e < p.bc_dim) bc[e] = hn;
        if (!GRU && e + H < p.bc_dim) bc[e + H] = cn;
      }
    }

    // ---- 3. the head on h' (chain's first __syncthreads orders it after the Hn writes)
    for (int o0 = 0; o0 < out; o0 += OT) {
      float acc[NB];
#pragma unroll
      for (int i = 0; i < NB; ++i) acc[i] = 0.f;
      chain(acc, Hn, H, w_head, o0, out);
      const int o = o0 + c;
      if (o < out) {
        float bp, bm;
        estk_form_pm(p.theta, nz, sigma, b_head + o, bp, bm);
        const float bias = minus ? bm : bp;
        float* const bc = minus ? p.bc_minus : p.bc_plus;
#pragma unroll
        for (int i = 0; i < NB; ++i) {
          const int bl = bsub + RSTEP * i;
          if (bl >= BC) continue;
          float y = acc[i] + bias;
          if constexpr (OUT_TANH) y = tanhf(y);
          const int b = b0 + bl;
          const int64_t e = (int64_t)b * YW + o;
          if (!(centre && minus) && b < p.B && b < p.bc_obs && e < p.bc_dim) bc[(size_t)j * p.bc_dim + e] = y;
        }
      }
    }
  }
}

size_t tile_bytes(int bc) { return sizeof(float) * 2 * KT * (rnn_ot(bc) + 1); }

template <int BC, int CELL, bool OUT_TANH>
int launch_rnn(estk_ctx* ctx, RnnParams& p, cudaStream_t stream, const char* who) {
  SlabLaunch l = {};
  l.items = (int64_t)p.pairs * p.chunks;
  l.slab_per_cta = (int64_t)rnn_act_width(CELL, p.in, p.H) * 2 * BC;
  l.smem_slab = tile_bytes(BC);
  l.smem_shared = l.smem_slab + sizeof(float) * (size_t)l.slab_per_cta;
  l.slab = l.smem_shared > kSmemBudget;
  return estk_launch_eval(ctx, act_rnn_kernel<BC, CELL, OUT_TANH, false>, act_rnn_kernel<BC, CELL, OUT_TANH, true>, p,
                          l, kThreads, stream, who, [] {});
}


}  // namespace

int eval_rnn_actions(estk_ctx* ctx, const EvalMlpCall& c, cudaStream_t stream) {
  const char* who = "estk_eval_mlp[recurrent cell, ESTK_ACTIONS]";
  if (const int rc = eval_actions_check(ctx, c)) return rc;
  const estk_mlp_desc& d = c.desc;
  ESTK_CHECK_ARG(d.n_layers == 2, "%s: a recurrent cell is n_layers = 2, dims = (in, H, out) (n_layers=%d)", who,
                 d.n_layers);
  for (int l = 0; l <= 2; ++l) ESTK_CHECK_ARG(d.dims[l] >= 1, "%s: dims[%d]=%d", who, l, d.dims[l]);
  // the parameter count and every row width fit comfortably in 32 bits for the widths accepted here
  ESTK_CHECK_ARG(d.dims[0] <= (1 << 16) && d.dims[1] <= (1 << 13) && d.dims[2] <= (1 << 16),
                 "%s: dims (%d, %d, %d) exceed (65536, 8192, 65536)", who, d.dims[0], d.dims[1], d.dims[2]);
  ESTK_CHECK_ARG(c.B >= 1, "%s: B must be positive", who);
  ESTK_CHECK_ARG(c.pairs >= 1 && c.pairs <= ESTK_MAX_POPULATION / 2, "%s: pairs=%d", who, c.pairs);
  RnnParams p = {};
  p.in = d.dims[0]; p.H = d.dims[1]; p.out = d.dims[2];
  p.theta = c.theta; p.table = c.table; p.table16 = c.table16; p.offsets = c.offsets; p.order = c.order;
  p.pairs = c.pairs; p.sigma = c.sigma; p.obs = c.obs; p.B = c.B;
  p.bc_plus = c.bc_plus; p.bc_minus = c.bc_minus; p.bc_obs = c.bc_obs; p.bc_dim = c.bc_dim;
  const int bc = estk_chunk_rows(c.B);
  p.chunks = (c.B + bc - 1) / bc;
  return estk_dispatch(EstkChunkRows{}, bc, [&](auto BC) {
    return estk_dispatch(EstkCells{}, d.activation & 0xff, [&](auto CELL) {
      return estk_dispatch(EstkActionOutputs{}, d.activation & ESTK_ACT_OUT_TANH,
                           [&](auto O) { return launch_rnn<BC, CELL, O != 0>(ctx, p, stream, who); });
    });
  });
}
