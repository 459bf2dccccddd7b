// estk_eval_mlp.cu -- kernel 1 of the ES generation (fp32 CUDA-core path):
// population evaluate for MLP policies over a synthetic observation batch.
//
// Replaces (reference file:line, /root/reference):
//   ES._sample_policy        estorch/estorch.py:187-193   theta +- sigma*eps, never materialised
//   ES._calculate_returns    estorch/estorch.py:195-202   vector_to_parameters + rollout per row
//   Policy.forward           examples/cartpole_es.py:14-20 (Linear-ReLU-Linear-ReLU-Linear; or Tanh
//                            hidden and / or output activations, estk.h ESTK_ACT_*)
//   Agent.rollout            synthetic agent of SURVEY 8d: -mean((policy(obs)-y)^2), or the
//                            soft-target cross-entropy (ESTK_LOSS_XENT), or the accuracy
//                            (ESTK_LOSS_ACCURACY)
//                            (+ behaviour characteristic, examples/nsra_es.py:45-49)
//
// One CTA = one antithetic pair x one chunk of BC observations.  The pair's
// noise row is read ONCE and serves both signs: each weight tile is formed in
// shared memory as W+ = theta + sigma*t and W- = theta - sigma*t (same two
// roundings as the reference: eps = sigma*t, then theta +- eps) and multiplied
// into the + and - activation rows.  Activations stay in shared memory across
// layers (k-major [width][ROWS], ROWS = 2*BC rows = sign-major), register tile
// 4 rows x 4 outputs per thread.  The last layer is fused with the squared
// error; with the cross-entropy it writes the logits to shared memory like a hidden
// layer, and one thread per row then reduces its row in column order (the accuracy likewise: the
// first argmax of the logits and of the target row, 1 per row where they agree).  Chunk partial sums are combined in fixed order by the last-arriving
// chunk CTA (deterministic, no float atomics).
//
// This is the exact-fp32 path used for parity and for small policies; algorithmic
// bytes per launch = 4*n*pairs (noise rows) + 4*n (theta) + 4*B*(in+out) + 4*P.
#include "estk_common.cuh"
#include <algorithm>

namespace {

constexpr int kThreads = 256;
constexpr int KT = 32;  // k-chunk of the weight tile

struct EvalParams {
  estk_mlp_desc desc;
  const float* theta;
  const float* table;
  const int64_t* offsets;  // null => centre evaluation (sigma ignored)
  const int32_t* order;
  int pairs;
  float sigma;
  const float* obs;
  const float* target;
  int B, BC, chunks, maxw;
  float* ret_plus;
  float* ret_minus;
  float* bc_plus;
  float* bc_minus;
  int bc_obs, bc_dim;
  float* partial;          // [pairs][2][chunks]
  unsigned int* counters;  // [pairs], zero on entry, zero on exit
};

// ACT = estk_mlp_desc.activation (a compile-time constant, so the ReLU / squared-error
// instantiations are the code they were before Tanh and the cross-entropy existed)
template <int ROWS, int ACT>
__global__ void __launch_bounds__(kThreads) eval_mlp_kernel(const EvalParams p) {
  constexpr int HID = ACT & 0xff;
  constexpr bool OUT_TANH = (ACT & ESTK_ACT_OUT_TANH) != 0;
  constexpr bool XENT = (ACT & ESTK_LOSS_XENT) != 0;
  constexpr bool ACC = (ACT & 0xff0000) == ESTK_LOSS_ACCURACY;
  constexpr int OT = 4096 / ROWS;  // output features per tile
  constexpr int OTP = OT + 4;      // padded row of the weight tile (keeps float4 alignment)
  constexpr int TC = OT / 4;       // thread columns
  constexpr int BC = ROWS / 2;
  extern __shared__ __align__(16) float smem[];
  float* X = smem;                             // [maxw][ROWS]
  float* Y = X + (size_t)p.maxw * ROWS;        // [maxw][ROWS]
  float* Wp = Y + (size_t)p.maxw * ROWS;       // [KT][OTP]
  float* Wm = Wp + KT * OTP;                   // [KT][OTP]
  __shared__ float s_red[2][kThreads / 32];
  __shared__ bool s_last;

  const int tid = threadIdx.x;
  const int slot = blockIdx.x / p.chunks;
  const int chunk = blockIdx.x % p.chunks;
  const int j = p.order ? p.order[slot] : slot;
  const bool centre = (p.offsets == nullptr);
  const NoiseRow nz{centre ? p.theta : p.table + p.offsets[j], nullptr};   // the fp32 table only
  const float sigma = centre ? 0.f : p.sigma;
  const int b0 = chunk * BC;
  const int L = p.desc.n_layers;

  // ---- stage the observation chunk for both signs: X[k][s*BC + b] = obs[b0+b][k]
  {
    const int in0 = p.desc.dims[0];
    for (int idx = tid; idx < BC * in0; idx += kThreads) {
      const int b = idx / in0, k = idx % in0;
      const float x = (b0 + b < p.B) ? __ldg(p.obs + (size_t)(b0 + b) * in0 + k) : 0.f;
      X[k * ROWS + b] = x;
      X[k * ROWS + BC + b] = x;
    }
  }

  const int tc = tid % TC;
  const int tr = tid / TC;
  const int r0 = tr * 4;                 // first of this thread's 4 rows
  const bool minus = r0 >= BC;           // all 4 rows share the sign
  const float* Wsel = minus ? Wm : Wp;
  float loss = 0.f;
  int64_t pbase = 0;

  for (int l = 0; l < L; ++l) {
    const int in = p.desc.dims[l], out = p.desc.dims[l + 1];
    const int64_t wbase = pbase, bbase = pbase + (int64_t)in * out;
    const bool last = (l == L - 1);
    for (int o0 = 0; o0 < out; o0 += OT) {
      float acc[4][4];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[i][c] = 0.f;
      for (int k0 = 0; k0 < in; k0 += KT) {
        __syncthreads();  // previous tile fully consumed (and X staged on first pass)
        // weight tile: element (o, k) <- theta/noise[wbase + (o0+o)*in + k0+k]
        for (int e = tid; e < OT * KT; e += kThreads) {
          const int k = e % KT, o = e / KT;
          float wp = 0.f, wm = 0.f;
          if (o0 + o < out && k0 + k < in) {
            const int64_t idx = wbase + (int64_t)(o0 + o) * in + k0 + k;
            const float th = __ldg(p.theta + idx);
            const float ep = __fmul_rn(sigma, nz(idx));
            wp = __fadd_rn(th, ep);
            wm = __fsub_rn(th, ep);
          }
          Wp[k * OTP + o] = wp;
          Wm[k * OTP + o] = wm;
        }
        __syncthreads();
        const int kmax = min(KT, in - k0);
#pragma unroll 4
        for (int k = 0; k < kmax; ++k) {
          const float4 x = *reinterpret_cast<const float4*>(X + (size_t)(k0 + k) * ROWS + r0);
          const float4 w = *reinterpret_cast<const float4*>(Wsel + k * OTP + tc * 4);
          acc[0][0] = fmaf(x.x, w.x, acc[0][0]); acc[0][1] = fmaf(x.x, w.y, acc[0][1]);
          acc[0][2] = fmaf(x.x, w.z, acc[0][2]); acc[0][3] = fmaf(x.x, w.w, acc[0][3]);
          acc[1][0] = fmaf(x.y, w.x, acc[1][0]); acc[1][1] = fmaf(x.y, w.y, acc[1][1]);
          acc[1][2] = fmaf(x.y, w.z, acc[1][2]); acc[1][3] = fmaf(x.y, w.w, acc[1][3]);
          acc[2][0] = fmaf(x.z, w.x, acc[2][0]); acc[2][1] = fmaf(x.z, w.y, acc[2][1]);
          acc[2][2] = fmaf(x.z, w.z, acc[2][2]); acc[2][3] = fmaf(x.z, w.w, acc[2][3]);
          acc[3][0] = fmaf(x.w, w.x, acc[3][0]); acc[3][1] = fmaf(x.w, w.y, acc[3][1]);
          acc[3][2] = fmaf(x.w, w.z, acc[3][2]); acc[3][3] = fmaf(x.w, w.w, acc[3][3]);
        }
      }
      // ---- tile epilogue: bias (+-), hidden activation or (output activation +) loss
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int o = o0 + tc * 4 + c;
        if (o >= out) continue;
        const float bias = estk_form_sign(p.theta, nz, sigma, bbase + o, minus);
        float y[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) y[i] = acc[i][c] + bias;
        if (!last) {
#pragma unroll
          for (int i = 0; i < 4; ++i) y[i] = estk_hidden_act<HID>(y[i]);
          *reinterpret_cast<float4*>(Y + (size_t)o * ROWS + r0) = make_float4(y[0], y[1], y[2], y[3]);
        } else if constexpr (XENT || ACC) {
          // the logits stay in shared memory for the row pass below
          *reinterpret_cast<float4*>(Y + (size_t)o * ROWS + r0) = make_float4(y[0], y[1], y[2], y[3]);
          float* bc = minus ? p.bc_minus : p.bc_plus;
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int b = b0 + ((r0 + i) % BC);
            const int64_t e = (int64_t)b * out + o;
            if (bc && b < p.B && b < p.bc_obs && e < p.bc_dim) bc[(size_t)j * p.bc_dim + e] = y[i];
          }
        } else {
          if constexpr (OUT_TANH) {
#pragma unroll
            for (int i = 0; i < 4; ++i) y[i] = tanhf(y[i]);
          }
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int b = b0 + ((r0 + i) % BC);
            if (b < p.B) {
              const float d = y[i] - __ldg(p.target + (size_t)b * out + o);
              loss = fmaf(d, d, loss);
              float* bc = minus ? p.bc_minus : p.bc_plus;
              const int64_t e = (int64_t)b * out + o;
              if (bc && b < p.bc_obs && e < p.bc_dim) bc[(size_t)j * p.bc_dim + e] = y[i];
            }
          }
        }
      }
    }
    // next layer reads what this one wrote (the __syncthreads at the top of the
    // next k-loop orders the Y writes before the X reads)
    float* t = X; X = Y; Y = t;
    pbase = bbase + out;
  }

  // ---- cross-entropy: thread r < ROWS reduces row r of the logits (now in X) in column order
  if constexpr (XENT) {
    __syncthreads();
    const int C = p.desc.dims[L];
    const int b = b0 + (tid % BC);
    if (tid < ROWS && b < p.B) {
      const float* t = p.target + (size_t)b * C;
      float m = -INFINITY;
      for (int c = 0; c < C; ++c) m = fmaxf(m, X[(size_t)c * ROWS + tid]);
      float s = 0.f, st = 0.f, sty = 0.f;
      for (int c = 0; c < C; ++c) {
        const float y = X[(size_t)c * ROWS + tid], tv = __ldg(t + c);
        s += expf(y - m);
        st += tv;
        sty = fmaf(tv, y, sty);
      }
      loss = fmaf(m + logf(s), st, -sty);
    }
  }
  // ---- accuracy: thread r < ROWS compares the first argmax of row r of the logits with its target's
  if constexpr (ACC) {
    __syncthreads();
    const int C = p.desc.dims[L];
    const int b = b0 + (tid % BC);
    if (tid < ROWS && b < p.B) {
      const float* t = p.target + (size_t)b * C;
      float ym = -INFINITY, tm = -INFINITY;
      int yi = INT_MAX, ti = INT_MAX;
      for (int c = 0; c < C; ++c) {
        estk_argmax_fold(ym, yi, X[(size_t)c * ROWS + tid], c);
        estk_argmax_fold(tm, ti, __ldg(t + c), c);
      }
      loss = yi == ti ? 1.f : 0.f;
    }
  }

  // ---- block reduction of the loss, per sign
  {
    const bool lminus = (XENT || ACC) ? tid >= BC : minus;   // cross-entropy, accuracy: the sign of row tid
    const float lp = warp_sum_f(lminus ? 0.f : loss);
    const float lm = warp_sum_f(lminus ? loss : 0.f);
    if ((tid & 31) == 0) { s_red[0][tid >> 5] = lp; s_red[1][tid >> 5] = lm; }
    __syncthreads();
    if (tid == 0) {
      float sp = 0.f, sm = 0.f;
      for (int w = 0; w < kThreads / 32; ++w) { sp += s_red[0][w]; sm += s_red[1][w]; }
      float* part = p.partial + ((size_t)slot * 2) * p.chunks;
      part[chunk] = sp;
      part[p.chunks + chunk] = sm;
      __threadfence();
      s_last = estk_pair_arrive(p.counters + slot, p.chunks);
    }
    __syncthreads();
    if (s_last && tid == 0)
      ESTK_PAIR_FINISH(p.partial + ((size_t)slot * 2) * p.chunks, p.chunks,
                       ACC ? -(float)p.B : XENT ? (float)p.B : (float)p.B * (float)p.desc.dims[L], p.ret_plus,
                       p.ret_minus, j, p.counters + slot);
  }
}

size_t smem_bytes(int rows, int maxw) {
  const int ot = 4096 / rows;
  return sizeof(float) * ((size_t)2 * maxw * rows + (size_t)2 * KT * (ot + 4));
}

template <int ROWS, int ACT>
int launch_act(const EvalParams& p, size_t smem, cudaStream_t stream) {
  ESTK_CUDA(cudaFuncSetAttribute(eval_mlp_kernel<ROWS, ACT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  eval_mlp_kernel<ROWS, ACT><<<p.pairs * p.chunks, kThreads, smem, stream>>>(p);
  ESTK_CUDA(cudaGetLastError());
  return ESTK_OK;
}

template <int ROWS>
int launch(const EvalParams& p, size_t smem, cudaStream_t stream) {
  switch (p.desc.activation) {
    case ESTK_ACT_TANH: return launch_act<ROWS, ESTK_ACT_TANH>(p, smem, stream);
    case ESTK_ACT_OUT_TANH: return launch_act<ROWS, ESTK_ACT_OUT_TANH>(p, smem, stream);
    case ESTK_ACT_TANH | ESTK_ACT_OUT_TANH: return launch_act<ROWS, ESTK_ACT_TANH | ESTK_ACT_OUT_TANH>(p, smem, stream);
    case ESTK_LOSS_XENT: return launch_act<ROWS, ESTK_LOSS_XENT>(p, smem, stream);
    case ESTK_LOSS_XENT | ESTK_ACT_TANH: return launch_act<ROWS, ESTK_LOSS_XENT | ESTK_ACT_TANH>(p, smem, stream);
    case ESTK_ACT_ELU: return launch_act<ROWS, ESTK_ACT_ELU>(p, smem, stream);
    case ESTK_ACT_ELU | ESTK_ACT_OUT_TANH: return launch_act<ROWS, ESTK_ACT_ELU | ESTK_ACT_OUT_TANH>(p, smem, stream);
    case ESTK_ACT_ELU | ESTK_LOSS_XENT: return launch_act<ROWS, ESTK_ACT_ELU | ESTK_LOSS_XENT>(p, smem, stream);
    case ESTK_ACT_SILU: return launch_act<ROWS, ESTK_ACT_SILU>(p, smem, stream);
    case ESTK_ACT_SILU | ESTK_ACT_OUT_TANH: return launch_act<ROWS, ESTK_ACT_SILU | ESTK_ACT_OUT_TANH>(p, smem, stream);
    case ESTK_ACT_SILU | ESTK_LOSS_XENT: return launch_act<ROWS, ESTK_ACT_SILU | ESTK_LOSS_XENT>(p, smem, stream);
    case ESTK_ACT_LEAKY_RELU: return launch_act<ROWS, ESTK_ACT_LEAKY_RELU>(p, smem, stream);
    case ESTK_ACT_LEAKY_RELU | ESTK_ACT_OUT_TANH: return launch_act<ROWS, ESTK_ACT_LEAKY_RELU | ESTK_ACT_OUT_TANH>(p, smem, stream);
    case ESTK_ACT_LEAKY_RELU | ESTK_LOSS_XENT: return launch_act<ROWS, ESTK_ACT_LEAKY_RELU | ESTK_LOSS_XENT>(p, smem, stream);
    case ESTK_LOSS_ACCURACY: return launch_act<ROWS, ESTK_LOSS_ACCURACY>(p, smem, stream);
    case ESTK_ACT_TANH | ESTK_LOSS_ACCURACY: return launch_act<ROWS, ESTK_ACT_TANH | ESTK_LOSS_ACCURACY>(p, smem, stream);
    case ESTK_ACT_ELU | ESTK_LOSS_ACCURACY: return launch_act<ROWS, ESTK_ACT_ELU | ESTK_LOSS_ACCURACY>(p, smem, stream);
    case ESTK_ACT_SILU | ESTK_LOSS_ACCURACY: return launch_act<ROWS, ESTK_ACT_SILU | ESTK_LOSS_ACCURACY>(p, smem, stream);
    case ESTK_ACT_LEAKY_RELU | ESTK_LOSS_ACCURACY: return launch_act<ROWS, ESTK_ACT_LEAKY_RELU | ESTK_LOSS_ACCURACY>(p, smem, stream);
    default: return launch_act<ROWS, ESTK_ACT_RELU>(p, smem, stream);
  }
}

// ---------------------------------------------------------------- streamed kernel
// eval_mlp_wide_kernel: the shapes eval_mlp_kernel cannot hold -- a layer too wide for 16 rows of
// activations in shared memory, or a batch of more than kEvalMaxChunks chunks.  Persistent CTAs loop
// over work items (pair slot, chunk of kWideBC observations); both signs share one read of the noise row.
// Hidden activations (and the logits of the cross-entropy) live in a per-CTA slab in global memory,
// [width][kWideRows] per buffer, two buffers that alternate by layer; layer 0 reads obs directly.  Each
// layer is an N-tiled (kWideOT outputs), K-chunked (kWideKT) product: the X chunk is copied into shared
// memory with cp.async, W+ / W- are formed in shared memory from theta and the table (loaded into
// registers one chunk ahead), both double-buffered so one barrier per chunk separates the stages.
// Thread tile: 4 rows x 8 outputs.  The per-element arithmetic is eval_mlp_kernel's.
constexpr int kWideRows = 128;                               // 64 observations x 2 signs
constexpr int kWideBC = kWideRows / 2;
constexpr int kWideOT = 64;
constexpr int kWideOTP = kWideOT + 4;
constexpr int kWideKT = 32;
constexpr int kWideWPer = kWideOT * kWideKT / kThreads;      // weights each thread forms per chunk
constexpr size_t kWideSmem = sizeof(float) * (2 * kWideKT * kWideRows + 2 * 2 * kWideKT * kWideOTP);

__device__ __forceinline__ void cp_async4(float* dst, const float* src, bool full) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"((unsigned)__cvta_generic_to_shared(dst)),
               "l"(src), "r"(full ? 4 : 0) : "memory");
}
// L2 only: the slab is written by this CTA's threads, never through the read-only path
__device__ __forceinline__ void cp_async16(float* dst, const float* src, bool full) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"((unsigned)__cvta_generic_to_shared(dst)),
               "l"(src), "r"(full ? 16 : 0) : "memory");
}

// slab: [gridDim.x][2][slab_w][kWideRows]; p.partial [pairs][2][chunks]
template <int ACT>
__global__ void __launch_bounds__(kThreads, 1) eval_mlp_wide_kernel(const EvalParams p, float* const slab,
                                                                    const int slab_w) {
  constexpr int HID = ACT & 0xff;
  constexpr bool OUT_TANH = (ACT & ESTK_ACT_OUT_TANH) != 0;
  constexpr bool XENT = (ACT & ESTK_LOSS_XENT) != 0;
  constexpr bool ACC = (ACT & 0xff0000) == ESTK_LOSS_ACCURACY;
  constexpr int ROWS = kWideRows, BC = kWideBC, OT = kWideOT, OTP = kWideOTP, KT = kWideKT;
  extern __shared__ __align__(16) float smem[];
  float* const Xs = smem;                     // [2][KT][ROWS]; layer 0 fills the first BC rows only
  float* const Ws = Xs + 2 * KT * ROWS;       // [2][sign][KT][OTP]
  __shared__ float s_red[2][kThreads / 32];

  const int tid = threadIdx.x;
  const int tc = tid % 8, r0 = (tid / 8) * 4;    // outputs tc*4 + {0..3} and 32 + tc*4 + {0..3}
  const bool minus = r0 >= BC;                   // all 4 rows share the sign
  const bool centre = (p.offsets == nullptr);
  const float sigma = centre ? 0.f : p.sigma;
  const int L = p.desc.n_layers;
  float* const act0 = slab + (size_t)blockIdx.x * 2 * slab_w * ROWS;
  float* const act1 = act0 + (size_t)slab_w * ROWS;
  const int64_t items = (int64_t)p.pairs * p.chunks;

  for (int64_t item = blockIdx.x; item < items; item += gridDim.x) {
    const int slot = (int)(item / p.chunks);
    const int chunk = (int)(item % p.chunks);
    const int j = p.order ? p.order[slot] : slot;
    const NoiseRow nz{centre ? p.theta : p.table + p.offsets[j], nullptr};   // the fp32 table only
    const int b0 = chunk * BC;
    float loss = 0.f;
    int64_t pbase = 0;

    for (int l = 0; l < L; ++l) {
      const int in = p.desc.dims[l], out = p.desc.dims[l + 1];
      const int64_t wbase = pbase, bbase = pbase + (int64_t)in * out;
      const bool last = (l == L - 1);
      const float* xin = (l & 1) ? act0 : act1;     // layer l-1's output
      float* const yout = (l & 1) ? act1 : act0;
      const int xr = (l == 0 && minus) ? r0 - BC : r0;   // layer 0: one copy of the observations serves both signs
      const int nk = (in + KT - 1) / KT;
      for (int o0 = 0; o0 < out; o0 += OT) {
        float th[kWideWPer], tv[kWideWPer];
        // chunk kc of X -> Xs[kc & 1] (zero past `in` and past B), of theta / noise -> th, tv (zero outside)
        auto stage = [&](int kc) {
          const int k0 = kc * KT;
          float* dst = Xs + (kc & 1) * KT * ROWS;
          if (l == 0) {
            for (int e = tid; e < KT * BC; e += kThreads) {
              const int b = e % BC, k = e / BC;
              const bool ok = b0 + b < p.B && k0 + k < in;
              cp_async4(dst + k * ROWS + b, ok ? p.obs + (size_t)(b0 + b) * in + k0 + k : p.obs, ok);
            }
          } else {
            for (int e = tid; e < KT * ROWS / 4; e += kThreads) {
              const int k = e / (ROWS / 4), r = (e % (ROWS / 4)) * 4;
              const bool ok = k0 + k < in;
              cp_async16(dst + k * ROWS + r, ok ? xin + (size_t)(k0 + k) * ROWS + r : xin, ok);
            }
          }
          asm volatile("cp.async.commit_group;" ::: "memory");
#pragma unroll
          for (int i = 0; i < kWideWPer; ++i) {
            const int e = tid + i * kThreads, k = e % KT, o = e / KT;
            th[i] = tv[i] = 0.f;
            if (o0 + o < out && k0 + k < in) {
              const int64_t idx = wbase + (int64_t)(o0 + o) * in + k0 + k;
              th[i] = __ldg(p.theta + idx);
              tv[i] = nz(idx);
            }
          }
        };
        float acc[4][8];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int c = 0; c < 8; ++c) acc[i][c] = 0.f;
        __syncthreads();   // the previous tile's readers of Xs / Ws are done, the previous layer's slab written
        stage(0);
        for (int kc = 0; kc < nk; ++kc) {
          float* const Wb = Ws + (kc & 1) * 2 * KT * OTP;
#pragma unroll
          for (int i = 0; i < kWideWPer; ++i) {
            const int e = tid + i * kThreads, k = e % KT, o = e / KT;
            const float ep = __fmul_rn(sigma, tv[i]);
            Wb[k * OTP + o] = __fadd_rn(th[i], ep);
            Wb[KT * OTP + k * OTP + o] = __fsub_rn(th[i], ep);
          }
          asm volatile("cp.async.wait_all;" ::: "memory");
          __syncthreads();   // chunk kc staged and formed; chunk kc-1 consumed by every thread
          if (kc + 1 < nk) stage(kc + 1);
          const float* X = Xs + (kc & 1) * KT * ROWS + xr;
          const float* W = Wb + (minus ? KT * OTP : 0) + tc * 4;
#pragma unroll 8
          for (int k = 0; k < KT; ++k) {
            const float4 x = *reinterpret_cast<const float4*>(X + k * ROWS);
            const float4 wa = *reinterpret_cast<const float4*>(W + k * OTP);
            const float4 wb = *reinterpret_cast<const float4*>(W + k * OTP + 32);
            const float xv[4] = {x.x, x.y, x.z, x.w};
            const float wv[8] = {wa.x, wa.y, wa.z, wa.w, wb.x, wb.y, wb.z, wb.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
              for (int c = 0; c < 8; ++c) acc[i][c] = fmaf(xv[i], wv[c], acc[i][c]);
          }
        }
        // ---- tile epilogue: as eval_mlp_kernel's, into the slab
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          const int o = o0 + (c >> 2) * 32 + tc * 4 + (c & 3);
          if (o >= out) continue;
          const float bias = estk_form_sign(p.theta, nz, sigma, bbase + o, minus);
          float y[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) y[i] = acc[i][c] + bias;
          if (!last) {
#pragma unroll
            for (int i = 0; i < 4; ++i) y[i] = estk_hidden_act<HID>(y[i]);
            *reinterpret_cast<float4*>(yout + (size_t)o * ROWS + r0) = make_float4(y[0], y[1], y[2], y[3]);
          } else if constexpr (XENT || ACC) {
            *reinterpret_cast<float4*>(yout + (size_t)o * ROWS + r0) = make_float4(y[0], y[1], y[2], y[3]);
            float* bc = minus ? p.bc_minus : p.bc_plus;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const int b = b0 + ((r0 + i) % BC);
              const int64_t e = (int64_t)b * out + o;
              if (bc && b < p.B && b < p.bc_obs && e < p.bc_dim) bc[(size_t)j * p.bc_dim + e] = y[i];
            }
          } else {
            if constexpr (OUT_TANH) {
#pragma unroll
              for (int i = 0; i < 4; ++i) y[i] = tanhf(y[i]);
            }
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const int b = b0 + ((r0 + i) % BC);
              if (b < p.B) {
                const float d = y[i] - __ldg(p.target + (size_t)b * out + o);
                loss = fmaf(d, d, loss);
                float* bc = minus ? p.bc_minus : p.bc_plus;
                const int64_t e = (int64_t)b * out + o;
                if (bc && b < p.bc_obs && e < p.bc_dim) bc[(size_t)j * p.bc_dim + e] = y[i];
              }
            }
          }
        }
      }
      pbase = bbase + out;
    }

    // ---- cross-entropy: thread r < ROWS reduces row r of the logits (in the slab) in column order
    if constexpr (XENT) {
      __syncthreads();
      const float* Y = ((L - 1) & 1) ? act1 : act0;
      const int C = p.desc.dims[L];
      const int b = b0 + (tid % BC);
      if (tid < ROWS && b < p.B) {
        const float* t = p.target + (size_t)b * C;
        float m = -INFINITY;
        for (int c = 0; c < C; ++c) m = fmaxf(m, __ldcg(Y + (size_t)c * ROWS + tid));
        float s = 0.f, st = 0.f, sty = 0.f;
        for (int c = 0; c < C; ++c) {
          const float y = __ldcg(Y + (size_t)c * ROWS + tid), tv = __ldg(t + c);
          s += expf(y - m);
          st += tv;
          sty = fmaf(tv, y, sty);
        }
        loss = fmaf(m + logf(s), st, -sty);
      }
    }
    // ---- accuracy: thread r < ROWS compares the first argmax of row r of the logits with its target's
    if constexpr (ACC) {
      __syncthreads();
      const float* Y = ((L - 1) & 1) ? act1 : act0;
      const int C = p.desc.dims[L];
      const int b = b0 + (tid % BC);
      if (tid < ROWS && b < p.B) {
        const float* t = p.target + (size_t)b * C;
        float ym = -INFINITY, tm = -INFINITY;
        int yi = INT_MAX, ti = INT_MAX;
        for (int c = 0; c < C; ++c) {
          estk_argmax_fold(ym, yi, __ldcg(Y + (size_t)c * ROWS + tid), c);
          estk_argmax_fold(tm, ti, __ldg(t + c), c);
        }
        loss = yi == ti ? 1.f : 0.f;
      }
    }

    // ---- block reduction of the loss per sign, chunk partials combined in chunk order by the last arrival
    const bool lminus = (XENT || ACC) ? tid >= BC : minus;
    const float lp = warp_sum_f(lminus ? 0.f : loss);
    const float lm = warp_sum_f(lminus ? loss : 0.f);
    if ((tid & 31) == 0) { s_red[0][tid >> 5] = lp; s_red[1][tid >> 5] = lm; }
    __syncthreads();
    if (tid == 0) {   // s_red is written again only after the next item's first barrier
      float sp = 0.f, sm = 0.f;
      for (int w = 0; w < kThreads / 32; ++w) { sp += s_red[0][w]; sm += s_red[1][w]; }
      float* part = p.partial + (size_t)slot * 2 * p.chunks;
      part[chunk] = sp;
      part[p.chunks + chunk] = sm;
      __threadfence();
      if (estk_pair_arrive(p.counters + slot, p.chunks))
        ESTK_PAIR_FINISH(part, p.chunks, ACC ? -(float)p.B : XENT ? (float)p.B : (float)p.B * (float)p.desc.dims[L],
                         p.ret_plus, p.ret_minus, j, p.counters + slot);
    }
  }
}

using WideKernel = void (*)(const EvalParams, float*, int);

WideKernel wide_kernel(int act) {
  switch (act) {
    case ESTK_ACT_TANH: return eval_mlp_wide_kernel<ESTK_ACT_TANH>;
    case ESTK_ACT_OUT_TANH: return eval_mlp_wide_kernel<ESTK_ACT_OUT_TANH>;
    case ESTK_ACT_TANH | ESTK_ACT_OUT_TANH: return eval_mlp_wide_kernel<ESTK_ACT_TANH | ESTK_ACT_OUT_TANH>;
    case ESTK_LOSS_XENT: return eval_mlp_wide_kernel<ESTK_LOSS_XENT>;
    case ESTK_LOSS_XENT | ESTK_ACT_TANH: return eval_mlp_wide_kernel<ESTK_LOSS_XENT | ESTK_ACT_TANH>;
    case ESTK_ACT_ELU: return eval_mlp_wide_kernel<ESTK_ACT_ELU>;
    case ESTK_ACT_ELU | ESTK_ACT_OUT_TANH: return eval_mlp_wide_kernel<ESTK_ACT_ELU | ESTK_ACT_OUT_TANH>;
    case ESTK_ACT_ELU | ESTK_LOSS_XENT: return eval_mlp_wide_kernel<ESTK_ACT_ELU | ESTK_LOSS_XENT>;
    case ESTK_ACT_SILU: return eval_mlp_wide_kernel<ESTK_ACT_SILU>;
    case ESTK_ACT_SILU | ESTK_ACT_OUT_TANH: return eval_mlp_wide_kernel<ESTK_ACT_SILU | ESTK_ACT_OUT_TANH>;
    case ESTK_ACT_SILU | ESTK_LOSS_XENT: return eval_mlp_wide_kernel<ESTK_ACT_SILU | ESTK_LOSS_XENT>;
    case ESTK_ACT_LEAKY_RELU: return eval_mlp_wide_kernel<ESTK_ACT_LEAKY_RELU>;
    case ESTK_ACT_LEAKY_RELU | ESTK_ACT_OUT_TANH: return eval_mlp_wide_kernel<ESTK_ACT_LEAKY_RELU | ESTK_ACT_OUT_TANH>;
    case ESTK_ACT_LEAKY_RELU | ESTK_LOSS_XENT: return eval_mlp_wide_kernel<ESTK_ACT_LEAKY_RELU | ESTK_LOSS_XENT>;
    case ESTK_LOSS_ACCURACY: return eval_mlp_wide_kernel<ESTK_LOSS_ACCURACY>;
    case ESTK_ACT_TANH | ESTK_LOSS_ACCURACY: return eval_mlp_wide_kernel<ESTK_ACT_TANH | ESTK_LOSS_ACCURACY>;
    case ESTK_ACT_ELU | ESTK_LOSS_ACCURACY: return eval_mlp_wide_kernel<ESTK_ACT_ELU | ESTK_LOSS_ACCURACY>;
    case ESTK_ACT_SILU | ESTK_LOSS_ACCURACY: return eval_mlp_wide_kernel<ESTK_ACT_SILU | ESTK_LOSS_ACCURACY>;
    case ESTK_ACT_LEAKY_RELU | ESTK_LOSS_ACCURACY: return eval_mlp_wide_kernel<ESTK_ACT_LEAKY_RELU | ESTK_LOSS_ACCURACY>;
    default: return eval_mlp_wide_kernel<ESTK_ACT_RELU>;
  }
}

// The streamed kernel for a checked call: a persistent grid of at most (resident CTAs per SM) x SMs,
// each with its slab of 2 x (widest hidden layer, or the logits of the cross-entropy or the accuracy) x
// kWideRows floats.
int run_wide(estk_ctx* ctx, EvalParams& p, cudaStream_t stream, const char* who) {
  const estk_mlp_desc& d = p.desc;
  int slab_w = ((d.activation & ESTK_LOSS_XENT) || estk_loss_accuracy(d.activation)) ? d.dims[d.n_layers] : 0;
  for (int l = 1; l < d.n_layers; ++l) slab_w = max(slab_w, d.dims[l]);
  p.BC = kWideBC;
  p.chunks = (p.B + kWideBC - 1) / kWideBC;
  const int64_t items = (int64_t)p.pairs * p.chunks;
  const WideKernel kern = wide_kernel(d.activation);
  ESTK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kWideSmem));
  int per_sm = 0;
  ESTK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kThreads, kWideSmem));
  const int grid = (int)std::min<int64_t>(items, (int64_t)ctx->sm_count * std::max(per_sm, 1));
  const int rc = estk_ctx_reserve(ctx, p.pairs, items * 2, stream, who, (int64_t)grid * 2 * slab_w * kWideRows);
  if (rc) return rc;
  p.partial = ctx->eval_partial;
  p.counters = estk_member_counters(ctx);
  kern<<<grid, kThreads, kWideSmem, stream>>>(p, ctx->eval_slab, slab_w);
  ESTK_CUDA(cudaGetLastError());
  return ESTK_OK;
}

int run_eval(estk_ctx* ctx, EvalParams& p, cudaStream_t stream, const char* who) {
  const estk_mlp_desc& d = p.desc;
  ESTK_CHECK_ARG(d.n_layers >= 1 && d.n_layers <= ESTK_MAX_LAYERS, "%s: n_layers=%d", who, d.n_layers);
  ESTK_CHECK_ARG(estk_act_valid(d.activation), "%s: activation=0x%x is not a defined ESTK_ACT_* combination",
                 who, d.activation);
  int maxw = 0;
  for (int l = 0; l <= d.n_layers; ++l) {
    ESTK_CHECK_ARG(d.dims[l] >= 1, "%s: dims[%d]=%d", who, l, d.dims[l]);
    if (d.dims[l] > maxw) maxw = d.dims[l];
  }
  ESTK_CHECK_ARG(p.B >= 1, "%s: B must be positive", who);
  ESTK_CHECK_ARG(p.pairs >= 1 && p.pairs <= ESTK_MAX_POPULATION / 2, "%s: pairs=%d", who, p.pairs);
  p.maxw = maxw;
  // largest observation chunk whose activations fit in shared memory
  // (prefer <= 100 KB so two CTAs share an SM; wide layers may take up to 200 KB)
  size_t budget = 100 * 1024;
  if (smem_bytes(32, maxw) > budget) budget = 200 * 1024;
  int rows = 256;
  while (rows > 32 && (smem_bytes(rows, maxw) > budget || rows / 2 >= 2 * p.B)) rows >>= 1;
  // 16 rows (8 observations) only where 32 do not fit: input widths up to ~1500, e.g. 784 (28 x 28 images)
  if (smem_bytes(rows, maxw) > budget) rows = 16;
  // what does not fit in shared memory at 16 rows, or needs more than kEvalMaxChunks chunks, streams
  if (smem_bytes(rows, maxw) > budget) return run_wide(ctx, p, stream, who);
  p.BC = rows / 2;
  p.chunks = (p.B + p.BC - 1) / p.BC;
  if (p.chunks > kEvalMaxChunks) return run_wide(ctx, p, stream, who);
  const int rc = estk_ctx_reserve(ctx, p.pairs, (int64_t)p.pairs * 2 * p.chunks, stream, who);
  if (rc) return rc;
  p.partial = ctx->eval_partial;
  p.counters = estk_member_counters(ctx);
  const size_t smem = smem_bytes(rows, maxw);
  switch (rows) {
    case 256: return launch<256>(p, smem, stream);
    case 128: return launch<128>(p, smem, stream);
    case 64: return launch<64>(p, smem, stream);
    case 32: return launch<32>(p, smem, stream);
    default: return launch<16>(p, smem, stream);
  }
}

}  // namespace

// The one evaluate entry point of every policy kind and precision: the precision check, the call record, then
// the back end of the activation code.  The dense MLP evaluate is this function's own: its argument checks,
// then run_eval (fp32, here) or eval_mlp_tc (estk_eval_mlp_tc.cu).
extern "C" int estk_eval_mlp(estk_ctx* ctx, const estk_mlp_desc* desc, int32_t precision, const float* theta,
                             const uint16_t* theta16, const float* table, const uint16_t* table16,
                             const int64_t* offsets, const int32_t* order, int32_t pairs, float sigma,
                             const float* obs, const float* target, int32_t B, float* returns_plus,
                             float* returns_minus, float* bc_plus, float* bc_minus, int32_t bc_obs, int32_t bc_dim,
                             float* centre_return_out, void* stream) {
  const bool f16 = precision == ESTK_PREC_F16 || precision == ESTK_PREC_F16_ANY;
  const bool tc = f16 || precision == ESTK_PREC_BF16 || precision == ESTK_PREC_BF16S;
  const bool shadows = precision == ESTK_PREC_BF16S;                 // reads theta16, and table16 as a bf16 shadow
  const bool t16 = shadows || f16;                                   // a population reads table16
  const bool centre = offsets == nullptr;
  ESTK_CHECK_ARG(tc || precision == ESTK_PREC_FP32, "estk_eval_mlp: unknown precision %d", precision);
  EvalMlpCall c = {};
  if (desc) c.desc = *desc;
  c.precision = precision; c.theta = theta; c.theta16 = theta16; c.obs = obs; c.target = target; c.B = B;
  c.ret_plus = returns_plus; c.bc_plus = bc_plus; c.bc_obs = bc_obs; c.bc_dim = bc_dim;
  c.centre_out = centre_return_out;
  if (centre) {
    c.pairs = 1;
  } else {
    c.table = table; c.table16 = table16; c.offsets = offsets; c.order = order; c.pairs = pairs; c.sigma = sigma;
    c.ret_minus = returns_minus; c.bc_minus = bc_minus;
  }
  const cudaStream_t s = (cudaStream_t)stream;
  switch (desc ? estk_eval_route(desc->activation) : kRouteDense) {
    case kRouteCnn: return eval_cnn(ctx, c, s);
    case kRouteActions: return eval_mlp_actions(ctx, c, s);
    case kRouteActionsCell: return eval_rnn_actions(ctx, c, s);
    case kRouteSequence: return eval_rnn_sequence(ctx, c, s);
    case kRouteDense: break;
  }
  ESTK_CHECK_ARG(ctx && desc && theta && obs && target && returns_plus && (theta16 || !shadows) &&
                 (centre || (table && (table16 || !t16) && returns_minus)), "estk_eval_mlp: null argument");
  ESTK_CHECK_ARG(centre || (bc_plus == nullptr) == (bc_minus == nullptr),
                 "estk_eval_mlp: bc_plus/bc_minus must both be set or both null");
  ESTK_CHECK_ARG(!bc_plus || (bc_obs > 0 && bc_dim > 0), "estk_eval_mlp: bc_obs/bc_dim must be positive with bc outputs");
  ESTK_CHECK_ARG(!centre_return_out || !centre, "estk_eval_mlp: centre_return_out needs a population (offsets)");
  ESTK_CHECK_ARG(!estk_loss_accuracy(desc->activation) || B <= kAccuracyMaxB,
                 "estk_eval_mlp: B=%d: the accuracy's count is exact in fp32 for B < 2^24 only", B);
  ESTK_CHECK_ARG(!tc || (ESTK_ALIGNED16(theta) && ESTK_ALIGNED16(obs) && ESTK_ALIGNED16(target) &&
                         (!shadows || ESTK_ALIGNED16(theta16)) &&
                         (centre || (ESTK_ALIGNED16(table) && (!t16 || ESTK_ALIGNED16(table16))))),
                 "estk_eval_mlp: tensor-core buffers must be 16-byte aligned");
  if (centre_return_out && !tc) {
    estk_set_error("estk_eval_mlp: centre_return_out (folded centre rollout) needs a tensor-core precision");
    return ESTK_ERR_UNSUPPORTED;
  }
  c.theta16 = shadows ? theta16 : nullptr;
  if (centre) {
    c.table = theta; c.table16 = c.theta16;
  } else if (!t16) {
    c.table16 = nullptr;
  }
  if (tc) return eval_mlp_tc(ctx, c, s);
  EvalParams p = {};
  p.desc = c.desc; p.theta = c.theta; p.table = c.table; p.offsets = c.offsets; p.order = c.order;
  p.pairs = c.pairs; p.sigma = c.sigma; p.obs = c.obs; p.target = c.target; p.B = c.B;
  p.ret_plus = c.ret_plus; p.ret_minus = c.ret_minus;
  p.bc_plus = c.bc_plus; p.bc_minus = c.bc_minus; p.bc_obs = c.bc_obs; p.bc_dim = c.bc_dim;
  return run_eval(ctx, p, s, "estk_eval_mlp");
}
