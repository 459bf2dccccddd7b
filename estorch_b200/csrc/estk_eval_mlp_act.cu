// estk_eval_mlp_act.cu -- estk_eval_mlp with ESTK_ACTIONS (fp32): every perturbed policy's outputs on
// that member's own observations, the per-step operation of an environment population.
//
// Replaces (reference file:line):
//   ES._calculate_returns    estorch/estorch.py:195-202   vector_to_parameters + rollout per row: here the
//                            rollout stays user code, and each environment step asks for all members'
//                            actions at once (estorch_b200.PopulationAgent)
//   Policy.forward           examples/cartpole_es.py:14-20, one observation (or a few) per member
//
// One CTA = one antithetic pair x one chunk of BC observations per member (B <= 8 is one chunk: the
// case of one environment per member).  The pair's noise row is read once and serves both signs: each
// weight tile is formed in shared memory as W+ = theta + sigma*t and W- = theta - sigma*t, exactly as
// eval_mlp_kernel forms it, and multiplied into the + member's rows and the - member's rows.  Rows are
// 2*BC (sign-major), so a B = 1 step uses 2 rows instead of the 32 that eval_mlp_kernel's smallest
// row tile computes.  Thread = one output column x NB rows of one sign; one fmaf chain per (row,
// output) from 0 in ascending k, + bias, then estk_hidden_act<H> (SiLU with its call-free divide, the same
// bits; tanhf for the output): the bits of
// the fp32 evaluate kernels' behaviour characteristic.
//
// Activations ([width][ROWS], k-major) stay in shared memory when two layers of them fit in the
// budget below; otherwise they live in a per-CTA slab of the context workspace and a persistent grid
// loops over the work items (the same code, global instead of shared addresses).
//
// Algorithmic bytes per launch = 4*n*pairs (noise rows; 2*n*pairs from table16) + 4*n (theta)
// + 4*P*B*(in+out) (observations and outputs).
#include "estk_common.cuh"
#include <cuda_fp16.h>
#include <algorithm>
#include <climits>

namespace {

constexpr int kThreads = 256;
constexpr int KT = 32;                       // k-chunk of the weight tile
constexpr size_t kSmemBudget = 96 * 1024;    // activations + tiles; above it the activations stream

// row groups per CTA: 2 (one per sign) for a single row per sign, else 4
__host__ __device__ constexpr int act_groups(int bc) { return bc == 1 ? 2 : 4; }
__host__ __device__ constexpr int act_ot(int bc) { return kThreads / act_groups(bc); }   // outputs per tile

struct ActParams {
  estk_mlp_desc desc;
  const float* theta;
  const float* table;
  const uint16_t* table16;   // non-null: read instead of table (its exact fp16 copy)
  const int64_t* offsets;    // null => centre (theta, sigma ignored, no - member)
  const int32_t* order;
  int pairs;
  float sigma;
  const float* obs;          // population [2*pairs][B][in], centre [B][in]
  int B, chunks, maxw;
  float* bc_plus;
  float* bc_minus;
  int bc_obs, bc_dim;
  float* slab;               // SLAB: [gridDim.x][2][maxw][ROWS]
};

__device__ __forceinline__ float ld_noise1h(const uint16_t* p) {
  unsigned short v;
  asm volatile("ld.global.nc.L1::no_allocate.u16 %0, [%1];" : "=h"(v) : "l"(p));
  return __half2float(__ushort_as_half(v));
}

template <int BC, int ACT, bool SLAB>
__global__ void __launch_bounds__(kThreads, 4) eval_mlp_act_kernel(const ActParams p) {
  constexpr int HID = ACT & 0xff;
  constexpr bool OUT_TANH = (ACT & ESTK_ACT_OUT_TANH) != 0;
  constexpr int ROWS = 2 * BC;
  constexpr int G = act_groups(BC), OT = act_ot(BC), OTP = OT + 1;   // +1: conflict-free tile stores
  constexpr int RSTEP = G / 2;                                       // row groups per sign
  constexpr int NB = (BC + RSTEP - 1) / RSTEP;                       // rows per thread
  extern __shared__ __align__(16) float smem[];
  float* const Wp = smem;                     // [KT][OTP]
  float* const Wm = Wp + KT * OTP;            // [KT][OTP]
  float* const act0 = SLAB ? p.slab + (size_t)blockIdx.x * 2 * p.maxw * ROWS : Wm + KT * OTP;
  float* const act1 = act0 + (size_t)p.maxw * ROWS;

  const int tid = threadIdx.x;
  const int c = tid % OT, q = tid / OT;
  const bool minus = (q & 1) != 0;
  const int bsub = q >> 1;                    // this thread's rows: b = bsub + RSTEP*i, row = minus*BC + b
  const float* const Wsel = minus ? Wm : Wp;
  const bool centre = (p.offsets == nullptr);
  const float sigma = centre ? 0.f : p.sigma;
  const int L = p.desc.n_layers;
  const int in0 = p.desc.dims[0];

  // work items (slot, chunk), slot-major, strided by the grid; 32-bit index arithmetic (a 64-bit divide
  // is a subroutine call, and its call site made ptxas spill)
  unsigned int slot = blockIdx.x / (unsigned)p.chunks, chunk = blockIdx.x % (unsigned)p.chunks;
  for (; slot < (unsigned)p.pairs; chunk += gridDim.x, slot += chunk / p.chunks, chunk %= p.chunks) {
    const int j = p.order ? p.order[slot] : (int)slot;
    const int64_t toff = centre ? 0 : p.offsets[j];
    const float* const trow = centre ? p.theta : p.table + toff;
    const uint16_t* const trow16 = (centre || !p.table16) ? nullptr : p.table16 + toff;
    const int b0 = chunk * BC;
    float* X = act0;
    float* Y = act1;

    __syncthreads();   // the previous item's readers of X / Y are done
    // ---- stage each member's own observations: X[k][s*BC + b] = obs[member_s][b0+b][k]
    for (int idx = tid; idx < ROWS * in0; idx += kThreads) {
      const int r = idx / in0, k = idx % in0;
      const int s = r / BC, b = r % BC;
      const bool ok = b0 + b < p.B && !(centre && s);
      const int64_t member = s ? (int64_t)p.pairs + j : j;
      X[k * ROWS + r] = ok ? __ldg(p.obs + ((size_t)member * p.B + b0 + b) * in0 + k) : 0.f;
    }

    int64_t pbase = 0;
    for (int l = 0; l < L; ++l) {
      const int in = p.desc.dims[l], out = p.desc.dims[l + 1];
      const int64_t wbase = pbase, bbase = pbase + (int64_t)in * out;
      const bool last = (l == L - 1);
      for (int o0 = 0; o0 < out; o0 += OT) {
        float acc[NB];
#pragma unroll
        for (int i = 0; i < NB; ++i) acc[i] = 0.f;
        for (int k0 = 0; k0 < in; k0 += KT) {
          __syncthreads();  // previous tile consumed (and X staged / written on the first pass)
          // weight tile: element (o, k) <- theta/noise[wbase + (o0+o)*in + k0+k], as eval_mlp_kernel
          for (int e = tid; e < OT * KT; e += kThreads) {
            const int k = e % KT, o = e / KT;
            float wp = 0.f, wm = 0.f;
            if (o0 + o < out && k0 + k < in) {
              const int64_t idx = wbase + (int64_t)(o0 + o) * in + k0 + k;
              const float th = __ldg(p.theta + idx);
              const float t = trow16 ? ld_noise1h(trow16 + idx) : ld_noise1(trow + idx);
              const float ep = __fmul_rn(sigma, t);
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
            const float w = Wsel[k * OTP + c];
            const float* xk = X + (size_t)(k0 + k) * ROWS + (minus ? BC : 0) + bsub;
#pragma unroll
            for (int i = 0; i < NB; ++i)
              if (bsub + RSTEP * i < BC) acc[i] = fmaf(xk[RSTEP * i], w, acc[i]);
          }
        }
        // ---- tile epilogue: bias (+-), hidden activation into Y, or the output activation into bc
        const int o = o0 + c;
        if (o < out) {
          const float th = __ldg(p.theta + bbase + o);
          const float t = trow16 ? ld_noise1h(trow16 + bbase + o) : ld_noise1(trow + bbase + o);
          const float ep = __fmul_rn(sigma, t);
          const float bias = minus ? __fsub_rn(th, ep) : __fadd_rn(th, ep);
          float* const bc = minus ? p.bc_minus : p.bc_plus;
#pragma unroll
          for (int i = 0; i < NB; ++i) {
            const int bl = bsub + RSTEP * i;
            if (bl >= BC) continue;
            float y = acc[i] + bias;
            if (!last) {
              Y[(size_t)o * ROWS + (minus ? BC : 0) + bl] = estk_hidden_act<HID, true>(y);
            } else {
              if constexpr (OUT_TANH) y = tanhf(y);
              const int b = b0 + bl;
              const int64_t e = (int64_t)b * out + o;
              if (!(centre && minus) && b < p.B && b < p.bc_obs && e < p.bc_dim)
                bc[(size_t)j * p.bc_dim + e] = y;
            }
          }
        }
      }
      // the next layer reads what this one wrote (ordered by the __syncthreads at the top of its k-loop)
      float* t = X; X = Y; Y = t;
      pbase = bbase + out;
    }
  }
}

size_t tile_bytes(int bc) { return sizeof(float) * 2 * KT * (act_ot(bc) + 1); }
size_t act_bytes(int bc, int maxw) { return sizeof(float) * 2 * (size_t)maxw * 2 * bc; }

template <int BC, int ACT>
int launch_act(estk_ctx* ctx, ActParams& p, cudaStream_t stream, const char* who) {
  const int64_t items = (int64_t)p.pairs * p.chunks;
  const size_t smem_all = tile_bytes(BC) + act_bytes(BC, p.maxw);
  if (smem_all <= kSmemBudget) {
    auto kern = eval_mlp_act_kernel<BC, ACT, false>;
    ESTK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_all));
    const int grid = (int)std::min<int64_t>(items, INT_MAX);
    kern<<<grid, kThreads, smem_all, stream>>>(p);
  } else {
    auto kern = eval_mlp_act_kernel<BC, ACT, true>;
    const size_t smem = tile_bytes(BC);
    ESTK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    ESTK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kThreads, smem));
    const int grid = (int)std::min<int64_t>(items, (int64_t)ctx->sm_count * std::max(per_sm, 1));
    const int rc = estk_ctx_reserve(ctx, 0, 0, stream, who, (int64_t)grid * 2 * p.maxw * 2 * BC);
    if (rc) return rc;
    p.slab = ctx->eval_slab;
    kern<<<grid, kThreads, smem, stream>>>(p);
  }
  ESTK_CUDA(cudaGetLastError());
  return ESTK_OK;
}

template <int BC>
int launch_bc(estk_ctx* ctx, ActParams& p, cudaStream_t stream, const char* who) {
  switch (p.desc.activation & 0xffff) {   // the loss field is ESTK_ACTIONS here
    case ESTK_ACT_TANH: return launch_act<BC, ESTK_ACT_TANH>(ctx, p, stream, who);
    case ESTK_ACT_ELU: return launch_act<BC, ESTK_ACT_ELU>(ctx, p, stream, who);
    case ESTK_ACT_SILU: return launch_act<BC, ESTK_ACT_SILU>(ctx, p, stream, who);
    case ESTK_ACT_LEAKY_RELU: return launch_act<BC, ESTK_ACT_LEAKY_RELU>(ctx, p, stream, who);
    case ESTK_ACT_OUT_TANH: return launch_act<BC, ESTK_ACT_OUT_TANH>(ctx, p, stream, who);
    case ESTK_ACT_TANH | ESTK_ACT_OUT_TANH: return launch_act<BC, ESTK_ACT_TANH | ESTK_ACT_OUT_TANH>(ctx, p, stream, who);
    case ESTK_ACT_ELU | ESTK_ACT_OUT_TANH: return launch_act<BC, ESTK_ACT_ELU | ESTK_ACT_OUT_TANH>(ctx, p, stream, who);
    case ESTK_ACT_SILU | ESTK_ACT_OUT_TANH: return launch_act<BC, ESTK_ACT_SILU | ESTK_ACT_OUT_TANH>(ctx, p, stream, who);
    case ESTK_ACT_LEAKY_RELU | ESTK_ACT_OUT_TANH:
      return launch_act<BC, ESTK_ACT_LEAKY_RELU | ESTK_ACT_OUT_TANH>(ctx, p, stream, who);
    default: return launch_act<BC, ESTK_ACT_RELU>(ctx, p, stream, who);
  }
}

}  // namespace

int eval_mlp_actions(estk_ctx* ctx, const estk_mlp_desc* desc, int precision, const float* theta,
                     const float* table, const uint16_t* table16, const int64_t* offsets, const int32_t* order,
                     int pairs, float sigma, const float* obs, int B, float* bc_plus, float* bc_minus, int bc_obs,
                     int bc_dim, const float* centre_return_out, cudaStream_t stream) {
  const char* who = "estk_eval_mlp[ESTK_ACTIONS]";
  const bool centre = offsets == nullptr;
  ESTK_CHECK_ARG(precision == ESTK_PREC_FP32 || precision == ESTK_PREC_F16 || precision == ESTK_PREC_BF16 ||
                 precision == ESTK_PREC_BF16S || precision == ESTK_PREC_F16_ANY, "%s: unknown precision %d", who,
                 precision);
  if (precision != ESTK_PREC_FP32) {
    estk_set_error("%s: actions are computed with ESTK_PREC_FP32 only (precision %d)", who, precision);
    return ESTK_ERR_UNSUPPORTED;
  }
  ESTK_CHECK_ARG(ctx && theta && obs && bc_plus && (centre || ((table || table16) && bc_minus)),
                 "%s: null argument (theta, obs, bc_plus, and for a population table or table16 and bc_minus)", who);
  ESTK_CHECK_ARG(bc_obs > 0 && bc_dim > 0, "%s: bc_obs/bc_dim must be positive", who);
  ESTK_CHECK_ARG(!centre_return_out, "%s: centre_return_out is not an ESTK_ACTIONS output", who);
  const estk_mlp_desc& d = *desc;
  ESTK_CHECK_ARG(d.n_layers >= 1 && d.n_layers <= ESTK_MAX_LAYERS, "%s: n_layers=%d", who, d.n_layers);
  int maxw = 0;
  for (int l = 0; l <= d.n_layers; ++l) {
    ESTK_CHECK_ARG(d.dims[l] >= 1, "%s: dims[%d]=%d", who, l, d.dims[l]);
    maxw = std::max(maxw, d.dims[l]);
  }
  ESTK_CHECK_ARG(B >= 1, "%s: B must be positive", who);
  ESTK_CHECK_ARG(centre || (pairs >= 1 && pairs <= ESTK_MAX_POPULATION / 2), "%s: pairs=%d", who, pairs);
  ActParams p = {};
  p.desc = d; p.theta = theta; p.offsets = offsets; p.obs = obs; p.B = B; p.maxw = maxw;
  p.bc_plus = bc_plus; p.bc_obs = bc_obs; p.bc_dim = bc_dim;
  if (centre) {
    p.pairs = 1;
  } else {
    p.table = table; p.table16 = table16; p.order = order; p.pairs = pairs; p.sigma = sigma; p.bc_minus = bc_minus;
  }
  const int bc = B <= 1 ? 1 : B <= 2 ? 2 : B <= 4 ? 4 : 8;
  p.chunks = (B + bc - 1) / bc;
  switch (bc) {
    case 1: return launch_bc<1>(ctx, p, stream, who);
    case 2: return launch_bc<2>(ctx, p, stream, who);
    case 4: return launch_bc<4>(ctx, p, stream, who);
    default: return launch_bc<8>(ctx, p, stream, who);
  }
}
