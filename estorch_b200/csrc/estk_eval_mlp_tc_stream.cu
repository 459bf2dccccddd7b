// estk_eval_mlp_tc_stream.cu -- the F16 arithmetic of the tensor-core evaluate (estk_eval_mlp_tc.cu)
// for every MLP shape: ESTK_PREC_F16_ANY where the cluster kernel's shape rule does not hold (any
// widths, any B).
//
// eval_mlp_tc_stream_kernel: persistent CTAs loop over items (pair slot, chunk of 64 observations), the
// structure of eval_mlp_wide_kernel (estk_eval_mlp.cu) with the operands of eval_mlp_tc_kernel.
//   warpgroup 0 evaluates W+ = theta + sigma*eps, warpgroup 1 W- = theta - sigma*eps; every thread forms
//   its share of both from ONE read of theta and the noise row.
//   Per layer, N tiles of 128 outputs, k-blocks of 64 in ascending order (layer 0: the x_hi k-block then
//   the x_lo k-block on the same weight tile, as the cluster kernel orders them), so every pre-activation
//   accumulator is the same wgmma m64n128k16 chain of the same operands as the cluster kernel's.
//   A: 64 rows x 64 fp16, 128B-swizzled, copied per k-block into shared memory with cp.async from
//      - layer 0: the observations, split into hi / lo halves once per call (split_obs_f16_kernel) into
//        the same tile image, rows past B and columns past dims[0] zero;
//      - layer l > 0: the CTA's slab in the context workspace, where layer l-1's epilogue stored its
//        fp16 activations in that tile image (one buffer per sign, two that alternate by layer).
//   B: [128 x 64] fp16 per sign, formed in shared memory: W16 = rn_f16(theta + s*sigma*eps) in fp32 from
//      the fp32 theta and the exact fp16 table16; zero past K and past N.
//   K padding meets zero weights and zero (finite) activations; padded output columns compute 0 + 0
//   (their bias is zero) and are never scored or stored as behaviour characteristics.
//   Two stages: while the MMAs of k-block kb run, the threads form k-block kb+1 from registers loaded one
//   k-block ahead; one CTA barrier per k-block.
//   Epilogue as the cluster kernel's: bias, ReLU / tanhf rounded once to fp16 (satfinite); the last layer
//   the output tanhf, squared error or the cross-entropy chain (running max, sum of exponentials,
//   sum t*y, sum t per row, carried across N tiles, then over the four lanes of a quad), and the
//   behaviour characteristic.  Rows past B are masked out.  Chunk partials are combined in chunk order
//   by the last arrival (no float atomics: the same bits from run to run, with or without `order`).
#include "estk_tc.cuh"
#include <algorithm>
#include <type_traits>

namespace {

constexpr int kRowsS = 64;                              // observations per item (wgmma M)
constexpr int kTileNS = 128;                            // outputs per N tile (wgmma N)
constexpr int kThreadsS = 256;                          // warpgroup 0: sign +, warpgroup 1: sign -
constexpr int kABytes = kRowsS * kBlockK * 2;           // one [64 x 64] fp16 k-block of activations: 8 KB
constexpr int kBBytes = kTileNS * kBlockK * 2;          // one [128 x 64] fp16 weight k-block: 16 KB
constexpr int kStageBytesS = 2 * kABytes + 2 * kBBytes; // A (two signs, or layer 0's hi / lo) + B (two signs)
constexpr int kPairsPT = kTileNS * kBlockK / 2 / kThreadsS;   // weight pairs (per sign) a thread forms: 16
constexpr size_t kSmemS = 1024 + 2 * (size_t)kStageBytesS + 2 * kTileNS * sizeof(float);

struct StreamParams {
  estk_mlp_desc desc;
  const float* theta;
  const float* table;       // fp32 table: the biases
  const uint16_t* table16;  // exact fp16 copy: the weights (null for the centre evaluation)
  const int64_t* offsets;   // null => centre evaluation
  const int32_t* order;
  int pairs;
  float sigma;
  const float* target;
  int B, chunks;            // chunks of kRowsS observations
  float* ret_plus;
  float* ret_minus;
  float* bc_plus;
  float* bc_minus;
  int bc_obs, bc_dim;
  float* partial;           // [pairs][2][chunks]
  unsigned int* counters;   // [pairs]
  const uint8_t* xin;       // [chunks][kb0][hi, lo] 8 KB tile images of the observations
  uint8_t* slab;            // [gridDim.x][layer parity][sign][slab_kb] 8 KB tile images
  int kb0, slab_kb;
};

__device__ __forceinline__ uint16_t ld_noise_u16(const uint16_t* p) {
  uint16_t v;
  asm volatile("ld.global.nc.L1::no_allocate.u16 %0, [%1];" : "=h"(v) : "l"(p));
  return v;
}
// L2 only: the slab is written by this CTA's threads, never through the read-only path
__device__ __forceinline__ void cp_async16_smem(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}

// obs [B][K0] -> xin: per chunk of 64 rows and k-block of 64 columns the x_hi = rn_f16(x) and
// x_lo = rn_f16(x - x_hi) tiles, in the 128B-swizzled image the wgmma A descriptor reads
__global__ void __launch_bounds__(256) split_obs_f16_kernel(const float* __restrict__ obs, int B, int K0, int kb0,
                                                            int64_t n16, uint8_t* __restrict__ xin) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += stride) {
    const int c8 = (int)(i & 7), r = (int)((i >> 3) & (kRowsS - 1));
    const int64_t t = i >> 9;                      // chunk * kb0 + kb
    const int64_t b = (t / kb0) * kRowsS + r;
    const int k0 = (int)(t % kb0) * kBlockK + c8 * 8;
    float x[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) x[q] = (b < B && k0 + q < K0) ? __ldg(obs + b * K0 + k0 + q) : 0.f;
    uint32_t hi[4], lo[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      hi[q] = pack_f16(x[2 * q], x[2 * q + 1]);
      const float2 f = unpack_f16(hi[q]);
      lo[q] = pack_f16(x[2 * q] - f.x, x[2 * q + 1] - f.y);
    }
    uint8_t* tile = xin + t * 2 * kABytes + sw128_offset(r, c8);
    *reinterpret_cast<uint4*>(tile) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
    *reinterpret_cast<uint4*>(tile + kABytes) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
  }
}

// (m, s) <- the chain (m, s) merged with (om, os): max and rescaled sum of exponentials; an empty side
// (s == 0, m == -inf) contributes nothing
__device__ __forceinline__ void lse_merge(float& m, float& s, float om, float os) {
  const float nm = fmaxf(m, om);
  s = (s > 0.f ? s * expf(m - nm) : 0.f) + (os > 0.f ? os * expf(om - nm) : 0.f);
  m = nm;
}

template <int ACT>
__global__ void __launch_bounds__(kThreadsS, 1) eval_mlp_tc_stream_kernel(const StreamParams p) {
  constexpr int HID = ACT & 0xff;
  constexpr bool OUT_TANH = (ACT & ESTK_ACT_OUT_TANH) != 0;
  constexpr bool XENT = (ACT & ESTK_LOSS_XENT) != 0;
  constexpr bool ACC = (ACT & 0xff0000) == ESTK_LOSS_ACCURACY;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* sBias = reinterpret_cast<float*>(smem + 2 * kStageBytesS);   // [sign][kTileNS]
  __shared__ float s_red[2][4];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int sg = warp >> 2;                        // this warpgroup's sign
  const int r0 = (warp & 3) * 16 + (lane >> 2);    // accumulator rows r0 and r0 + 8
  const int cq = (lane & 3) * 2;                   // accumulator columns 8j + cq, +1
  const int fk = (tid & 31) * 2, fr = tid >> 5;    // forming: columns fk, fk+1 of rows fr + 8i
  const bool centre = (p.offsets == nullptr);
  const int L = p.desc.n_layers;
  uint8_t* const slab = p.slab + (size_t)blockIdx.x * 4 * p.slab_kb * kABytes;
  const int64_t items = (int64_t)p.pairs * p.chunks;
  const uint32_t smem0 = smem_u32(smem);

  for (int64_t item = blockIdx.x; item < items; item += gridDim.x) {
    const int slot = (int)(item / p.chunks);
    const int chunk = (int)(item % p.chunks);
    const int j = p.order ? p.order[slot] : slot;
    const float* trow = centre ? p.theta : p.table + p.offsets[j];
    const uint16_t* trow16 = centre ? nullptr : p.table16 + p.offsets[j];
    const float sig = centre ? 0.f : p.sigma;
    float* const bc = sg ? p.bc_minus : p.bc_plus;
    float loss = 0.f;
    float xm[2] = {-INFINITY, -INFINITY}, xs[2] = {0.f, 0.f}, xsty[2] = {0.f, 0.f}, xst[2] = {0.f, 0.f};
    // accuracy: per row h the (max, first index) of the logits over this thread's columns
    float am[2] = {-INFINITY, -INFINITY};
    int ai[2] = {INT_MAX, INT_MAX};
    int64_t wbase = 0;

    for (int l = 0; l < L; ++l) {
      const int K = p.desc.dims[l], N = p.desc.dims[l + 1];
      const int64_t bbase = wbase + (int64_t)K * N;
      const bool last = (l == L - 1);
      const int nk = (K + kBlockK - 1) / kBlockK;
      // k-block kb of A: two 8 KB pieces -- layer 0: x_hi, x_lo; else the + and - activations
      const uint8_t* a0 = l == 0 ? p.xin + (size_t)chunk * p.kb0 * 2 * kABytes
                                 : slab + (size_t)((l - 1) & 1) * 2 * p.slab_kb * kABytes;
      const size_t a_step = l == 0 ? 2 * kABytes : kABytes;
      const size_t a_second = l == 0 ? kABytes : (size_t)p.slab_kb * kABytes;
      uint8_t* const aout = slab + (size_t)(l & 1) * 2 * p.slab_kb * kABytes + (size_t)sg * p.slab_kb * kABytes;

      for (int n0 = 0; n0 < N; n0 += kTileNS) {
        float th[2 * kPairsPT];
        uint32_t ev[kPairsPT];             // two fp16 noise values per register
        const int rows = (N - n0 - fr + 7) / 8;    // this thread's forming rows inside the layer
        auto load = [&](int kb) {
          const int k = kb * kBlockK + fk;
          // opaque to the compiler: otherwise it keeps 2 x 16 row pointers live across the k loop (spills)
          int64_t base = wbase + (int64_t)(n0 + fr) * K + k;
          asm("" : "+l"(base));
          const float* tp = p.theta + base;
          const uint16_t* ep = trow16 + base;
#pragma unroll
          for (int i = 0; i < kPairsPT; ++i, tp += 8 * (int64_t)K, ep += 8 * (int64_t)K) {
            uint16_t e2[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const bool ok = i < rows && k + e < K;
              th[2 * i + e] = ok ? __ldg(tp + e) : 0.f;
              e2[e] = (ok && trow16) ? ld_noise_u16(ep + e) : (uint16_t)0;
            }
            ev[i] = (uint32_t)e2[0] | ((uint32_t)e2[1] << 16);
          }
        };
        auto stage_a = [&](int kb) {
          const uint32_t dst = smem0 + (kb & 1) * kStageBytesS;
          const uint8_t* src = a0 + kb * a_step;
#pragma unroll
          for (int u = 0; u < 2 * kABytes / 16 / kThreadsS; ++u) {
            const int c = tid + u * kThreadsS, piece = c / (kABytes / 16), off = (c % (kABytes / 16)) * 16;
            cp_async16_smem(dst + piece * kABytes + off, src + piece * a_second + off);
          }
          asm volatile("cp.async.commit_group;" ::: "memory");
        };
        // the previous tile's MMAs and epilogue (sBias, slab stores) are done in both warpgroups
        __syncthreads();
        {
          const int s = tid / kTileNS, o = tid % kTileNS;
          float bv = 0.f;
          if (n0 + o < N) bv = fmaf(s ? -sig : sig, ld_noise1(trow + bbase + n0 + o), __ldg(p.theta + bbase + n0 + o));
          sBias[tid] = bv;
        }
        load(0);
        stage_a(0);
        float d[64];                       // the first MMA of the tile overwrites (scale-d = 0)
        // NP = 2: layer 0, the x_hi then the x_lo k-block on the same weight tile (a separate
        // instantiation, so that no wgmma sits under a branch)
        auto k_loop = [&](auto np_tag) {
          constexpr int NP = decltype(np_tag)::value;
          for (int kb = 0; kb < nk; ++kb) {
            const uint32_t a_addr = smem0 + (kb & 1) * kStageBytesS, b_addr = a_addr + 2 * kABytes;
            // W+ / W- of k-block kb into stage kb & 1 (its readers, the MMAs of k-block kb-2, completed
            // before the barrier of k-block kb-1)
#pragma unroll
            for (int i = 0; i < kPairsPT; ++i) {
              const float2 e = unpack_f16(ev[i]);
              const uint32_t off = sw128_offset(fr + 8 * i, fk >> 3) + (fk & 7) * 2;
              st_shared_u32(b_addr + off, pack_f16(fmaf(sig, e.x, th[2 * i]), fmaf(sig, e.y, th[2 * i + 1])));
              st_shared_u32(b_addr + kBBytes + off, pack_f16(fmaf(-sig, e.x, th[2 * i]), fmaf(-sig, e.y, th[2 * i + 1])));
            }
            if (kb + 1 < nk) load(kb + 1);
            asm volatile("cp.async.wait_all;" ::: "memory");
            fence_proxy_async();             // the formed tile and the copied activations -> wgmma
            wgmma_wait<0>();                 // this warpgroup's MMAs of k-block kb-1 are done
            __syncthreads();
            if (kb + 1 < nk) stage_a(kb + 1);   // stage (kb+1) & 1: its MMAs (k-block kb-1) are done
            wgmma_fence();
#pragma unroll
            for (int pass = 0; pass < NP; ++pass) {
              const uint32_t a = a_addr + (NP == 2 ? pass : sg) * kABytes;
#pragma unroll
              for (int k = 0; k < kBlockK / 16; ++k)
                wgmma_m64n128k16<true>(d, make_sw128_desc(a + k * 32), make_sw128_desc(b_addr + sg * kBBytes + k * 32),
                                       (kb | k | pass) != 0 ? 1u : 0u);
            }
            wgmma_commit();
          }
        };
        if (l == 0) k_loop(std::integral_constant<int, 2>{});
        else k_loop(std::integral_constant<int, 1>{});
        wgmma_wait<0>();
        fence_acc(d);
        const float* bias = sBias + sg * kTileNS;
        // ---- epilogue of the tile
        if (!last) {
#pragma unroll
          for (int jb = 0; jb < kTileNS / 8; ++jb) {
            const int c = jb * 8 + cq, col = n0 + c;
            const float2 bv = *reinterpret_cast<const float2*>(bias + c);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int r = r0 + 8 * h;
              const float y0 = d[jb * 4 + 2 * h] + bv.x, y1 = d[jb * 4 + 2 * h + 1] + bv.y;
              *reinterpret_cast<uint32_t*>(aout + (size_t)(col >> 6) * kABytes + sw128_offset(r, (col & 63) >> 3) +
                                           (col & 7) * 2) =
                  HID == ESTK_ACT_RELU ? pack_f16_relu(y0, y1)
                                       : pack_f16(estk_hidden_act<HID>(y0), estk_hidden_act<HID>(y1));
            }
          }
        } else if constexpr (XENT) {
          float tm[2] = {-INFINITY, -INFINITY}, ts[2] = {0.f, 0.f};
#pragma unroll
          for (int jb = 0; jb < kTileNS / 8; ++jb) {
            const int c = jb * 8 + cq, col = n0 + c;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int b = chunk * kRowsS + r0 + 8 * h;
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                if (b < p.B && col + e < N) {
                  const float y = d[jb * 4 + 2 * h + e] + bias[c + e];
                  const float t = __ldg(p.target + (size_t)b * N + col + e);
                  d[jb * 4 + 2 * h + e] = y;
                  tm[h] = fmaxf(tm[h], y);
                  xsty[h] = fmaf(t, y, xsty[h]);
                  xst[h] += t;
                  const int64_t idx = (int64_t)b * N + col + e;
                  if (bc && b < p.bc_obs && idx < p.bc_dim) bc[(size_t)j * p.bc_dim + idx] = y;
                }
              }
            }
          }
#pragma unroll
          for (int jb = 0; jb < kTileNS / 8; ++jb)
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
              for (int e = 0; e < 2; ++e)
                if (chunk * kRowsS + r0 + 8 * h < p.B && n0 + jb * 8 + cq + e < N)
                  ts[h] += expf(d[jb * 4 + 2 * h + e] - tm[h]);
#pragma unroll
          for (int h = 0; h < 2; ++h) lse_merge(xm[h], xs[h], tm[h], ts[h]);
        } else if constexpr (ACC) {
#pragma unroll
          for (int jb = 0; jb < kTileNS / 8; ++jb) {
            const int c = jb * 8 + cq, col = n0 + c;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int b = chunk * kRowsS + r0 + 8 * h;
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                if (b < p.B && col + e < N) {
                  const float y = d[jb * 4 + 2 * h + e] + bias[c + e];
                  estk_argmax_fold(am[h], ai[h], y, col + e);
                  const int64_t idx = (int64_t)b * N + col + e;
                  if (bc && b < p.bc_obs && idx < p.bc_dim) bc[(size_t)j * p.bc_dim + idx] = y;
                }
              }
            }
          }
        } else {
#pragma unroll
          for (int jb = 0; jb < kTileNS / 8; ++jb) {
            const int c = jb * 8 + cq, col = n0 + c;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int b = chunk * kRowsS + r0 + 8 * h;
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                if (b < p.B && col + e < N) {
                  float y = d[jb * 4 + 2 * h + e] + bias[c + e];
                  if constexpr (OUT_TANH) y = tanhf(y);
                  const float df = y - __ldg(p.target + (size_t)b * N + col + e);
                  loss = fmaf(df, df, loss);
                  const int64_t idx = (int64_t)b * N + col + e;
                  if (bc && b < p.bc_obs && idx < p.bc_dim) bc[(size_t)j * p.bc_dim + idx] = y;
                }
              }
            }
            // one column block's targets at a time: all 64 in flight at once would spill
            asm volatile("" ::: "memory");
          }
        }
      }
      wbase = bbase + N;
    }

    if constexpr (XENT) {
      // the row's four lanes (the quad) hold disjoint columns: combine them, then ce once per row
#pragma unroll
      for (int o = 1; o <= 2; o <<= 1)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float om = __shfl_xor_sync(0xffffffffu, xm[h], o), os = __shfl_xor_sync(0xffffffffu, xs[h], o);
          xsty[h] += __shfl_xor_sync(0xffffffffu, xsty[h], o);
          xst[h] += __shfl_xor_sync(0xffffffffu, xst[h], o);
          lse_merge(xm[h], xs[h], om, os);
        }
#pragma unroll
      for (int h = 0; h < 2; ++h)
        if ((lane & 3) == 0 && chunk * kRowsS + r0 + 8 * h < p.B)
          loss += fmaf(xm[h] + logf(xs[h]), xst[h], -xsty[h]);
    }
    if constexpr (ACC) {
      // the quad's lanes hold disjoint columns of the row; the target's label is read here, once per row
      const int C = p.desc.dims[L];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int b = chunk * kRowsS + r0 + 8 * h;
        estk_argmax_quad(am[h], ai[h]);
        const int label = estk_quad_label(p.target + (size_t)b * C, b < p.B ? C : 0, lane & 3);
        if ((lane & 3) == 0 && b < p.B && ai[h] == label) loss += 1.f;
      }
    }

    // ---- loss of each sign over the chunk; the last arriving chunk combines the partials in chunk order
    loss = warp_sum_f(loss);
    if (lane == 0) s_red[sg][warp & 3] = loss;
    __syncthreads();
    if (tid == 0) {   // s_red is written again only after the next item's first barrier
      const float sp = (s_red[0][0] + s_red[0][1]) + (s_red[0][2] + s_red[0][3]);
      const float sm = (s_red[1][0] + s_red[1][1]) + (s_red[1][2] + s_red[1][3]);
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

using StreamKernel = void (*)(const StreamParams);

StreamKernel stream_kernel(int act) {
  switch (act) {
    case ESTK_ACT_TANH: return eval_mlp_tc_stream_kernel<ESTK_ACT_TANH>;
    case ESTK_ACT_OUT_TANH: return eval_mlp_tc_stream_kernel<ESTK_ACT_OUT_TANH>;
    case ESTK_ACT_TANH | ESTK_ACT_OUT_TANH: return eval_mlp_tc_stream_kernel<ESTK_ACT_TANH | ESTK_ACT_OUT_TANH>;
    case ESTK_LOSS_XENT: return eval_mlp_tc_stream_kernel<ESTK_LOSS_XENT>;
    case ESTK_LOSS_XENT | ESTK_ACT_TANH: return eval_mlp_tc_stream_kernel<ESTK_LOSS_XENT | ESTK_ACT_TANH>;
    case ESTK_ACT_ELU: return eval_mlp_tc_stream_kernel<ESTK_ACT_ELU>;
    case ESTK_ACT_ELU | ESTK_ACT_OUT_TANH: return eval_mlp_tc_stream_kernel<ESTK_ACT_ELU | ESTK_ACT_OUT_TANH>;
    case ESTK_ACT_ELU | ESTK_LOSS_XENT: return eval_mlp_tc_stream_kernel<ESTK_ACT_ELU | ESTK_LOSS_XENT>;
    case ESTK_ACT_SILU: return eval_mlp_tc_stream_kernel<ESTK_ACT_SILU>;
    case ESTK_ACT_SILU | ESTK_ACT_OUT_TANH: return eval_mlp_tc_stream_kernel<ESTK_ACT_SILU | ESTK_ACT_OUT_TANH>;
    case ESTK_ACT_SILU | ESTK_LOSS_XENT: return eval_mlp_tc_stream_kernel<ESTK_ACT_SILU | ESTK_LOSS_XENT>;
    case ESTK_ACT_LEAKY_RELU: return eval_mlp_tc_stream_kernel<ESTK_ACT_LEAKY_RELU>;
    case ESTK_ACT_LEAKY_RELU | ESTK_ACT_OUT_TANH: return eval_mlp_tc_stream_kernel<ESTK_ACT_LEAKY_RELU | ESTK_ACT_OUT_TANH>;
    case ESTK_ACT_LEAKY_RELU | ESTK_LOSS_XENT: return eval_mlp_tc_stream_kernel<ESTK_ACT_LEAKY_RELU | ESTK_LOSS_XENT>;
    case ESTK_LOSS_ACCURACY: return eval_mlp_tc_stream_kernel<ESTK_LOSS_ACCURACY>;
    case ESTK_ACT_TANH | ESTK_LOSS_ACCURACY: return eval_mlp_tc_stream_kernel<ESTK_ACT_TANH | ESTK_LOSS_ACCURACY>;
    case ESTK_ACT_ELU | ESTK_LOSS_ACCURACY: return eval_mlp_tc_stream_kernel<ESTK_ACT_ELU | ESTK_LOSS_ACCURACY>;
    case ESTK_ACT_SILU | ESTK_LOSS_ACCURACY: return eval_mlp_tc_stream_kernel<ESTK_ACT_SILU | ESTK_LOSS_ACCURACY>;
    case ESTK_ACT_LEAKY_RELU | ESTK_LOSS_ACCURACY: return eval_mlp_tc_stream_kernel<ESTK_ACT_LEAKY_RELU | ESTK_LOSS_ACCURACY>;
    default: return eval_mlp_tc_stream_kernel<ESTK_ACT_RELU>;
  }
}

}  // namespace

int eval_mlp_tc_stream_supported(const estk_mlp_desc& d, int B, const char** why) {
  if (d.n_layers < 1 || d.n_layers > ESTK_MAX_LAYERS) { *why = "n_layers"; return 0; }
  if (!estk_act_valid(d.activation)) { *why = "activation is not a defined ESTK_ACT_* combination"; return 0; }
  for (int l = 0; l <= d.n_layers; ++l)
    if (d.dims[l] < 1) { *why = "layer widths must be positive"; return 0; }
  if (B < 1) { *why = "batch must be positive"; return 0; }
  return 1;
}

// Two launches: the observations' hi / lo tiles, then the streamed kernel on a persistent grid of one
// CTA per SM.  Workspace (the context's slab): the observation tiles, then per CTA two layer buffers x
// two signs x the widest hidden layer, rounded up to whole N tiles (the epilogue stores whole tiles).
int eval_mlp_tc_stream(estk_ctx* ctx, const EvalMlpCall& c, cudaStream_t stream) {
  const char* why = "";
  if (!eval_mlp_tc_stream_supported(c.desc, c.B, &why)) {
    estk_set_error("estk_eval_mlp: shape not supported by the streamed tensor-core kernel (%s)", why);
    return ESTK_ERR_UNSUPPORTED;
  }
  if (c.centre_out) {
    estk_set_error("estk_eval_mlp: centre_return_out is served by the cluster kernel only; this shape runs the "
                   "streamed tensor-core kernel");
    return ESTK_ERR_UNSUPPORTED;
  }
  ESTK_CHECK_ARG(c.pairs >= 1 && c.pairs <= ESTK_MAX_POPULATION / 2, "estk_eval_mlp: pairs=%d", c.pairs);
  const estk_mlp_desc& d = c.desc;
  StreamParams p = {};
  p.desc = d; p.theta = c.theta; p.table = c.table; p.table16 = c.table16; p.offsets = c.offsets; p.order = c.order;
  p.pairs = c.pairs; p.sigma = c.sigma; p.target = c.target; p.B = c.B;
  p.ret_plus = c.ret_plus; p.ret_minus = c.ret_minus;
  p.bc_plus = c.bc_plus; p.bc_minus = c.bc_minus; p.bc_obs = c.bc_obs; p.bc_dim = c.bc_dim;
  p.chunks = (c.B + kRowsS - 1) / kRowsS;
  p.kb0 = (d.dims[0] + kBlockK - 1) / kBlockK;
  int widest = 0;
  for (int l = 1; l < d.n_layers; ++l) widest = std::max(widest, d.dims[l]);
  p.slab_kb = (widest + kTileNS - 1) / kTileNS * (kTileNS / kBlockK);
  const int64_t items = (int64_t)p.pairs * p.chunks;
  const StreamKernel kern = stream_kernel(d.activation);
  ESTK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemS));
  int per_sm = 0;
  ESTK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kThreadsS, kSmemS));
  const int grid = (int)std::min<int64_t>(items, (int64_t)ctx->sm_count * std::max(per_sm, 1));
  const int64_t xin_bytes = (int64_t)p.chunks * p.kb0 * 2 * kABytes;
  const int64_t slab_bytes = (int64_t)grid * 4 * p.slab_kb * kABytes;
  const int rc = estk_ctx_reserve(ctx, p.pairs, items * 2, stream, "estk_eval_mlp", (xin_bytes + slab_bytes) / 4);
  if (rc) return rc;
  p.partial = ctx->eval_partial;
  p.counters = estk_member_counters(ctx);
  uint8_t* ws = reinterpret_cast<uint8_t*>(ctx->eval_slab);
  p.xin = ws;
  p.slab = ws + xin_bytes;
  const int64_t n16 = xin_bytes / 2 / 16;
  const int blocks = (int)std::min<int64_t>((n16 + 255) / 256, (int64_t)ctx->sm_count * 16);
  split_obs_f16_kernel<<<blocks, 256, 0, stream>>>(c.obs, c.B, d.dims[0], p.kb0, n16, ws);
  ESTK_CUDA(cudaGetLastError());
  kern<<<grid, kThreadsS, kSmemS, stream>>>(p);
  ESTK_CUDA(cudaGetLastError());
  return ESTK_OK;
}
