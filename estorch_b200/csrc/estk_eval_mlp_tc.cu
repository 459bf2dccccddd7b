// estk_eval_mlp_tc.cu -- kernel 1 of the ES generation (population evaluate) on the Hopper
// tensor cores: warpgroup MMA (wgmma), 16-bit operands / fp32 accumulation.
//
// Same contract as estk_eval_mlp (estk_eval_mlp.cu; reference estorch.py:187-202 +
// Policy.forward examples/cartpole_es.py:14-20 + synthetic agent of SURVEY 8d),
// for policies whose dense layers are worth a GEMM.
//
// Work unit ("task") = (antithetic pair j, sign s, chunk of 64 observations), one CTA.  A cluster of
// four CTAs runs the four consecutive chunks of one (j, s) -- the same weights -- at the same time.
// Per layer
//   D[obs, out] = H[obs, in] * W_s[out, in]^T       (wgmma m64n128k16, N tiles of 128)
//   A  activations H, 64 rows, 16-bit, K-major, 128B-swizzled, resident in shared memory:
//      two buffers (64 KB each) swapped per layer, so a layer's output never overwrites its input;
//   B  W_s = theta + s*sigma*eps, formed ON THE FLY by producer warps into a ring of
//      [128 x 64] stages (16 KB) -- the perturbed weights never exist in global memory.  CTA q of
//      the cluster forms tile rows [q*w/4, (q+1)*w/4) of each stage and copies them into the same
//      slot of the other three CTAs (cp.async.bulk over distributed shared memory), so every weight
//      is read from L2 and formed once per 256 observations;
//   D  64 x 128 fp32 in the registers of the consumer warpgroup that owns the tile (the two
//      consumer warpgroups take alternate N tiles); the epilogue adds the bias,
//      applies the hidden activation (ReLU, or tanhf in fp32) and rounds to 16 bits straight into
//      the other activation buffer.  The last layer is fused with the optional output tanhf (fp32),
//      the squared-error reduction and the behaviour characterisation; with the cross-entropy
//      (ESTK_LOSS_XENT) each thread carries an online softmax of its two rows over its columns
//      (running max, rescaled sum of exponentials, sum t*y, sum t) from tile to tile, and the
//      warpgroup that drains the last tile combines the four lanes of each quad.
// Operand modes (template MODE):
//   kModeBF16   bf16 operands formed from fp32 theta + fp32 table (one FMA in fp32, one rounding)
//   kModeBF16S  bf16 operands formed from bf16 shadows of theta and table (fma.rn.bf16x2)
//   kModeF16    fp16 operands (11-bit significand, the TF32 class) from fp32 theta and the EXACT
//               16-bit copy of the noise table: W16 = rn_f16(theta + s*sigma*eps), sum in fp32; the
//               observations enter layer 0 as x_hi + x_lo (two fp16 k-block sets, same B tile)
// Warp roles: warpgroups 0 and 1 = consumers (MMA issue + epilogue) of alternate N tiles, so one
// warpgroup's epilogue runs under the other's MMAs; warps 8..15 = weight producers in
// four groups of two, each group forming every fourth stage of the flattened
// (task, layer, N tile, k-block) sequence.  full / empty mbarriers per ring stage: full[s] completes
// on the local group's arrival plus the bytes the three peers copy in; empty[s] counts the warps of
// the consuming warpgroup in all four CTAs, because a producer writes slot s of every CTA.  Persistent: clusters loop
// over groups of four tasks; the two signs of a pair run on neighbouring clusters at the same time,
// so the second read of the noise row is an L2 hit.
#include "estk_tc.cuh"
#include <type_traits>

namespace {

constexpr int kRows = 64;                          // observation rows per CTA (wgmma M)
constexpr int kTileN = 128;                        // wgmma N
constexpr int kHBlockBytes = kRows * kBlockK * 2;  // one [64 x 64] 16-bit k-block of activations = 8 KB
constexpr int kHBytes = (kMaxW / kBlockK) * kHBlockBytes;   // 64 KB per activation buffer
constexpr int kStageBytes = kTileN * kBlockK * 2;  // one [128 x 64] 16-bit B stage = 16 KB
constexpr int kStages = 5;
constexpr int kCluster = 4;                        // CTAs (observation chunks) sharing every B stage
constexpr int kProdWarps = 8, kProdGroups = 4, kProdGroupWarps = kProdWarps / kProdGroups;
constexpr int kPT = 32 * kProdGroupWarps;          // threads per producer group
constexpr int kConsWG = 2, kConsThreads = 128 * kConsWG;   // consumer warpgroups 0 and 1
constexpr int kThreadsTC = kConsThreads + 32 * kProdWarps; // 512
// Registers per thread after the role split (setmaxnreg).  At 512 threads the launch allows 128; a
// consumer holds a 64-float accumulator tile plus the task state and the last layer's target batch,
// a bf16-mode producer thread four items of 2 x 8 fp32 loads in flight plus their addresses.  The two
// warpgroups of each role must fit the 64K-register file: 2*128*kConsRegs + 2*128*kProdRegs <= 65536.
// The consumer spills below 152 and the bf16 producer below 104, so 152/104 is the one split with no
// local memory in either role for all three modes; it holds with target batches of two column blocks
// (four spill at 152) and with the producer's barrier id and CTA rank re-read instead of kept live.
constexpr int kConsRegs = 152, kProdRegs = 104;
static_assert(kConsRegs + kProdRegs <= 256, "setmaxnreg split exceeds the register file");
// Named barriers: 0 unused, 1 all consumers, 2..5 the producer groups, kBarOrder + w / kBarLoss + w
// hand tile ordering / the loss chain to consumer warpgroup w, kBarWG + w warpgroup w alone.
constexpr int kBarCons = 1, kBarOrder = 6, kBarLoss = 8, kBarWG = 10;
// Producers: a group waits for the release of the slot it is about to fill, kStages stages back; its
// previous stage, kProdGroups back, already saw the release before that.  So no group runs a full phase
// ahead of an empty barrier, which a parity wait could not tell apart.
// Consumers: the warpgroup that owns tile t waits on full for t's first stage only after the other
// warpgroup has issued every MMA of tile t-1, so every stage before it has been seen formed and the
// wait is within one lap of the barrier.  Without that order a warpgroup skipping the other's tile
// (up to 8 stages) would wait two phases ahead, and the parity wait would return on an unformed stage.
static_assert(kProdGroups <= kStages, "parity waits need kProdGroups <= kStages");
// 16-byte items per producer thread per stage: the CTA's quarter of the widest tile, in one batch
constexpr int kItemsPT = kTileN / kCluster * (kBlockK / 8) / kPT;
constexpr int kTgtBatch = 2;                       // last-layer epilogue: column blocks per target batch
constexpr int kTgtBatchX = 1;                      // the same with the cross-entropy (its 8-float chain
                                                   // state spills at 2 in the bf16 mode)
constexpr int kModeBF16 = 0, kModeBF16S = 1, kModeF16 = 2;

// ESTK_PREC_* -> operand mode; -1 for a precision without a tensor-core kernel
constexpr int mode_of(int precision) {
  return precision == ESTK_PREC_F16 ? kModeF16 : precision == ESTK_PREC_BF16 ? kModeBF16
       : precision == ESTK_PREC_BF16S ? kModeBF16S : -1;
}

struct EvalTCParams {
  estk_mlp_desc desc;
  const float* theta;
  const float* table;
  const uint16_t* theta16;  // bf16 shadows of theta / table (kModeBF16S)
  const uint16_t* table16;  // bf16 shadow (kModeBF16S) or exact fp16 copy (kModeF16) of the table
  const int64_t* offsets;   // null => centre evaluation
  const int32_t* order;
  int pairs;
  float sigma;
  const float* obs;
  const float* target;
  int B, chunks;            // chunks of kRows observations
  float* ret_plus;
  float* ret_minus;
  float* bc_plus;
  float* bc_minus;
  int bc_obs, bc_dim;
  float* partial;           // [pairs*2 + 1][chunks]
  unsigned int* counters;   // [pairs*2 + 1]
  float* centre_out;        // optional: also evaluate theta itself (sigma = 0) into centre_out[0]
  int n_centre;             // number of leading centre tasks (0 or chunks)
  int n_tasks;              // n_centre + pairs * n_signs * chunks
  int n_signs;              // 2, or 1 for the centre evaluation
  int mode;
#ifdef ESTK_TC_PROFILE
  unsigned long long* prof;  // [gridDim.x][warps][kPrBuckets] clock64() cycles, written at exit
#endif
};

#ifdef ESTK_TC_PROFILE
// Profile build only (-DESTK_TC_PROFILE): every warp sums clock64() deltas per role bucket in
// registers and lane 0 writes them once at exit.  Producer loads are waited for before the empty
// wait here (in the product they are still in flight during it), so kPrLoad is their full latency.
enum { kPrFull, kPrMma, kPrDrain, kPrLayer, kPrTask, kPrOther, kPrLoad, kPrEmpty, kPrForm, kPrBuckets };
unsigned long long* g_prof_buf = nullptr;
#define ESTK_PROF_DECL long long pr_[kPrBuckets] = {}; long long pr_t_ = clock64();
#define ESTK_PROF(b) do { const long long n_ = clock64(); pr_[b] += n_ - pr_t_; pr_t_ = n_; } while (0)
#else
#define ESTK_PROF_DECL
#define ESTK_PROF(b) do {} while (0)
#endif

struct Layer { int K, N; int64_t wbase, bbase; };

// task -> (slot, sign, chunk); the first n_centre tasks evaluate theta itself
struct TaskId { int slot, sgn, chunk; bool centre; };
__device__ __forceinline__ TaskId decode_task(const EvalTCParams& p, int task, bool all_centre) {
  TaskId t;
  if (task < p.n_centre) { t.slot = 0; t.sgn = 0; t.chunk = task; t.centre = true; return t; }
  const int q = task - p.n_centre;
  t.chunk = q % p.chunks;
  t.sgn = (q / p.chunks) % p.n_signs;
  t.slot = q / (p.chunks * p.n_signs);
  t.centre = all_centre;
  return t;
}

// ACT = estk_mlp_desc.activation, a compile-time constant: the ReLU / identity / squared-error
// instantiations are the code they were before Tanh and the cross-entropy existed, and no epilogue
// carries a branch on the activation or the loss.
template <int MODE, int ACT>
__global__ void __launch_bounds__(kThreadsTC, 1) eval_mlp_tc_kernel(const EvalTCParams p) {
  constexpr bool S16 = (MODE == kModeBF16S), F16 = (MODE == kModeF16);
  constexpr int HID = ACT & 0xff;
  constexpr bool OUT_TANH = (ACT & ESTK_ACT_OUT_TANH) != 0;
  constexpr bool XENT = (ACT & ESTK_LOSS_XENT) != 0;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sH = smem;                                  // 2 activation buffers x 8 k-blocks x 8 KB
  uint8_t* sB = sH + 2 * kHBytes;                      // ring
  float* sBias = reinterpret_cast<float*>(sB + kStages * kStageBytes);   // [2][512], by layer parity
  uint64_t* bar_full = reinterpret_cast<uint64_t*>(sBias + 2 * kMaxW);  // [kStages] stage formed
  uint64_t* bar_empty = bar_full + kStages;                             // [kStages] stage consumed
  float* s_loss = reinterpret_cast<float*>(bar_empty + kStages);        // [4]
  float* s_chain = s_loss + 4;                                          // [128] loss chain handoff
                                                                        // ([8][128] with the cross-entropy)
  __shared__ Layer lay[ESTK_MAX_LAYERS];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int L = p.desc.n_layers;
  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(smem_u32(bar_full + s), 1);                // the forming group's elected thread (+ peer bytes)
      mbar_init(smem_u32(bar_empty + s), 4 * kCluster);    // the consuming warpgroup's warps, every CTA
    }
    fence_barrier_init();
    int64_t pb = 0;
    for (int l = 0; l < L; ++l) {
      lay[l].K = p.desc.dims[l];
      lay[l].N = p.desc.dims[l + 1];
      lay[l].wbase = pb;
      lay[l].bbase = pb + (int64_t)lay[l].K * lay[l].N;
      pb = lay[l].bbase + lay[l].N;
    }
  }
  cluster_sync();   // barriers initialised in every CTA before any remote arrive or copy
  const bool centre = (p.offsets == nullptr);
  ESTK_PROF_DECL

  if (warp < 4 * kConsWG) {
    // =================================================================== consumer warpgroups
    // Tile t of the CTA's running (task, layer, N tile) sequence belongs to warpgroup t % 2.  The
    // alternation does not restart per task: a task has an odd number of tiles at the north star (19).
    setmaxnreg_inc<kConsRegs>();
    const int cw = warp >> 2;                        // consumer warpgroup
    const int ctid = threadIdx.x;                    // 0..255
    const int tid = ctid & 127;                      // thread of the warpgroup
    const int r0 = (warp & 3) * 16 + (lane >> 2);    // accumulator rows r0 and r0 + 8
    const int cq = (lane & 3) * 2;                   // accumulator columns 8j + cq, +1
    uint32_t kst = 0;                                // global stage index
    bool mine = (cw == 0);                           // the next tile is this warpgroup's
    bool after = (cw != 0);                          // a tile precedes this warpgroup's next one
    // gridDim.x and chunks (B % 256 == 0) are multiples of kCluster: the CTAs of a cluster always hold
    // the kCluster consecutive chunks of one (pair, sign), CTA rank = chunk % kCluster
    for (int task = blockIdx.x; task < p.n_tasks; task += gridDim.x) {
      const TaskId tk = decode_task(p, task, centre);
      const int chunk = tk.chunk, sgn = tk.sgn, slot = tk.slot;
      const int j = (!tk.centre && p.order) ? p.order[slot] : slot;
      const float* trow = tk.centre ? p.theta : p.table + p.offsets[j];
      const float ssig = tk.centre ? 0.f : (sgn ? -p.sigma : p.sigma);
      const bool with_bc = !(tk.centre && !centre) && p.bc_plus;   // the row pointer is formed at use
      const bool final_task = task + (int)gridDim.x >= p.n_tasks;
      // every MMA of the previous task has completed (buffer 0 and sBias[0] are free) and its loss
      // has been combined
      named_bar_sync(kBarCons, kConsThreads);
      // ---- this CTA's observations as the layer-0 A operand (buffer 0)
      {
        const int K0 = lay[0].K, per_row = K0 / 8;
        for (int it = ctid; it < kRows * per_row; it += kConsThreads) {
          const int r = it / per_row, c = it % per_row;
          const float* src = p.obs + (size_t)(chunk * kRows + r) * K0 + c * 8;
          const float4 x0 = __ldg(reinterpret_cast<const float4*>(src));
          const float4 x1 = __ldg(reinterpret_cast<const float4*>(src + 4));
          const uint32_t addr = smem_u32(sH + (c >> 3) * kHBlockBytes) + sw128_offset(r, c & 7);
          const uint32_t h0 = pack16<F16>(x0.x, x0.y), h1 = pack16<F16>(x0.z, x0.w);
          const uint32_t h2 = pack16<F16>(x1.x, x1.y), h3 = pack16<F16>(x1.z, x1.w);
          st_shared_v4(addr, h0, h1, h2, h3);
          if constexpr (F16) {
            // x_lo = rn_f16(x - x_hi): the observation enters layer 0 with ~22 significant bits
            const float2 f0 = unpack_f16(h0), f1 = unpack_f16(h1), f2 = unpack_f16(h2), f3 = unpack_f16(h3);
            st_shared_v4(addr + (K0 / kBlockK) * kHBlockBytes, pack_f16(x0.x - f0.x, x0.y - f0.y),
                         pack_f16(x0.z - f1.x, x0.w - f1.y), pack_f16(x1.x - f2.x, x1.y - f2.y),
                         pack_f16(x1.z - f3.x, x1.w - f3.y));
          }
        }
      }
      ESTK_PROF(kPrTask);
      float loss = 0.f;
      for (int l = 0; l < L; ++l) {
        const int K = lay[l].K, N = lay[l].N;
        const bool last = (l == L - 1);
        const uint32_t h_in = smem_u32(sH + (l & 1) * kHBytes);
        const uint32_t h_out = smem_u32(sH + ((l + 1) & 1) * kHBytes);
        // Layer l's bias goes to sBias[l & 1].  Its last readers, layer l-2's epilogues, finished
        // before the barrier that opened layer l-1, which this thread has passed.
        float* bias = sBias + (l & 1) * kMaxW;
        {
          // every load first: a store between two loads would make each wait for the one before
          float bz[kMaxW / kConsThreads], bt[kMaxW / kConsThreads];
#pragma unroll
          for (int i = 0; i < kMaxW / kConsThreads; ++i) {
            const int o = ctid + i * kConsThreads;
            if (o < N) {
              bz[i] = ld_noise1(trow + lay[l].bbase + o);
              bt[i] = __ldg(p.theta + lay[l].bbase + o);
            }
          }
#pragma unroll
          for (int i = 0; i < kMaxW / kConsThreads; ++i)
            if (ctid + i * kConsThreads < N) bias[ctid + i * kConsThreads] = fmaf(ssig, bz[i], bt[i]);
        }
        // This layer's input, written by both warpgroups (generic-proxy stores) -> wgmma.  Past this
        // barrier every MMA of layer l-1 has completed too, so its input buffer may be overwritten.
        fence_proxy_async();
        named_bar_sync(kBarCons, kConsThreads);
        ESTK_PROF(kPrLayer);
        const int lo_kb = (F16 && l == 0) ? K / kBlockK : 0;   // layer 0 in fp16: x_lo k-blocks
        for (int n0 = 0; n0 < N; n0 += kTileN, mine = !mine) {
          if (!mine) {                       // the other warpgroup's tile
            kst += K / kBlockK;
            continue;
          }
          const int width = min(kTileN, N - n0);
          const bool last_tile = n0 + kTileN >= N;
          if (after) named_bar_sync(kBarOrder + cw, kConsThreads);    // the previous tile's MMAs issued
          after = true;
          ESTK_PROF(kPrOther);
          float d[64];                     // the first MMA of the tile overwrites (scale-d = 0)
          uint32_t prev = 0;
          // NP = 2: layer 0 in fp16, x_lo on the same B tile (a separate instantiation, so that no
          // wgmma sits under a branch)
          auto k_loop = [&](auto np_tag) {
            constexpr int NP = decltype(np_tag)::value;
            for (int kb = 0; kb < K / kBlockK; ++kb, ++kst) {
              const uint32_t stage = kst % kStages, phase = (kst / kStages) & 1u;
              mbar_wait(smem_u32(bar_full + stage), phase);
              ESTK_PROF(kPrFull);
              const uint32_t a_addr = h_in + kb * kHBlockBytes, b_addr = smem_u32(sB + stage * kStageBytes);
              wgmma_fence();
#pragma unroll
              for (int pass = 0; pass < NP; ++pass) {
                const uint32_t a = a_addr + pass * lo_kb * kHBlockBytes;
#pragma unroll
                for (int k = 0; k < kBlockK / 16; ++k)
                  wgmma_m64n128k16<F16>(d, make_sw128_desc(a + k * 32), make_sw128_desc(b_addr + k * 32),
                                        (kb | k | pass) != 0 ? 1u : 0u);
              }
              wgmma_commit();
              wgmma_wait<1>();             // the previous stage's MMAs are done: release its slot
              if (kb > 0 && lane < kCluster) mbar_arrive_cluster(mapa_shared(smem_u32(bar_empty + prev), lane));
              prev = stage;
              ESTK_PROF(kPrMma);
            }
          };
          if (F16 && lo_kb) k_loop(std::integral_constant<int, 2>{});
          else k_loop(std::integral_constant<int, 1>{});
          if (!(last && last_tile && final_task)) named_bar_arrive(kBarOrder + (cw ^ 1), kConsThreads);
          wgmma_wait<0>();
          fence_acc(d);
          if (lane < kCluster) mbar_arrive_cluster(mapa_shared(smem_u32(bar_empty + prev), lane));
          // ---- epilogue of the tile
          if (XENT && last) {
            // Cross-entropy.  Per thread and row h (r0 + 8h): first this tile's max, sum t*y and sum t
            // over the thread's columns, with d turned into the logits; then the sum of exp(y - max).
            float tm[2] = {-INFINITY, -INFINITY}, tsty[2] = {0.f, 0.f}, tst[2] = {0.f, 0.f};
#pragma unroll
            for (int jg = 0; jg < kTileN / 8; jg += kTgtBatchX) {
              float2 t[kTgtBatchX][2];
#pragma unroll
              for (int jb = jg; jb < jg + kTgtBatchX; ++jb)
#pragma unroll
                for (int h = 0; h < 2; ++h)
                  if (jb * 8 < width)
                    t[jb - jg][h] = __ldg(reinterpret_cast<const float2*>(
                        p.target + (size_t)(chunk * kRows + r0 + 8 * h) * N + n0 + jb * 8 + cq));
#pragma unroll
              for (int jb = jg; jb < jg + kTgtBatchX; ++jb) {
                if (jb * 8 < width) {
                  const int col = n0 + jb * 8 + cq;
                  const float2 bv = *reinterpret_cast<const float2*>(bias + col);
#pragma unroll
                  for (int h = 0; h < 2; ++h) {
                    const int b = chunk * kRows + r0 + 8 * h;
                    const float y0 = d[jb * 4 + 2 * h] + bv.x, y1 = d[jb * 4 + 2 * h + 1] + bv.y;
                    d[jb * 4 + 2 * h] = y0;
                    d[jb * 4 + 2 * h + 1] = y1;
                    tm[h] = fmaxf(fmaxf(tm[h], y0), y1);
                    tsty[h] = fmaf(t[jb - jg][h].y, y1, fmaf(t[jb - jg][h].x, y0, tsty[h]));
                    tst[h] = (tst[h] + t[jb - jg][h].x) + t[jb - jg][h].y;
                    if (with_bc && b < p.bc_obs) {
                      float* bc = sgn ? p.bc_minus : p.bc_plus;
                      const int64_t idx = (int64_t)b * N + col;
                      if (idx < p.bc_dim) bc[(size_t)j * p.bc_dim + idx] = y0;
                      if (idx + 1 < p.bc_dim) bc[(size_t)j * p.bc_dim + idx + 1] = y1;
                    }
                  }
                }
              }
            }
            float ts[2] = {0.f, 0.f};
#pragma unroll
            for (int jb = 0; jb < kTileN / 8; ++jb)
              if (jb * 8 < width)
#pragma unroll
                for (int h = 0; h < 2; ++h)
                  ts[h] = (ts[h] + expf(d[jb * 4 + 2 * h] - tm[h])) + expf(d[jb * 4 + 2 * h + 1] - tm[h]);
            // the chain (max, sum exp, sum t*y, sum t) continues from the previous tile, which the
            // other warpgroup drained; thread tid of both warpgroups holds the same rows and columns
            if (n0 > 0) {
              ESTK_PROF(kPrDrain);
              named_bar_sync(kBarLoss + cw, kConsThreads);
              ESTK_PROF(kPrOther);
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const float cm = s_chain[(4 * h) * 128 + tid], nm = fmaxf(cm, tm[h]);
                ts[h] = s_chain[(4 * h + 1) * 128 + tid] * expf(cm - nm) + ts[h] * expf(tm[h] - nm);
                tm[h] = nm;
                tsty[h] = s_chain[(4 * h + 2) * 128 + tid] + tsty[h];
                tst[h] = s_chain[(4 * h + 3) * 128 + tid] + tst[h];
              }
            }
            if (!last_tile) {                // hand the chain to the warpgroup of the next tile
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                s_chain[(4 * h) * 128 + tid] = tm[h];
                s_chain[(4 * h + 1) * 128 + tid] = ts[h];
                s_chain[(4 * h + 2) * 128 + tid] = tsty[h];
                s_chain[(4 * h + 3) * 128 + tid] = tst[h];
              }
              named_bar_arrive(kBarLoss + (cw ^ 1), kConsThreads);
            } else {
              // the row's four lanes (the quad) hold disjoint columns: combine them, lane distance 1
              // then 2, and form ce once per row on the quad's first lane
#pragma unroll
              for (int o = 1; o <= 2; o <<= 1)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                  const float om = __shfl_xor_sync(0xffffffffu, tm[h], o);
                  const float os = __shfl_xor_sync(0xffffffffu, ts[h], o);
                  const float osty = __shfl_xor_sync(0xffffffffu, tsty[h], o);
                  const float ost = __shfl_xor_sync(0xffffffffu, tst[h], o);
                  const float nm = fmaxf(tm[h], om);
                  ts[h] = ts[h] * expf(tm[h] - nm) + os * expf(om - nm);
                  tm[h] = nm;
                  tsty[h] += osty;
                  tst[h] += ost;
                }
              if ((lane & 3) == 0)
                loss = fmaf(tm[0] + logf(ts[0]), tst[0], -tsty[0]) + fmaf(tm[1] + logf(ts[1]), tst[1], -tsty[1]);
            }
          } else if (last) {
            // the targets of kTgtBatch column blocks are loaded before any is used: the behaviour-
            // characterisation stores would otherwise hold each load until the one before returned
#pragma unroll
            for (int jg = 0; jg < kTileN / 8; jg += kTgtBatch) {
              float2 t[kTgtBatch][2];
#pragma unroll
              for (int jb = jg; jb < jg + kTgtBatch; ++jb)
#pragma unroll
                for (int h = 0; h < 2; ++h)
                  if (jb * 8 < width)
                    t[jb - jg][h] = __ldg(reinterpret_cast<const float2*>(
                        p.target + (size_t)(chunk * kRows + r0 + 8 * h) * N + n0 + jb * 8 + cq));
              if (jg == 0 && n0 > 0) {
                // the squared-error chain continues from the previous tile, which the other
                // warpgroup drained; thread tid of both warpgroups holds the same rows and columns
                ESTK_PROF(kPrDrain);
                named_bar_sync(kBarLoss + cw, kConsThreads);
                loss = s_chain[tid];
                ESTK_PROF(kPrOther);
              }
#pragma unroll
              for (int jb = jg; jb < jg + kTgtBatch; ++jb) {
                if (jb * 8 < width) {
                  const int col = n0 + jb * 8 + cq;
                  const float2 bv = *reinterpret_cast<const float2*>(bias + col);
#pragma unroll
                  for (int h = 0; h < 2; ++h) {
                    const int b = chunk * kRows + r0 + 8 * h;
                    float y0 = d[jb * 4 + 2 * h] + bv.x, y1 = d[jb * 4 + 2 * h + 1] + bv.y;
                    if constexpr (OUT_TANH) { y0 = tanhf(y0); y1 = tanhf(y1); }
                    const float e0 = y0 - t[jb - jg][h].x, e1 = y1 - t[jb - jg][h].y;
                    loss = fmaf(e0, e0, loss);
                    loss = fmaf(e1, e1, loss);
                    if (with_bc && b < p.bc_obs) {
                      float* bc = sgn ? p.bc_minus : p.bc_plus;
                      const int64_t idx = (int64_t)b * N + col;
                      if (idx < p.bc_dim) bc[(size_t)j * p.bc_dim + idx] = y0;
                      if (idx + 1 < p.bc_dim) bc[(size_t)j * p.bc_dim + idx + 1] = y1;
                    }
                  }
                }
              }
            }
            if (!last_tile) {                // hand the chain to the warpgroup of the next tile
              s_chain[tid] = loss;
              named_bar_arrive(kBarLoss + (cw ^ 1), kConsThreads);
            }
          } else {
#pragma unroll
            for (int jb = 0; jb < kTileN / 8; ++jb) {
              if (jb * 8 < width) {
                const int col = n0 + jb * 8 + cq;
                const float2 bv = *reinterpret_cast<const float2*>(bias + col);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                  const int r = r0 + 8 * h;
                  const float y0 = d[jb * 4 + 2 * h] + bv.x, y1 = d[jb * 4 + 2 * h + 1] + bv.y;
                  // ReLU fused into the conversion; any other kind: fp32 activation, then the one rounding
                  // to 16 bits (saturating in fp16; |tanh| <= 1, so for Tanh it never fires).  SiLU divides
                  // without div.rn's out-of-line call, which spills the bf16 consumer.
                  st_shared_u32(h_out + (col >> 6) * kHBlockBytes + sw128_offset(r, (col & 63) >> 3) + (col & 7) * 2,
                                HID == ESTK_ACT_RELU ? pack16_relu<F16>(y0, y1)
                                                     : pack16<F16>(estk_hidden_act<HID, true>(y0),
                                                                   estk_hidden_act<HID, true>(y1)));
                }
              }
            }
          }
          ESTK_PROF(kPrDrain);
        }
      }
      // ---- squared-error partial of this CTA, from the warpgroup that drained the task's last tile;
      // the last arriver combines them in fixed order
      if (mine) continue;
      loss = warp_sum_f(loss);
      if (lane == 0) s_loss[warp & 3] = loss;
      named_bar_sync(kBarWG + cw, 128);
      if (tid == 0) {
        const float tot = (s_loss[0] + s_loss[1]) + (s_loss[2] + s_loss[3]);
        const int parts = p.chunks;
        const bool folded = tk.centre && !centre;                 // centre task riding in a population launch
        const int cell = folded ? p.pairs * 2 : slot * 2 + sgn;
        float* part = p.partial + (size_t)cell * parts;
        part[chunk] = tot;
        __threadfence();
        const unsigned int arrived = atomicAdd(p.counters + cell, 1u);
        if (arrived == (unsigned int)parts - 1) {
          __threadfence();
          float s = 0.f;
          for (int c = 0; c < parts; ++c) s += __ldcg(part + c);
          const float r = XENT ? -(s / (float)p.B) : -(s / ((float)p.B * (float)lay[L - 1].N));
          if (folded) p.centre_out[0] = r;
          else if (sgn) p.ret_minus[j] = r;
          else p.ret_plus[j] = r;
          p.counters[cell] = 0u;
        }
      }
      ESTK_PROF(kPrTask);
    }
  } else {
    // =================================================================== weight producers
    // Group g forms stages g, g+G, g+2G, ... of the flattened (task, layer, N tile, k-block)
    // sequence, this CTA's quarter of each: tile rows [rank*w/4, (rank+1)*w/4).  w % 32 == 0, so a
    // quarter is whole 8-row swizzle atoms, one contiguous 1024-B-aligned byte range of the stage.
    // Item `it` of the quarter = its row it/8, 16-byte output chunk it%8 (8 weights).
    setmaxnreg_dec<kProdRegs>();
    const int pwarp = warp - 4 * kConsWG;
    const int pgroup = pwarp / kProdGroupWarps;
    const int ptid = (pwarp % kProdGroupWarps) * 32 + lane;
    bool new_task = true;                 // the per-task row pointers are stale
    const float* trow = p.theta;
    const uint16_t* trow16 = nullptr;
    float ssig = 0.f;
    int task = blockIdx.x, l = 0, n0 = 0, kb = 0;
    auto advance = [&]() -> bool {
      if (++kb >= lay[l].K / kBlockK) {
        kb = 0;
        n0 += kTileN;
        if (n0 >= lay[l].N) {
          n0 = 0;
          if (++l == L) { l = 0; task += gridDim.x; new_task = true; }
        }
      }
      return task < p.n_tasks;
    };
    bool has = task < p.n_tasks;
    for (int sk = 0; sk < pgroup && has; ++sk) has = advance();
    uint32_t kst = pgroup;
    while (has) {
      if (new_task) {                       // two dependent global loads: once per task, not per stage
        new_task = false;
        const TaskId tk = decode_task(p, task, centre);
        const int jj = (!tk.centre && p.order) ? p.order[tk.slot] : tk.slot;
        trow = tk.centre ? p.theta : p.table + p.offsets[jj];
        trow16 = tk.centre ? (S16 ? p.theta16 : nullptr) : p.table16 + p.offsets[jj];
        ssig = tk.centre ? 0.f : (tk.sgn ? -p.sigma : p.sigma);
      }
      const uint32_t stage = kst % kStages, phase = (kst / kStages) & 1u;
      const uint32_t sbase = smem_u32(sB + stage * kStageBytes);
      const int K = lay[l].K;
      const int qrows = min(kTileN, lay[l].N - n0) / kCluster;
      const int n_items = qrows * 8;
      const uint32_t rank = cluster_ctarank();
      const uint32_t qbase = sbase + rank * qrows * 128, qbytes = qrows * 128;
      const int64_t rbase = lay[l].wbase + (int64_t)(n0 + rank * qrows) * K + kb * kBlockK;
      {
        float4 th[kItemsPT][2], ep[kItemsPT][2];
        uint4 t16[kItemsPT], e16[kItemsPT];
        // every load of the stage is issued up front ...
#pragma unroll
        for (int u = 0; u < kItemsPT; ++u) {
          const int it = u * kPT + ptid;
          if (it < n_items) {
            const int64_t off = rbase + (int64_t)(it >> 3) * K + (it & 7) * 8;
            if constexpr (S16) {
              t16[u] = ld_noise4u(reinterpret_cast<const uint4*>(p.theta16 + off));
              e16[u] = ld_noise4u(reinterpret_cast<const uint4*>(trow16 + off));
            } else if constexpr (F16) {
              th[u][0] = ld_noise4(reinterpret_cast<const float4*>(p.theta + off));
              th[u][1] = ld_noise4(reinterpret_cast<const float4*>(p.theta + off + 4));
              e16[u] = trow16 ? ld_noise4u(reinterpret_cast<const uint4*>(trow16 + off)) : make_uint4(0u, 0u, 0u, 0u);
            } else {
              th[u][0] = ld_noise4(reinterpret_cast<const float4*>(p.theta + off));
              th[u][1] = ld_noise4(reinterpret_cast<const float4*>(p.theta + off + 4));
              ep[u][0] = ld_noise4(reinterpret_cast<const float4*>(trow + off));
              ep[u][1] = ld_noise4(reinterpret_cast<const float4*>(trow + off + 4));
            }
          }
        }
#ifdef ESTK_TC_PROFILE
        uint32_t ready = 0;
#pragma unroll
        for (int u = 0; u < kItemsPT; ++u) {
          if constexpr (S16) ready ^= t16[u].x ^ e16[u].x;
          else if constexpr (F16) ready ^= __float_as_uint(th[u][1].w) ^ e16[u].x;
          else ready ^= __float_as_uint(th[u][1].w) ^ __float_as_uint(ep[u][1].w);
        }
        if (ready == 0x7fc00001u) pr_[kPrForm] -= 1;   // makes the clock read below wait for the data
        ESTK_PROF(kPrLoad);
#endif
        // ... then wait for the ring slot, free in all four CTAs
        mbar_wait(smem_u32(bar_empty + stage), phase ^ 1);
        ESTK_PROF(kPrEmpty);
#pragma unroll
        for (int u = 0; u < kItemsPT; ++u) {
          const int it = u * kPT + ptid;
          if (it < n_items) {
            const float sg = ssig;
            uint32_t w[4];
            if constexpr (S16) {
              // W = theta16 + (s*sigma)_bf16 * eps16: exact product-sum, one rounding to bf16
              const uint32_t sg2 = pack_bf16(sg, sg);
              const uint32_t tw[4] = {t16[u].x, t16[u].y, t16[u].z, t16[u].w};
              const uint32_t ew[4] = {e16[u].x, e16[u].y, e16[u].z, e16[u].w};
#pragma unroll
              for (int c = 0; c < 4; ++c) asm("fma.rn.bf16x2 %0, %1, %2, %3;" : "=r"(w[c]) : "r"(sg2), "r"(ew[c]), "r"(tw[c]));
            } else if constexpr (F16) {
              const float2 e0 = unpack_f16(e16[u].x), e1 = unpack_f16(e16[u].y);
              const float2 e2 = unpack_f16(e16[u].z), e3 = unpack_f16(e16[u].w);
              w[0] = pack_f16(fmaf(sg, e0.x, th[u][0].x), fmaf(sg, e0.y, th[u][0].y));
              w[1] = pack_f16(fmaf(sg, e1.x, th[u][0].z), fmaf(sg, e1.y, th[u][0].w));
              w[2] = pack_f16(fmaf(sg, e2.x, th[u][1].x), fmaf(sg, e2.y, th[u][1].y));
              w[3] = pack_f16(fmaf(sg, e3.x, th[u][1].z), fmaf(sg, e3.y, th[u][1].w));
            } else {
              w[0] = pack_bf16(fmaf(sg, ep[u][0].x, th[u][0].x), fmaf(sg, ep[u][0].y, th[u][0].y));
              w[1] = pack_bf16(fmaf(sg, ep[u][0].z, th[u][0].z), fmaf(sg, ep[u][0].w, th[u][0].w));
              w[2] = pack_bf16(fmaf(sg, ep[u][1].x, th[u][1].x), fmaf(sg, ep[u][1].y, th[u][1].y));
              w[3] = pack_bf16(fmaf(sg, ep[u][1].z, th[u][1].z), fmaf(sg, ep[u][1].w, th[u][1].w));
            }
            st_shared_v4(qbase + sw128_offset(it >> 3, it & 7), w[0], w[1], w[2], w[3]);
          }
        }
      }
      fence_proxy_async();                  // the quarter -> async proxy (local wgmma, bulk copies)
      named_bar_sync(2 + (int)(threadIdx.x / kPT) - kConsThreads / kPT, kPT);   // 2 + pgroup
      if (ptid == 0) {
        // full[stage] of this CTA: this arrival + the three quarters the peers copy in.  A peer's
        // bytes may land before the expect_tx (the transaction count goes negative meanwhile); the
        // phase cannot complete before this arrival either way.
        const uint32_t full = smem_u32(bar_full + stage);
        mbar_arrive_expect_tx(full, (kCluster - 1) * qbytes);
        for (uint32_t r = 1; r < kCluster; ++r) {
          const uint32_t peer = (rank + r) % kCluster;
          bulk_copy_to_cluster(mapa_shared(qbase, peer), qbase, qbytes, mapa_shared(full, peer));
        }
      }
      for (int sk = 0; sk < kProdGroups && has; ++sk) has = advance();
      kst += kProdGroups;
      ESTK_PROF(kPrForm);
    }
  }
#ifdef ESTK_TC_PROFILE
  if (lane == 0 && p.prof) {
    unsigned long long* o = p.prof + ((size_t)blockIdx.x * (blockDim.x / 32) + warp) * kPrBuckets;
    for (int b = 0; b < kPrBuckets; ++b) o[b] = (unsigned long long)pr_[b];
  }
#endif
  // No CTA leaves while a peer may still arrive on its barriers or copy into its ring: every copy into
  // this CTA completed on its full barriers before its consumer finished, and every peer reaches this
  // point only after its last remote arrival.
  cluster_sync();
}

// the cross-entropy's loss chain carries 8 floats per consumer thread instead of 1
size_t tc_smem_bytes(bool xent) {
  return 1024 + 2 * (size_t)kHBytes + (size_t)kStages * kStageBytes + 2 * kMaxW * sizeof(float) +
         2 * kStages * sizeof(uint64_t) + (4 + (xent ? 8 : 1) * 128) * sizeof(float);
}

// Clusters of kCluster CTAs, one per SM, persistent over groups of kCluster tasks.  The number of
// clusters that fit at once comes from the occupancy API: the GPCs' SM counts need not be multiples of
// kCluster, so it can be less than sm_count / kCluster.
template <int MODE, int ACT>
int launch_tc(const EvalTCParams& p, cudaStream_t stream) {
  const size_t smem = tc_smem_bytes((ACT & ESTK_LOSS_XENT) != 0);
  ESTK_CUDA(cudaFuncSetAttribute(eval_mlp_tc_kernel<MODE, ACT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = kCluster;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(kCluster);
  cfg.blockDim = dim3(kThreadsTC);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  int clusters = 0;
  ESTK_CUDA(cudaOccupancyMaxActiveClusters(&clusters, eval_mlp_tc_kernel<MODE, ACT>, &cfg));
  if (clusters < 1) {
    estk_set_error("eval_mlp_tc_kernel: no cluster of %d CTAs fits on this device", kCluster);
    return ESTK_ERR_CUDA;
  }
  const int items = p.n_tasks / kCluster;
  cfg.gridDim = dim3(kCluster * (clusters < items ? clusters : items));
  ESTK_CUDA(cudaLaunchKernelEx(&cfg, eval_mlp_tc_kernel<MODE, ACT>, p));
  return ESTK_OK;
}

int tc_supported(const estk_mlp_desc& d, int B, const char** why, int mode) {
  if (mode == kModeF16 && d.n_layers >= 1 && 2 * d.dims[0] > kMaxW) {
    *why = "fp16 mode splits the observations into hi + lo halves: input width <= 256"; return 0;
  }
  if (d.n_layers < 1 || d.n_layers > ESTK_MAX_LAYERS) { *why = "n_layers"; return 0; }
  if (!estk_act_valid(d.activation)) { *why = "activation is not a defined ESTK_ACT_* combination"; return 0; }
  for (int l = 0; l < d.n_layers; ++l) {
    if (d.dims[l] % 64 || d.dims[l] > kMaxW || d.dims[l] < 64) { *why = "layer input width must be a multiple of 64 in [64,512]"; return 0; }
    const int N = d.dims[l + 1];
    if (N % 32 || N > kMaxW || N < 32) { *why = "layer output width must be a multiple of 32 in [32,512]"; return 0; }
  }
  if (B % 256) { *why = "batch must be a multiple of 256"; return 0; }
  return 1;
}

template <int MODE>
int launch_tc_act(const EvalTCParams& p, cudaStream_t stream) {
  switch (p.desc.activation) {
    case ESTK_ACT_TANH: return launch_tc<MODE, ESTK_ACT_TANH>(p, stream);
    case ESTK_ACT_OUT_TANH: return launch_tc<MODE, ESTK_ACT_OUT_TANH>(p, stream);
    case ESTK_ACT_TANH | ESTK_ACT_OUT_TANH: return launch_tc<MODE, ESTK_ACT_TANH | ESTK_ACT_OUT_TANH>(p, stream);
    case ESTK_LOSS_XENT: return launch_tc<MODE, ESTK_LOSS_XENT>(p, stream);
    case ESTK_LOSS_XENT | ESTK_ACT_TANH: return launch_tc<MODE, ESTK_LOSS_XENT | ESTK_ACT_TANH>(p, stream);
    case ESTK_ACT_ELU: return launch_tc<MODE, ESTK_ACT_ELU>(p, stream);
    case ESTK_ACT_ELU | ESTK_ACT_OUT_TANH: return launch_tc<MODE, ESTK_ACT_ELU | ESTK_ACT_OUT_TANH>(p, stream);
    case ESTK_ACT_ELU | ESTK_LOSS_XENT: return launch_tc<MODE, ESTK_ACT_ELU | ESTK_LOSS_XENT>(p, stream);
    case ESTK_ACT_SILU: return launch_tc<MODE, ESTK_ACT_SILU>(p, stream);
    case ESTK_ACT_SILU | ESTK_ACT_OUT_TANH: return launch_tc<MODE, ESTK_ACT_SILU | ESTK_ACT_OUT_TANH>(p, stream);
    case ESTK_ACT_SILU | ESTK_LOSS_XENT: return launch_tc<MODE, ESTK_ACT_SILU | ESTK_LOSS_XENT>(p, stream);
    case ESTK_ACT_LEAKY_RELU: return launch_tc<MODE, ESTK_ACT_LEAKY_RELU>(p, stream);
    case ESTK_ACT_LEAKY_RELU | ESTK_ACT_OUT_TANH: return launch_tc<MODE, ESTK_ACT_LEAKY_RELU | ESTK_ACT_OUT_TANH>(p, stream);
    case ESTK_ACT_LEAKY_RELU | ESTK_LOSS_XENT: return launch_tc<MODE, ESTK_ACT_LEAKY_RELU | ESTK_LOSS_XENT>(p, stream);
    default: return launch_tc<MODE, ESTK_ACT_RELU>(p, stream);
  }
}

int run_tc(estk_ctx* ctx, EvalTCParams& p, cudaStream_t stream, const char* who) {
  const char* why = "";
  if (!tc_supported(p.desc, p.B, &why, p.mode)) {
    estk_set_error("%s: shape not supported by the tensor-core path (%s)", who, why);
    return ESTK_ERR_UNSUPPORTED;
  }
  ESTK_CHECK_ARG(p.pairs >= 1 && p.pairs <= ESTK_MAX_POPULATION / 2, "%s: pairs=%d", who, p.pairs);
  p.chunks = p.B / kRows;
  ESTK_CHECK_ARG(p.chunks <= 2 * kEvalMaxChunks, "%s: batch too large", who);
  p.n_centre = p.centre_out ? p.chunks : 0;
  p.n_tasks = p.n_centre + p.pairs * p.n_signs * p.chunks;
  const int64_t cells = (int64_t)p.pairs * 2 + (p.centre_out ? 1 : 0);   // [pairs][sign], then the folded centre
  const int rc = estk_ctx_reserve(ctx, cells, cells * p.chunks, stream, who);
  if (rc) return rc;
  p.partial = ctx->eval_partial;
  p.counters = estk_member_counters(ctx);
#ifdef ESTK_TC_PROFILE
  p.prof = g_prof_buf;
#endif
  if (p.mode == kModeF16) return launch_tc_act<kModeF16>(p, stream);
  if (p.mode == kModeBF16S) return launch_tc_act<kModeBF16S>(p, stream);
  return launch_tc_act<kModeBF16>(p, stream);
}

}  // namespace

// estk_eval_mlp with a tensor-core precision (estk_eval_mlp.cu has checked the arguments).
// ESTK_PREC_F16_ANY: this file's kernel in fp16 mode where its shape rule holds, else the streamed kernel.
int eval_mlp_tc(estk_ctx* ctx, const EvalMlpCall& c, cudaStream_t stream) {
  int precision = c.precision;
  if (precision == ESTK_PREC_F16_ANY) {
    const char* why = "";
    if (!tc_supported(c.desc, c.B, &why, kModeF16)) return eval_mlp_tc_stream(ctx, c, stream);
    precision = ESTK_PREC_F16;
  }
  EvalTCParams p = {};
  p.desc = c.desc; p.theta = c.theta; p.table = c.table; p.theta16 = c.theta16; p.table16 = c.table16;
  p.offsets = c.offsets; p.order = c.order;
  p.pairs = c.pairs; p.sigma = c.sigma; p.obs = c.obs; p.target = c.target; p.B = c.B;
  p.ret_plus = c.ret_plus; p.ret_minus = c.ret_minus;
  p.bc_plus = c.bc_plus; p.bc_minus = c.bc_minus; p.bc_obs = c.bc_obs; p.bc_dim = c.bc_dim;
  p.n_signs = c.offsets ? 2 : 1; p.centre_out = c.centre_out; p.mode = mode_of(precision);
  return run_tc(ctx, p, stream, "estk_eval_mlp");
}

__global__ void __launch_bounds__(256) shadow_bf16_kernel(const float4* __restrict__ src, uint2* __restrict__ dst, int64_t n4) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 v = src[i];
    uint2 o;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(o.x) : "f"(v.y), "f"(v.x));
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(o.y) : "f"(v.w), "f"(v.z));
    dst[i] = o;
  }
}

extern "C" int estk_shadow_bf16(estk_ctx* ctx, const float* src, uint16_t* dst, int64_t n, void* stream) {
  ESTK_CHECK_ARG(ctx && src && dst && n > 0 && (n % 4) == 0, "estk_shadow_bf16: null argument or n not a multiple of 4");
  ESTK_CHECK_ARG(ESTK_ALIGNED16(src) && ((uintptr_t)dst & 7u) == 0, "estk_shadow_bf16: unaligned buffers");
  int blocks = (int)((n / 4 + 255) / 256);
  if (blocks > ctx->sm_count * 16) blocks = ctx->sm_count * 16;
  shadow_bf16_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4*>(src),
                                                             reinterpret_cast<uint2*>(dst), n / 4);
  ESTK_CUDA(cudaGetLastError());
  return ESTK_OK;
}

// ---- fp16 operands from fp32 theta + the exact 16-bit noise table (the default tensor-core mode).
__global__ void __launch_bounds__(256) shadow_f16_kernel(const float4* __restrict__ src, uint2* __restrict__ dst, int64_t n4,
                                                         unsigned long long* __restrict__ inexact) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  unsigned int bad = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 v = src[i];
    const __half2 a = __floats2half2_rn(v.x, v.y), b = __floats2half2_rn(v.z, v.w);
    const float2 fa = __half22float2(a), fb = __half22float2(b);
    bad += (fa.x != v.x) + (fa.y != v.y) + (fb.x != v.z) + (fb.y != v.w);
    uint2 o;
    o.x = *reinterpret_cast<const uint32_t*>(&a);
    o.y = *reinterpret_cast<const uint32_t*>(&b);
    dst[i] = o;
  }
  if (inexact && bad) atomicAdd(inexact, (unsigned long long)bad);
}

extern "C" int estk_shadow_f16(estk_ctx* ctx, const float* src, uint16_t* dst, int64_t n, uint64_t* inexact_count,
                               void* stream) {
  ESTK_CHECK_ARG(ctx && src && dst && n > 0 && (n % 4) == 0, "estk_shadow_f16: null argument or n not a multiple of 4");
  ESTK_CHECK_ARG(ESTK_ALIGNED16(src) && ((uintptr_t)dst & 7u) == 0, "estk_shadow_f16: unaligned buffers");
  int blocks = (int)((n / 4 + 255) / 256);
  if (blocks > ctx->sm_count * 16) blocks = ctx->sm_count * 16;
  shadow_f16_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4*>(src),
                                                            reinterpret_cast<uint2*>(dst), n / 4,
                                                            reinterpret_cast<unsigned long long*>(inexact_count));
  ESTK_CUDA(cudaGetLastError());
  return ESTK_OK;
}

#ifdef ESTK_TC_PROFILE
// Profile build only: the next evaluate launches write their per-warp buckets into `buf` (null: off);
// reports the block's warp count and how many of them are consumers.
extern "C" ESTK_API int estk_tc_profile(void* buf, int32_t* warps, int32_t* consumer_warps) {
  g_prof_buf = static_cast<unsigned long long*>(buf);
  *warps = kThreadsTC / 32;
  *consumer_warps = 4 * kConsWG;
  return kPrBuckets;
}
#endif

extern "C" int estk_eval_mlp_supported(const estk_mlp_desc* desc, int32_t precision, int32_t B) {
  const char* why = "";
  if (desc && precision == ESTK_PREC_F16_ANY) return eval_mlp_tc_stream_supported(*desc, B, &why);
  const int mode = mode_of(precision);
  return desc && mode >= 0 ? tc_supported(*desc, B, &why, mode) : 0;
}
