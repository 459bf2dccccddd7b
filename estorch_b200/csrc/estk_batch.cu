// estk_batch.cu -- minibatch selection on the device: the rows of generation g's batch (a keyed permutation of
// the dataset per epoch, include/estk_batch.h states the construction) gathered into the evaluate's batch buffers.
//
// One launch at the head of a captured generation: the generation index is read from estk_state, so a replayed
// graph draws the next batch, and every rank draws the same one.
#include "estk_common.cuh"
#include "estk_batch.h"

#define ESTK_BATCH_SALT 0x6261746368657321ull   // "batches!": keeps the epoch keys apart from the offsets' bases

// (seed, epoch) -> the 4 round keys of that epoch's Feistel network
__host__ __device__ __forceinline__ void batch_round_keys(uint64_t seed, uint64_t epoch, uint64_t k[4]) {
  const uint64_t ke = estk_mix64(estk_mix64(seed ^ ESTK_BATCH_SALT) + epoch);
#pragma unroll
  for (int r = 0; r < 4; ++r) k[r] = estk_mix64(ke + (uint64_t)r);
}

// pi_e(x) for x in [0, n): 4 Feistel rounds over 2h bits (h bits per half), cycle-walked back into [0, n)
__host__ __device__ __forceinline__ uint64_t batch_permute(uint64_t x, uint64_t n, int h, const uint64_t k[4]) {
  const uint64_t mask = (1ull << h) - 1ull;
  do {
    uint64_t L = x >> h, R = x & mask;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const uint64_t f = estk_mix64(k[r] ^ R) & mask;
      const uint64_t t = L ^ f;
      L = R;
      R = t;
    }
    x = (L << h) | R;
  } while (x >= n);
  return x;
}

// the smallest h >= 1 with 2^(2h) >= n
static inline int batch_half_bits(int64_t n) {
  int h = 1;
  while ((1ll << (2 * h)) < n) ++h;
  return h;
}

struct SampleBatchArgs {
  uint64_t seed;
  const estk_state* state;
  int64_t gen_host;
  int64_t n;
  int32_t batch;
  int h;
  const float* obs_src;
  int64_t obs_row;
  float* obs_dst;
  const float* tgt_src;
  int64_t tgt_row;
  float* tgt_dst;
  int64_t* index_out;
};

// One row of `row` floats from src to dst by `lanes` threads: 16-byte vectors where both rows are 16-byte
// aligned and the row is a multiple of 4 floats, else 8-byte pairs where both are 8-byte aligned and the row is
// even, else single floats.  The bytes are copied as they are (no arithmetic).
__device__ __forceinline__ void copy_row(const float* __restrict__ src, float* __restrict__ dst, int64_t row,
                                         int lane, int lanes) {
  const uintptr_t a = (uintptr_t)src | (uintptr_t)dst;
  if ((a & 15u) == 0 && (row & 3) == 0) {
    const float4* s = reinterpret_cast<const float4*>(src);
    float4* d = reinterpret_cast<float4*>(dst);
    for (int64_t i = lane; i < row / 4; i += lanes) d[i] = __ldg(s + i);
  } else if ((a & 7u) == 0 && (row & 1) == 0) {
    const float2* s = reinterpret_cast<const float2*>(src);
    float2* d = reinterpret_cast<float2*>(dst);
    for (int64_t i = lane; i < row / 2; i += lanes) d[i] = __ldg(s + i);
  } else {
    for (int64_t i = lane; i < row; i += lanes) dst[i] = __ldg(src + i);
  }
}

// A group of LANES threads per batch row (grid-stride over rows).  Every thread of the group computes the row's
// index itself: the same integer work in lock-step, no shared memory and no barrier.
template <int LANES>
__global__ void __launch_bounds__(128) sample_batch_kernel(const SampleBatchArgs p) {
  const uint64_t g = (uint64_t)((p.state ? p.state->generation : 0) + p.gen_host);
  const uint64_t n = (uint64_t)p.n, B = (uint64_t)p.batch;
  // p = g*B + j without a 128-bit product: g*B = (g div n)*n*B + (g mod n)*B, and (g mod n)*B < 2^62
  const uint64_t gm = (g % n) * B;
  const uint64_t e0 = (g / n) * B + gm / n, r0 = gm % n;
  uint64_t k0[4], k1[4];
  batch_round_keys(p.seed, e0, k0);
  batch_round_keys(p.seed, e0 + 1, k1);
  const int lane = threadIdx.x % LANES;
  const int64_t groups = (int64_t)gridDim.x * (128 / LANES);
  for (int64_t j = (int64_t)blockIdx.x * (128 / LANES) + threadIdx.x / LANES; j < p.batch; j += groups) {
    uint64_t r = r0 + (uint64_t)j;                 // < 2n: the batch spans epochs e0 and e0 + 1 at most
    const bool next = r >= n;
    if (next) r -= n;
    uint64_t k[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) k[q] = next ? k1[q] : k0[q];   // selects registers (no indexed local array)
    const int64_t idx = (int64_t)batch_permute(r, n, p.h, k);
    if (lane == 0 && p.index_out) p.index_out[j] = idx;
    copy_row(p.obs_src + idx * p.obs_row, p.obs_dst + j * p.obs_row, p.obs_row, lane, LANES);
    copy_row(p.tgt_src + idx * p.tgt_row, p.tgt_dst + j * p.tgt_row, p.tgt_row, lane, LANES);
  }
}

extern "C" int estk_sample_batch(estk_ctx* ctx, uint64_t seed, const estk_state* state, int64_t gen_host,
                                 int64_t n_rows, int32_t batch, const float* obs_src, int64_t obs_row_floats,
                                 float* obs_dst, const float* tgt_src, int64_t tgt_row_floats, float* tgt_dst,
                                 int64_t* index_out, void* stream) {
  ESTK_CHECK_ARG(ctx, "estk_sample_batch: null context");
  ESTK_CHECK_ARG(obs_src && obs_dst && tgt_src && tgt_dst, "estk_sample_batch: null source or destination");
  ESTK_CHECK_ARG(n_rows > 0 && n_rows < (1ll << 31), "estk_sample_batch: n_rows=%lld outside [1, 2^31)",
                 (long long)n_rows);
  ESTK_CHECK_ARG(batch > 0 && batch <= n_rows, "estk_sample_batch: batch=%d outside [1, n_rows=%lld]", batch,
                 (long long)n_rows);
  ESTK_CHECK_ARG(obs_row_floats > 0 && tgt_row_floats > 0, "estk_sample_batch: row sizes must be positive");
  ESTK_CHECK_ARG(gen_host >= 0, "estk_sample_batch: gen_host=%lld is negative", (long long)gen_host);
  SampleBatchArgs a{seed, state, gen_host, n_rows, batch, batch_half_bits(n_rows), obs_src, obs_row_floats,
                    obs_dst, tgt_src, tgt_row_floats, tgt_dst, index_out};
  // rows of up to 1024 floats: a warp each; longer ones: the whole CTA
  const bool wide = obs_row_floats > 1024 || tgt_row_floats > 1024;
  const int per_cta = wide ? 1 : 4;
  int64_t blocks = ((int64_t)batch + per_cta - 1) / per_cta;
  if (blocks > (int64_t)ctx->sm_count * 16) blocks = (int64_t)ctx->sm_count * 16;
  if (wide)
    sample_batch_kernel<128><<<(unsigned)blocks, 128, 0, (cudaStream_t)stream>>>(a);
  else
    sample_batch_kernel<32><<<(unsigned)blocks, 128, 0, (cudaStream_t)stream>>>(a);
  ESTK_CUDA(cudaGetLastError());
  return ESTK_OK;
}
