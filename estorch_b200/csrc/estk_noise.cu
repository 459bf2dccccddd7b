// estk_noise.cu -- noise table fill, per-generation row offsets, row materialisation.
//
// Replaces the reference's per-generation `Normal(0, sigma).sample([P/2, n])`
// + two `torch.cat`s (estorch/estorch.py:187-193, 96 % of its generation time)
// by indexing a shared, device-resident unit-normal table.
#include "estk_common.cuh"
#include "estk_sort.cuh"
#include <cooperative_groups.h>
#include <cuda_fp16.h>

// ------------------------------------------------------------------ Philox
#define PHILOX_M0 0xD2511F53u
#define PHILOX_M1 0xCD9E8D57u
#define PHILOX_W0 0x9E3779B9u
#define PHILOX_W1 0xBB67AE85u

__device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                              uint32_t k0, uint32_t k1, uint32_t out[4]) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(PHILOX_M0, c0), lo0 = PHILOX_M0 * c0;
    const uint32_t hi1 = __umulhi(PHILOX_M1, c2), lo1 = PHILOX_M1 * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
    c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
    k0 += PHILOX_W0; k1 += PHILOX_W1;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

__device__ __forceinline__ float u01(uint32_t x) {
  return __fmul_rn(__fadd_rn((float)(x >> 8), 0.5f), 5.9604644775390625e-08f);  // 2^-24
}

__global__ void __launch_bounds__(256) fill_noise_kernel(float4* __restrict__ table4, int64_t n4,
                                                         uint32_t k0, uint32_t k1) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < n4; c += stride) {
    uint32_t x[4];
    philox4x32_10((uint32_t)c, (uint32_t)((uint64_t)c >> 32), 0u, 0u, k0, k1, x);
    float4 o;
    {
      const float r = sqrtf(__fmul_rn(-2.0f, logf(u01(x[0]))));
      float s, co;
      sincosf(__fmul_rn(6.283185307179586f, u01(x[1])), &s, &co);
      o.x = __fmul_rn(r, co); o.y = __fmul_rn(r, s);
    }
    {
      const float r = sqrtf(__fmul_rn(-2.0f, logf(u01(x[2]))));
      float s, co;
      sincosf(__fmul_rn(6.283185307179586f, u01(x[3])), &s, &co);
      o.z = __fmul_rn(r, co); o.w = __fmul_rn(r, s);
    }
    // every entry is rounded to the nearest fp16-representable value (11 significant bits: plenty for a
    // random number), so that the 16-bit copy the evaluate kernel streams (estk_shadow_f16) is EXACT
    o.x = __half2float(__float2half_rn(o.x)); o.y = __half2float(__float2half_rn(o.y));
    o.z = __half2float(__float2half_rn(o.z)); o.w = __half2float(__float2half_rn(o.w));
    table4[c] = o;
  }
}

extern "C" int estk_fill_noise_table(estk_ctx* ctx, float* table, int64_t len, uint64_t seed,
                                     void* stream) {
  ESTK_CHECK_ARG(ctx && table, "estk_fill_noise_table: null argument");
  ESTK_CHECK_ARG(len > 0 && (len % 4) == 0, "estk_fill_noise_table: len %lld must be a positive multiple of 4", (long long)len);
  ESTK_CHECK_ARG(ESTK_ALIGNED16(table), "estk_fill_noise_table: table must be 16-byte aligned");
  const int64_t n4 = len / 4;
  int blocks = (int)((n4 + 255) / 256);
  if (blocks > ctx->sm_count * 16) blocks = ctx->sm_count * 16;
  fill_noise_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>((float4*)table, n4, (uint32_t)seed,
                                                              (uint32_t)(seed >> 32));
  ESTK_CUDA(cudaGetLastError());
  return ESTK_OK;
}

// ------------------------------------------------------------------ offsets
// Hash every local pair to a 128-byte-aligned table slot; pair i's slot depends on (seed, generation,
// pair_begin + i) only.
__device__ __forceinline__ uint64_t pair_slot(uint64_t base, int64_t pair_begin, int i, uint64_t nslots) {
  return estk_mix64(base + (uint64_t)(pair_begin + i)) % nslots;
}

__device__ __forceinline__ uint64_t offsets_base(uint64_t seed, const estk_state* state, int64_t gen_host) {
  const uint64_t gen = (uint64_t)((state ? state->generation : 0) + gen_host);
  return estk_mix64(seed ^ (gen * ESTK_GEN_MUL));
}

// Offsets only (no evaluation order requested).
__global__ void __launch_bounds__(1024) make_offsets_kernel(uint64_t seed, const estk_state* state,
                                                            int64_t gen_host, int64_t pair_begin,
                                                            int pairs, uint64_t nslots,
                                                            int64_t* __restrict__ offsets_out) {
  const uint64_t base = offsets_base(seed, state, gen_host);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < pairs; i += gridDim.x * blockDim.x)
    offsets_out[i] = (int64_t)(pair_slot(base, pair_begin, i, nslots) * 32ull);
}

// More than kBucketSortMax pairs: one cooperative grid hashes the offsets and sorts (slot, local index)
// with the grid-wide stable radix sort (estk_sort.cuh).  The input is in index order, so equal slots
// keep index order: the unique order by (offset, index), as the bucket kernel gives below.
constexpr int kOffsetsSortThreads = 512;
__global__ void __launch_bounds__(kOffsetsSortThreads) make_offsets_sort_kernel(
    uint64_t seed, const estk_state* state, int64_t gen_host, int64_t pair_begin, int pairs, uint64_t nslots,
    int slot_bits, int64_t* __restrict__ offsets_out, int32_t* __restrict__ order_out, const estk_sort::Workspace ws) {
  extern __shared__ __align__(16) uint32_t s_sort[];
  cooperative_groups::grid_group grid = cooperative_groups::this_grid();
  const uint64_t base = offsets_base(seed, state, gen_host);
  const int gthreads = gridDim.x * kOffsetsSortThreads;
  for (int i = blockIdx.x * kOffsetsSortThreads + threadIdx.x; i < pairs; i += gthreads)
    offsets_out[i] = (int64_t)(pair_slot(base, pair_begin, i, nslots) * 32ull);
  auto load = [&](int i) { return (unsigned long long)pair_slot(base, pair_begin, i, nslots); };
  const int b = estk_sort::grid_sort<unsigned long long, kOffsetsSortThreads>(grid, ws, pairs, slot_bits, load, s_sort);
  for (int s = blockIdx.x * kOffsetsSortThreads + threadIdx.x; s < pairs; s += gthreads)
    order_out[s] = (int32_t)__ldcg((b ? ws.vals[1] : ws.vals[0]) + s);
}

// Up to 4096 pairs: one CTA, ~6 block-wide steps.  The slots are uniform hashes, so a bucket per expected key (bucket = slot * NB / nslots, monotone in the key) holds
// ~1 key; count, scan, scatter, then every bucket's handful of keys is put in order by one thread.  The result
// is the unique sorted order of the (offset << 16 | index) keys, the same order the radix sort gives above.
constexpr int kBucketSortMax = 4096;
__global__ void __launch_bounds__(1024) make_offsets_bucket_kernel(uint64_t seed, const estk_state* state,
                                                                   int64_t gen_host, int64_t pair_begin,
                                                                   int pairs, uint64_t nslots,
                                                                   int64_t* __restrict__ offsets_out,
                                                                   int32_t* __restrict__ order_out, int nb) {
  extern __shared__ uint64_t sorted[];                       // [nb] keys in bucket order
  uint32_t* count = reinterpret_cast<uint32_t*>(sorted + nb);   // [nb] keys per bucket, then exclusive starts
  __shared__ uint32_t warp_tot[32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int kPer = kBucketSortMax / 1024;                // keys (and buckets) per thread
  const uint64_t gen = (uint64_t)((state ? state->generation : 0) + gen_host);
  const uint64_t base = estk_mix64(seed ^ (gen * ESTK_GEN_MUL));
  for (int b = tid; b < nb; b += 1024) count[b] = 0u;
  __syncthreads();
  uint64_t key[kPer];
  uint32_t bucket[kPer], slot_in[kPer];
#pragma unroll
  for (int e = 0; e < kPer; ++e) {
    const int i = tid + e * 1024;
    if (i < pairs) {
      const uint64_t slot = estk_mix64(base + (uint64_t)(pair_begin + i)) % nslots;
      const uint64_t off = slot * 32ull;
      offsets_out[i] = (int64_t)off;
      key[e] = (off << 16) | (uint64_t)i;
      bucket[e] = (uint32_t)((slot * (uint64_t)nb) / nslots);
      slot_in[e] = atomicAdd(&count[bucket[e]], 1u);
    }
  }
  __syncthreads();
  // exclusive scan of count[0..nb): kPer consecutive buckets per thread, warp scan, scan of the warp totals
  uint32_t mine[kPer], run = 0;
#pragma unroll
  for (int e = 0; e < kPer; ++e) {
    const int b = tid * kPer + e;
    mine[e] = b < nb ? count[b] : 0u;
    run += mine[e];
  }
  uint32_t incl = run;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t up = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += up;
  }
  if (lane == 31) warp_tot[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    uint32_t t = warp_tot[lane], ti = t;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t up = __shfl_up_sync(0xffffffffu, ti, d);
      if (lane >= d) ti += up;
    }
    warp_tot[lane] = ti - t;                                  // exclusive
  }
  __syncthreads();
  uint32_t start = warp_tot[warp] + incl - run;
  uint32_t first[kPer];
#pragma unroll
  for (int e = 0; e < kPer; ++e) {
    const int b = tid * kPer + e;
    first[e] = start;
    if (b < nb) count[b] = start;                             // count[] now holds the bucket starts
    start += mine[e];
  }
  __syncthreads();
#pragma unroll
  for (int e = 0; e < kPer; ++e)
    if (tid + e * 1024 < pairs) sorted[count[bucket[e]] + slot_in[e]] = key[e];
  __syncthreads();
  // order inside each bucket (insertion sort of a handful of keys; the buckets are disjoint segments)
#pragma unroll
  for (int e = 0; e < kPer; ++e) {
    const uint32_t lo = first[e], c = mine[e];
    for (uint32_t a = 1; a < c; ++a) {
      const uint64_t k = sorted[lo + a];
      uint32_t q = a;
      while (q > 0 && sorted[lo + q - 1] > k) { sorted[lo + q] = sorted[lo + q - 1]; --q; }
      sorted[lo + q] = k;
    }
  }
  __syncthreads();
  for (int i = tid; i < pairs; i += 1024) order_out[i] = (int32_t)(sorted[i] & 0xFFFFull);
}

extern "C" int estk_make_offsets(estk_ctx* ctx, uint64_t seed, const estk_state* state,
                                 int64_t gen_host, int64_t pair_begin, int32_t pairs,
                                 int64_t table_len, int64_t n, int64_t* offsets_out,
                                 int32_t* order_out, void* stream) {
  ESTK_CHECK_ARG(ctx && offsets_out, "estk_make_offsets: null argument");
  ESTK_CHECK_ARG(pairs > 0 && pairs <= ESTK_MAX_POPULATION / 2, "estk_make_offsets: pairs=%d out of range", pairs);
  ESTK_CHECK_ARG(n > 0 && pair_begin >= 0, "estk_make_offsets: bad n/pair_begin");
  const int64_t n_pad = (n + 31) / 32 * 32;
  ESTK_CHECK_ARG(table_len >= n_pad, "estk_make_offsets: table_len %lld < padded row %lld", (long long)table_len, (long long)n_pad);
  ESTK_CHECK_ARG(table_len <= ESTK_MAX_TABLE_LEN, "estk_make_offsets: table of %lld entries is longer than %lld",
                 (long long)table_len, (long long)ESTK_MAX_TABLE_LEN);
  const uint64_t nslots = (uint64_t)((table_len - n_pad) / 32 + 1);
  if (order_out && pairs <= kBucketSortMax) {
    int sort_len = 1;
    while (sort_len < pairs) sort_len <<= 1;
    const int nb = sort_len < 32 ? 32 : sort_len;
    if ((size_t)nb * 12 > 40 * 1024)
      ESTK_CUDA(cudaFuncSetAttribute(make_offsets_bucket_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     kBucketSortMax * 12));
    make_offsets_bucket_kernel<<<1, 1024, (size_t)nb * 12, (cudaStream_t)stream>>>(
        seed, state, gen_host, pair_begin, pairs, nslots, offsets_out, order_out, nb);
    ESTK_CUDA(cudaGetLastError());
    return ESTK_OK;
  }
  if (!order_out) {
    int blocks = (pairs + 1023) / 1024;
    if (blocks > ctx->sm_count * 4) blocks = ctx->sm_count * 4;
    make_offsets_kernel<<<blocks, 1024, 0, (cudaStream_t)stream>>>(seed, state, gen_host, pair_begin, pairs, nslots,
                                                                  offsets_out);
    ESTK_CUDA(cudaGetLastError());
    return ESTK_OK;
  }
  // 8-byte slot keys for `pairs` elements: the sort buffers of 2 * pairs members
  const int rc = estk_ctx_reserve(ctx, 2 * (int64_t)pairs, 0, (cudaStream_t)stream, "estk_make_offsets");
  if (rc) return rc;
  int slot_bits = 0;
  while (slot_bits < 64 && ((nslots - 1) >> slot_bits) != 0) ++slot_bits;
  constexpr size_t kSmem = estk_sort::smem_bytes(kOffsetsSortThreads);
  int occ = 0;
  ESTK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, make_offsets_sort_kernel, kOffsetsSortThreads, kSmem));
  if (occ < 1) {
    estk_set_error("make_offsets_sort_kernel cannot be resident");
    return ESTK_ERR_CUDA;
  }
  int grid = (pairs + kOffsetsSortThreads - 1) / kOffsetsSortThreads;
  if (grid > occ * ctx->sm_count) grid = occ * ctx->sm_count;
  if (grid > ctx->max_grid) grid = ctx->max_grid;
  const estk_sort::Workspace ws = estk_sort::workspace_of(ctx);
  void* args[] = {&seed, (void*)&state, &gen_host, &pair_begin, &pairs, (void*)&nslots, &slot_bits, &offsets_out,
                  &order_out, (void*)&ws};
  ESTK_CUDA(cudaLaunchCooperativeKernel((void*)make_offsets_sort_kernel, dim3(grid), dim3(kOffsetsSortThreads), args,
                                        kSmem, (cudaStream_t)stream));
  return ESTK_OK;
}

// ------------------------------------------------------------------ rows
// population_parameters / epsilon rows exactly as estorch.py:189-193 builds
// them: eps = sigma * t (one rounding), row = theta +- eps (second rounding).
__global__ void __launch_bounds__(256) perturb_rows_kernel(const float* __restrict__ theta, int64_t n,
                                                           const float* __restrict__ table,
                                                           const int64_t* __restrict__ offsets,
                                                           int pairs, float sigma, int member_begin,
                                                           float* __restrict__ rows_out,
                                                           float* __restrict__ eps_out) {
  const int mloc = blockIdx.y;
  const int member = member_begin + mloc;
  const bool minus = member >= pairs;
  const int j = minus ? member - pairs : member;
  const float* trow = table + offsets[j];
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += stride) {
    float e = __fmul_rn(sigma, ld_noise1(trow + k));
    if (minus) e = -e;
    if (rows_out) rows_out[(int64_t)mloc * n + k] = __fadd_rn(theta[k], e);
    if (eps_out) eps_out[(int64_t)mloc * n + k] = e;
  }
}

extern "C" int estk_perturb_rows(estk_ctx* ctx, const float* theta, int64_t n, const float* table,
                                 const int64_t* offsets, int32_t pairs, float sigma,
                                 int32_t member_begin, int32_t member_count, float* rows_out,
                                 float* eps_out, void* stream) {
  ESTK_CHECK_ARG(ctx && theta && table && offsets, "estk_perturb_rows: null argument");
  ESTK_CHECK_ARG(rows_out || eps_out, "estk_perturb_rows: no output requested");
  ESTK_CHECK_ARG(n > 0 && pairs > 0, "estk_perturb_rows: bad n/pairs");
  ESTK_CHECK_ARG(member_begin >= 0 && member_count > 0 && member_begin + member_count <= 2 * pairs,
                 "estk_perturb_rows: members [%d,+%d) outside population of %d", member_begin, member_count, 2 * pairs);
  ESTK_CHECK_ARG(member_count <= 65535, "estk_perturb_rows: at most 65535 rows per call");
  int bx = (int)((n + 255) / 256);
  if (bx > 1024) bx = 1024;
  dim3 grid(bx, member_count);
  perturb_rows_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(theta, n, table, offsets, pairs, sigma,
                                                              member_begin, rows_out, eps_out);
  ESTK_CUDA(cudaGetLastError());
  return ESTK_OK;
}
