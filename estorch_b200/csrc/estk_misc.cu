// estk_misc.cu -- best-policy tracking and novelty (k-nearest-neighbour) kernels.
#include "estk_common.cuh"

// ------------------------------------------------------------------ best tracking
// estorch/estorch.py:181-185 `_after_optimize`: episode_reward = rollout(policy);
// if it beats best_reward, keep it and snapshot the parameters (the reference
// deep-copies state_dict(); here theta -> best_theta on the device), then
// `self.step += 1` (:248).  Every thread evaluates the same predicate from the
// same two scalars, thread 0 of block 0 publishes the new state afterwards.
__global__ void __launch_bounds__(256) track_best_kernel(estk_state* state, const float* __restrict__ reward,
                                                         const float* __restrict__ theta,
                                                         float* __restrict__ best_theta, int64_t n,
                                                         unsigned int* ticket) {
  const float r = __ldg(reward);
  const bool better = r > state->best_reward;          // read by every CTA before it takes a ticket
  if (better) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += stride)
      best_theta[k] = theta[k];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(ticket, 1u) == gridDim.x - 1) {       // last CTA: publish the new state
      state->episode_reward = r;
      if (better) state->best_reward = r;
      state->improved = better ? 1 : 0;
      state->generation += 1;
      *ticket = 0u;
    }
  }
}

extern "C" int estk_track_best(estk_ctx* ctx, estk_state* state, const float* reward,
                               const float* theta, float* best_theta, int64_t n, void* stream) {
  ESTK_CHECK_ARG(ctx && state && reward && theta && best_theta && n > 0, "estk_track_best: bad argument");
  int blocks = (int)((n + 255) / 256);
  if (blocks > ctx->sm_count * 4) blocks = ctx->sm_count * 4;
  track_best_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(state, reward, theta, best_theta, n,
                                                             ctx->counters + kTicketTrackBest);
  ESTK_CUDA(cudaGetLastError());
  return ESTK_OK;
}

// ------------------------------------------------------------------ novelty
// estorch/estorch.py:412-417: kd = cKDTree(archive); d,_ = kd.query(bc, k);
// d = d[d < inf]; novelty = sum(d) / np.linalg.norm(archive).  Brute force in
// fp64 (scipy works in float64): one warp per behaviour characteristic.
__global__ void __launch_bounds__(256) frob_kernel(const float* __restrict__ a, int64_t count,
                                                   double* __restrict__ out) {
  __shared__ double s[8];
  double acc = 0.0;
  for (int64_t i = threadIdx.x; i < count; i += blockDim.x) {
    const double x = (double)a[i];
    acc += x * x;
  }
  acc = warp_sum_d(acc);
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < 8; ++w) t += s[w];
    out[0] = sqrt(t);
  }
}

constexpr int kMaxK = 32;

__global__ void __launch_bounds__(256) knn_novelty_kernel(const float* __restrict__ bc, int count,
                                                          const float* __restrict__ archive, int A,
                                                          int dim, int k,
                                                          const double* __restrict__ frob,
                                                          float* __restrict__ out) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= count) return;
  const float* q = bc + (size_t)warp * dim;
  double best[kMaxK];  // ascending; only lane 0's copy is meaningful
  int have = 0;
  for (int a = 0; a < A; ++a) {
    const float* row = archive + (size_t)a * dim;
    double acc = 0.0;
    for (int d = lane; d < dim; d += 32) {
      const double diff = (double)row[d] - (double)q[d];
      acc += diff * diff;
    }
    acc = warp_sum_d(acc);
    if (lane == 0) {
      const double dist = sqrt(acc);
      if (have < k) {
        int i = have++;
        while (i > 0 && best[i - 1] > dist) { best[i] = best[i - 1]; --i; }
        best[i] = dist;
      } else if (dist < best[k - 1]) {
        int i = k - 1;
        while (i > 0 && best[i - 1] > dist) { best[i] = best[i - 1]; --i; }
        best[i] = dist;
      }
    }
  }
  if (lane == 0) {
    double s = 0.0;
    for (int i = 0; i < have; ++i) s += best[i];
    out[warp] = (float)(s / frob[0]);
  }
}

extern "C" int estk_knn_novelty(estk_ctx* ctx, const float* bc, int32_t count, const float* archive,
                                int32_t archive_len, int32_t dim, int32_t k, float* novelty_out,
                                void* stream) {
  ESTK_CHECK_ARG(ctx && bc && archive && novelty_out, "estk_knn_novelty: null argument");
  ESTK_CHECK_ARG(count > 0 && archive_len > 0 && dim > 0, "estk_knn_novelty: bad sizes");
  ESTK_CHECK_ARG(k >= 1 && k <= kMaxK, "estk_knn_novelty: k=%d must be in [1,%d]", k, kMaxK);
  frob_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(archive, (int64_t)archive_len * dim, ctx->scalars);
  ESTK_CUDA(cudaGetLastError());
  const int warps_per_block = 8;
  const int blocks = (count + warps_per_block - 1) / warps_per_block;
  knn_novelty_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(bc, count, archive, archive_len, dim, k,
                                                               ctx->scalars, novelty_out);
  ESTK_CUDA(cudaGetLastError());
  return ESTK_OK;
}
