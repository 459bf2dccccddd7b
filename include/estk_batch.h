/*
 * estk_batch.h -- minibatches drawn on the device: the sampler entry point of libestk.so.
 *
 * A companion of estk.h (whose types, status codes and conventions it uses), declared apart from the
 * ABI-200 core so that the core's symbol set stays fixed; libestk.so exports both.
 */
#ifndef ESTK_BATCH_H_
#define ESTK_BATCH_H_

#include "estk.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Gather generation g's minibatch of a device-resident dataset: obs_dst[j] = obs_src[idx_j] and
 * tgt_dst[j] = tgt_src[idx_j] for j in [0, batch), rows of obs_row_floats / tgt_row_floats floats, copied
 * byte for byte in batch order; index_out (nullable, int64 [batch]) receives idx_j.  Only the chosen rows
 * are read.  g = gen_host, plus state->generation when `state` is non-null (the rule of estk_make_offsets:
 * a generation replayed from a CUDA graph passes a constant gen_host and draws the next batch).
 *
 * With N = n_rows and B = batch, generation g takes the positions p = g*B + j (exact integers) of the
 * stream pi_0, pi_1, ..., each pi_e a permutation of [0, N): idx_j = pi_e(r), e = p div N, r = p mod N.
 * So every epoch visits every row exactly once, and a batch repeats a row only where it straddles two
 * epochs.  pi_e, in uint64 arithmetic with mix64 the splitmix64 finaliser of estk_make_offsets:
 *   h = the smallest h >= 1 with 2^(2h) >= N; mask = 2^h - 1;
 *   K_e = mix64(mix64(seed ^ 0x6261746368657321) + e); k_r = mix64(K_e + r) for r = 0..3;
 *   F(x): L = x >> h, R = x & mask; four rounds (L, R) <- (R, L ^ (mix64(k_r ^ R) & mask)); (L << h) | R;
 *   pi_e(r) = the first of F(r), F(F(r)), ... that is < N (cycle walking: F is a bijection of [0, 2^(2h))).
 * N <= 0 or N >= 2^31, batch <= 0 or batch > N, a row size <= 0, a NULL context, source or destination,
 * and gen_host < 0 are ESTK_ERR_INVALID before any launch. */
ESTK_API int estk_sample_batch(estk_ctx* ctx, uint64_t seed, const estk_state* state, int64_t gen_host,
                      int64_t n_rows, int32_t batch,
                      const float* obs_src, int64_t obs_row_floats, float* obs_dst,
                      const float* tgt_src, int64_t tgt_row_floats, float* tgt_dst,
                      int64_t* index_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ESTK_BATCH_H_ */
