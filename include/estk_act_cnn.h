/*
 * estk_act_cnn.h -- population mode for convolutional policies: every perturbed member's outputs on its own
 * images, one launch per environment step.
 *
 * A companion of estk.h (whose types, status codes, packed CNN descriptor and conventions it uses), declared
 * apart from the ABI-200 core so that the core's symbol set stays fixed; libestk.so exports both.
 */
#ifndef ESTK_ACT_CNN_H_
#define ESTK_ACT_CNN_H_

#include "estk.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The policy of the convolutional evaluate of estk.h (Conv2d stack, flatten, Linear head) run on each
 * member's own observations, returning its outputs instead of a loss.
 *
 * desc: the packing of the convolutional evaluate, unchanged: dims[0] = ESTK_CNN_INPUT(c, h, w), then
 * ESTK_CNN_CONV(out_c, k, stride, pad) per conv, then the Linear widths; activation bits 24-31 hold n_conv
 * (1..7), bits 16-23 must be ESTK_ACTIONS, bits 8-15 are 0 (identity output) or ESTK_ACT_OUT_TANH, and bits
 * 0-7 are a hidden kind (ESTK_ACT_RELU, ESTK_ACT_TANH, ESTK_ACT_ELU, ESTK_ACT_SILU, ESTK_ACT_LEAKY_RELU):
 * 10 codes per n_conv.  The parameters are in parameters_to_vector order, as for the evaluate.
 *
 * Population form (offsets != NULL): obs is [2*pairs][B][c][h][w]; block j holds the images of the + member
 * of local pair j (W = theta + (sigma*t), t the table row at offsets[j]) and block pairs + j those of its
 * mirror (W = theta - (sigma*t)).  out_plus and out_minus are each [pairs][B][out], out the last Linear's
 * width.  order (nullable) affects the schedule only.  table is the fp32 noise table (there is no 16-bit
 * form of this call).
 * Centre form (offsets == NULL): obs is [B][c][h][w] and out_plus [B][out], computed for theta; table,
 * order, pairs, sigma and out_minus are not read, and nothing outside obs [B][c][h][w] and out_plus [B][out]
 * is read or written.
 *
 * Arithmetic, fp32, exactly that of the convolutional evaluate in estk.h: W = theta +- (sigma*t) with two
 * roundings; each output one fmaf chain from 0 over the taps in ascending (ci, kh, kw) order, taps in the
 * zero padding skipped; then + bias, then the hidden activation (tanhf for the Tanh output).  So when every
 * member is given the same B images, a member's outputs are bit for bit the behaviour characteristic that
 * estk_eval_mlp's convolutional evaluate writes for that member with bc_obs = B and bc_dim = B*out, in the
 * population and in the centre form; sigma = 0 gives every member the centre's bits.  A member's outputs never
 * depend on another member's images.  No float atomics: the same bits from run to run, with or without
 * order, whatever chunking the launch picks.  Offsets into obs and out are 64-bit: 2*pairs*B*c*h*w may
 * exceed 2^31.  The activations of a work item live in shared memory, or in a slab of the context workspace
 * for large images (grown like the evaluate's buffers: ESTK_ERR_NOMEM under capture when it must grow).
 *
 * ESTK_ERR_INVALID before any launch, with nothing written: a NULL ctx, desc, theta, obs or out_plus; for a
 * population a NULL table or out_minus; B < 1; for a population pairs outside 1..ESTK_MAX_POPULATION/2;
 * n_conv outside 1..7; bits 0-23 other than the 10 codes above (a loss field other than ESTK_ACTIONS, a
 * recurrent cell, ESTK_LOSS_XENT included); and every malformed packed field the convolutional evaluate
 * refuses, by the same rules (n_layers <= n_conv or > ESTK_MAX_LAYERS, zero channels or widths, pad >= k, a
 * conv larger than its padded input, more than 2^30 inputs, taps or outputs per image in one layer). */
ESTK_API int estk_act_cnn(estk_ctx* ctx, const estk_mlp_desc* desc,
                          const float* theta, const float* table,
                          const int64_t* offsets, const int32_t* order, int32_t pairs, float sigma,
                          const float* obs, int32_t B,
                          float* out_plus, float* out_minus, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ESTK_ACT_CNN_H_ */
