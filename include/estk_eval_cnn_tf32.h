/*
 * estk_eval_cnn_tf32.h -- the convolutional evaluate of estk.h (Conv2d stack, flatten, Linear head) on TF32
 * tensor cores: every perturbed member's return on a fixed batch of B images.
 *
 * A companion of estk.h (whose types, status codes, packed CNN descriptor and conventions it uses), declared
 * apart from the ABI-200 core so that the core's symbol set and precision codes stay fixed; libestk.so exports
 * both.  estk_eval_mlp's convolutional route stays fp32 only.
 */
#ifndef ESTK_EVAL_CNN_TF32_H_
#define ESTK_EVAL_CNN_TF32_H_

#include "estk.h"

#ifdef __cplusplus
extern "C" {
#endif

/* desc: the packing of the convolutional evaluate of estk.h, unchanged: dims[0] = ESTK_CNN_INPUT(c, h, w), then
 * ESTK_CNN_CONV(out_c, k, stride, pad) per conv, then the Linear widths; activation bits 24-31 hold n_conv
 * (1..7) and bits 0-23 one of the codes with a return: a hidden kind (ESTK_ACT_RELU, ESTK_ACT_TANH,
 * ESTK_ACT_ELU, ESTK_ACT_SILU, ESTK_ACT_LEAKY_RELU) with the identity output and the squared error, with
 * ESTK_ACT_OUT_TANH and the squared error, with ESTK_LOSS_XENT or with ESTK_LOSS_ACCURACY (20 codes per
 * n_conv).  The parameters are in parameters_to_vector order.  obs is [B][c][h][w] and target [B][out].
 *
 * Forms, as for estk_eval_mlp's convolutional evaluate: population (offsets != NULL): ret_plus[j] / ret_minus[j]
 * are the returns of W = theta + (sigma*t) and theta - (sigma*t), t the fp32 table row at offsets[j]; order
 * (nullable) affects the schedule only.  Centre (offsets == NULL): ret_plus[0] is theta's return; table, order,
 * sigma, ret_minus and bc_minus are not read and pairs is ignored.  bc_plus / bc_minus (both or neither, with
 * bc_obs, bc_dim > 0) receive policy(obs[:bc_obs]).flatten()[:bc_dim] per member.
 *
 * Arithmetic (per member, every layer, conv or Linear; a Linear is the 1x1 convolution of its flattened input):
 *   formed weight  W = fp32(theta +- fp32(sigma*t)), the fp32 evaluate's two roundings, then the operand
 *                  w = rna_tf32(W) (cvt.rna.tf32.f32: round to nearest, ties away from zero, to 11 significand
 *                  bits; the low 13 bits are zero).  Biases are formed the same way and NOT rounded.
 *   input operand  x = rna_tf32(v), v the image for layer 0 and the previous layer's fp32 activation otherwise
 *                  (taps in the zero padding are zeros).
 *   output         acc = the fp32 tensor-core accumulation (mma.sync m16n8k8 tf32) of w * x over the taps in
 *                  ascending (ci, kh, kw) order, in steps of 8 taps from 0, the same walk for every member,
 *                  image, position and launch; then y = acc + bias in fp32, then the hidden activation of
 *                  estk.h (or, for the last layer, identity / tanhf).  The product of two TF32 operands is exact
 *                  in fp32.
 *   return         the per-image loss of the fp32 evaluate (squared error, cross-entropy or accuracy, in column
 *                  order) summed over b in ascending order from 0, then the fp32 evaluate's return formula.
 * No float atomics: the same bits from run to run, with or without order, whatever chunking the launch picks;
 * sigma = 0 gives every member the centre's bits, and a member's return and outputs are the centre form's on
 * that member's parameter row (estk_perturb_rows).
 *
 * Shapes served: every descriptor the convolutional evaluate accepts whose largest layer output
 * (out_c * H' * W', or a Linear width) is at most 2^26 floats per image, at any B >= 1 and pairs
 * 1..ESTK_MAX_POPULATION/2.  The activations of a work item (one pair, a chunk of images) live in a per-CTA
 * slab of the context workspace, within 1 GB for the whole grid (ESTK_ERR_NOMEM under capture when it must grow).
 *
 * ESTK_ERR_INVALID before any launch, with nothing written, by the rules of the fp32 route: a NULL ctx, desc,
 * theta, obs, target or ret_plus; for a population a NULL table or ret_minus; bc_plus / bc_minus not both set
 * or both null, or bc_obs / bc_dim < 1 with them; B < 1 (or B >= 2^24 with the accuracy); pairs outside
 * 1..ESTK_MAX_POPULATION/2; n_conv outside 1..7; bits 0-23 other than the 20 codes above (ESTK_ACTIONS and the
 * recurrent cells included); every malformed packed field the convolutional evaluate refuses.
 * ESTK_ERR_UNSUPPORTED before any launch: a valid call whose shape is not served (above).
 * estk_eval_cnn_tf32_supported returns 1 exactly when such a call with a valid desc, code and B would not be
 * refused (0 for a NULL desc and for every call refused above that desc and B decide). */
ESTK_API int estk_eval_cnn_tf32(estk_ctx* ctx, const estk_mlp_desc* desc, const float* theta, const float* table,
                                const int64_t* offsets, const int32_t* order, int32_t pairs, float sigma,
                                const float* obs, const float* target, int32_t B,
                                float* ret_plus, float* ret_minus, float* bc_plus, float* bc_minus,
                                int32_t bc_obs, int32_t bc_dim, void* stream);
ESTK_API int estk_eval_cnn_tf32_supported(const estk_mlp_desc* desc, int32_t B);

#ifdef __cplusplus
}
#endif
#endif /* ESTK_EVAL_CNN_TF32_H_ */
