/*
 * estk.h -- C ABI of the H100 Evolution-Strategies kernel library (libestk.so).
 *
 * This is the drop-in boundary for the ES generation hot path of
 * goktug97/estorch (estorch/estorch.py:211-250, ES._master).  The reference has
 * no FFI layer of its own (pure Python); each entry point below names the
 * reference function(s) whose arithmetic it replaces.  The only caller is the
 * host-side mirror of the reference classes (estorch_b200/estorch.py) through
 * ctypes; INTEGRATION.md shows the binding a reference maintainer would add.
 *
 * Conventions
 *   - plain C: no C++ types, no exceptions, no torch types in any signature;
 *   - every function returns ESTK_OK (0) or a negative estk_status; the text of
 *     the last failure on the calling thread is estk_last_error();
 *   - all buffers are CALLER-OWNED DEVICE pointers (fp32 / int32 / int64,
 *     contiguous, 16-byte aligned) unless a parameter says "host";
 *   - every launch is asynchronous on the caller's stream (`stream` is a
 *     cudaStream_t passed as void*); the library does not synchronise, except
 *     that a call which grows the context workspace (below) waits on `stream`
 *     for the new buffers' zero fill;
 *   - the library keeps no global mutable state: one estk_ctx per device
 *     holds an opaque workspace (partial sums, centred-rank scratch, sort
 *     buffers, activation slabs of the streamed fp32 and F16_ANY evaluates).  It is sized for 32768 members at estk_ctx_create; an entry
 *     point that needs more grows it first, and returns ESTK_ERR_NOMEM instead
 *     when its stream is being captured into a CUDA graph -- run a
 *     configuration once before capturing it.  The buffers a growth replaces
 *     stay allocated until estk_ctx_destroy, so graphs captured earlier replay
 *     correctly (after 16 growths of one context the library waits for the
 *     device and frees them: re-capture graphs after that many); if the new
 *     allocation fails the context keeps its old buffers.
 *
 * Member / pair layout (estorch.py:190-193): population_size P = 2*pairs;
 * member j < pairs is theta + sigma*T[off_j : off_j+n], member j+pairs is
 * theta - sigma*T[off_j : off_j+n].  T is the shared unit-normal noise table.
 */
#ifndef ESTK_H_
#define ESTK_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define ESTK_API __attribute__((visibility("default")))
#else
#define ESTK_API
#endif

#define ESTK_VERSION 200          /* 0.2.0 */
#define ESTK_MAX_LAYERS 8
#define ESTK_MAX_POPULATION (1 << 22) /* P: 4,194,304 members */
/* Longest noise table (entries) every kernel reads correctly: 2^34 (64 GiB in fp32).  estk_make_offsets refuses
 * longer ones.  The fp32-table loop of estk_rank_grad* holds a row as its 32-bit float4 index offsets[j] / 4;
 * every other table reader addresses a row with 64-bit arithmetic. */
#define ESTK_MAX_TABLE_LEN (1ll << 34)

typedef enum {
  ESTK_OK = 0,
  ESTK_ERR_INVALID = -1,      /* bad argument (shape, alignment, null) */
  ESTK_ERR_CUDA = -2,         /* a CUDA runtime call failed */
  ESTK_ERR_UNSUPPORTED = -3,  /* valid request this build cannot serve */
  ESTK_ERR_NOMEM = -4
} estk_status;

typedef struct estk_ctx estk_ctx;

/* Device-resident per-run state (caller-owned, 32 bytes, zero-initialised by
 * the caller except best_reward = -inf).  Kept on the device so that a whole
 * generation can be replayed from a CUDA graph with no host-side scalars. */
typedef struct {
  int64_t generation;   /* estorch.py:248 `self.step`; read by estk_make_offsets,
                           advanced by estk_track_best */
  int64_t adam_step;    /* torch Adam `state['step']`; advanced by the Adam epilogue */
  float episode_reward; /* estorch.py:182 */
  float best_reward;    /* estorch.py:183-184 */
  int32_t improved;     /* 1 when the last estk_track_best took a new best */
  int32_t reserved;
} estk_state;

/* Policy description: Linear -> act -> ... -> Linear [-> out_act] over a flat
 * parameter vector in torch.nn.utils.parameters_to_vector order (weight [out,in]
 * row-major, then bias, per layer) -- examples/cartpole_es.py:6-20.
 *
 * `activation` is three bit fields:
 *   bits 0-7   hidden activation, applied after every Linear but the last:
 *              ESTK_ACT_RELU (0) max(y, 0), ESTK_ACT_TANH (1) tanh(y),
 *              ESTK_ACT_ELU (3) y > 0 ? y : expm1(y)             (torch.nn.ELU(), alpha = 1),
 *              ESTK_ACT_SILU (4) y / (1 + exp(-y))               (torch.nn.SiLU()),
 *              ESTK_ACT_LEAKY_RELU (5) y > 0 ? y : y * 0.01      (torch.nn.LeakyReLU(), slope 0.01);
 *              or a recurrent cell (one step with ESTK_ACTIONS, or the sequence evaluate; below):
 *              ESTK_CELL_GRU (8) torch.nn.GRUCell, ESTK_CELL_LSTM (9) torch.nn.LSTMCell;
 *              2, 6, 7 and every value above 9 are undefined (2 is kept unassigned: callers have
 *              used it as the example of a refused code);
 *   bits 8-15  output activation, applied after the last Linear, before the squared
 *              error and the behaviour characteristic: 0 identity, ESTK_ACT_OUT_TANH tanh(y);
 *   bits 16-23 the loss, i.e. what a member's return is:
 *              0 the squared error, return = -sum_bc (y_bc - t_bc)^2 / (B*C);
 *              ESTK_LOSS_XENT soft-target cross-entropy on the logits y (the last Linear's
 *              output, acc + bias), target rows t_b = class weights (one-hot or soft labels):
 *                m_b = max_c y_bc,  lse_b = m_b + logf(sum_c expf(y_bc - m_b)),
 *                ce_b = lse_b * sum_c t_bc - sum_c t_bc * y_bc,  return = -sum_b ce_b / B.
 *              All of it fp32 with IEEE expf / logf, reductions in a fixed order (the same
 *              bits from run to run); the max shift keeps it finite for finite logits and a
 *              NaN logit gives a NaN return.  The behaviour characteristic stays the logits.
 *              Valid with the identity output only (the softmax is the output map).
 *              ESTK_LOSS_ACCURACY classification accuracy on the logits y (acc + bias), target rows
 *              t_b = class weights as for ESTK_LOSS_XENT:
 *                label_b = the first index of the maximum of t_b,
 *                pred_b  = the first index of the maximum of y_b (torch.argmax's rule: ties go to the
 *                          lowest index and a NaN counts as the maximum, so the first NaN wins),
 *                return  = (float)count / (float)B, count = #{b : pred_b == label_b}, an IEEE divide.
 *              count is an exact integer (per-row 0 / 1 values summed without float atomics), so the
 *              return is the same bits from run to run and, on the same logits, those of
 *              torch's (y.argmax(1) == t.argmax(1)).float().mean() on the CPU.  B < 2^24 keeps the
 *              count exact (a larger B is ESTK_ERR_INVALID with this loss).  The behaviour
 *              characteristic stays the logits.  Valid with the identity output only, for the hidden
 *              kinds of bits 0-7 (not with a recurrent cell), in the dense MLP evaluate (every
 *              precision, under the shape rules of the cross-entropy) and in the convolutional evaluate.
 *              ESTK_ACTIONS: no return at all -- the outputs themselves, on each member's OWN
 *              observations (one forward of every perturbed policy per environment step):
 *                population (offsets != NULL): obs is [2*pairs][B][dims[0]]; block j holds the
 *                observations of the + member of local pair j, block pairs + j those of its - member;
 *                bc_plus[j] / bc_minus[j] receive policy_m(obs_m[:bc_obs]).flatten()[:bc_dim] (the
 *                behaviour-characteristic definition above, on the member's own observations);
 *                centre (offsets == NULL): obs is [B][dims[0]] and bc_plus receives theta's outputs.
 *              target, returns_plus, returns_minus and centre_return_out are not read (NULL is fine;
 *              centre_return_out must be NULL); bc_plus (and bc_minus for a population) must be set.
 *              order keeps its meaning (scheduling only).  table16, when non-null, is read INSTEAD
 *              of table: it must be the exact fp16 copy (estk_shadow_f16 with inexact_count 0), so
 *              the values and the bits are the same at half the noise bytes.
 *              ESTK_PREC_FP32 only (tensor-core precisions are ESTK_ERR_UNSUPPORTED before any
 *              launch).  Arithmetic: that of the fp32 evaluate -- W = theta +- (sigma*t) with two
 *              roundings, one fmaf chain per output from 0 in ascending k, + bias, the hidden
 *              activation, tanhf for ESTK_ACT_OUT_TANH -- so a member's outputs are bit-identical to
 *              the behaviour characteristic the squared-error fp32 evaluate writes for that member
 *              when every member is given the same observations.  A member's outputs never depend on
 *              another member's observations; no float atomics (the same bits from run to run, with
 *              or without order, from table or table16).  Any widths, any B >= 1.
 *              Recurrent cells (ESTK_CELL_GRU / ESTK_CELL_LSTM in bits 0-7, with ESTK_ACTIONS and
 *              an identity or ESTK_ACT_OUT_TANH output): one step of a policy that is one
 *              GRUCell / LSTMCell (bias=True) followed by one Linear head.  n_layers must be 2 and
 *              dims = (in, H, out).  The parameters are torch's, in registration order: weight_ih
 *              [G*H][in], weight_hh [G*H][H], bias_ih [G*H], bias_hh [G*H] (G = 3 gates r, z, n
 *              for GRU; G = 4 gates i, f, g, o for LSTM), then the head's weight [out][H] and bias.
 *              The step is the function [x | state] -> [y | state']: obs rows are in + S wide
 *              and output rows out + S, S = H (GRU: h) or 2H (LSTM: h then c); bc_plus /
 *              bc_minus receive the output rows exactly as above (bc_obs = B, bc_dim =
 *              B*(out+S) for all of them).  Arithmetic, fp32: W = theta +- (sigma*t) with two
 *              roundings; per gate row the input half (x against weight_ih) and the hidden half
 *              (h against weight_hh) are separate fmaf chains from 0 in ascending k, each + its own
 *              bias, a = chain_ih + b_ih and b = chain_hh + b_hh; s(v) = 1.0f / (1.0f + expf(-v))
 *              with an IEEE divide, tanhf as above.
 *                GRU:  r = s(a_r + b_r), z = s(a_z + b_z), n = tanhf(fmaf(r, b_n, a_n)),
 *                      h' = fmaf(z, h - n, n)          (= (1 - z)*n + z*h, torch's form)
 *                LSTM: i = s(a_i + b_i), f = s(a_f + b_f), g = tanhf(a_g + b_g), o = s(a_o + b_o),
 *                      c' = fmaf(f, c, i*g), h' = o * tanhf(c')
 *              then the head is the act-mode layer above on h' (fmaf chain, + bias, tanhf for
 *              ESTK_ACT_OUT_TANH).  n_layers != 2 is ESTK_ERR_INVALID; the same determinism
 *              guarantees hold.
 * Recurrent sequence evaluate (a cell in bits 0-7 with the squared error, identity or ESTK_ACT_OUT_TANH
 * output, or with ESTK_LOSS_XENT, identity output): every member runs over B sequences of T steps and
 * its return scores all B*T steps.  n_layers = 2, dims = (in, H, out) as for the step and dims[3] = T >= 1
 * (the entry a 2-layer desc otherwise leaves unused); obs is [B][T][in] and target [B][T][out], the same
 * for every member.  Every member starts from a zero state (h, and c for LSTM); at step t it reads
 * x = obs[b][t] and the state the previous step left, and computes the ESTK_ACTIONS step above element by
 * element, so its outputs are the bits that T chained ESTK_ACTIONS launches produce when each launch is fed
 * the previous launch's [h' | c'].  Per step (b, t) in fp32: the squared error s_bt = fmaf chain over c
 * ascending from 0 of d*d, d = y_btc - t_btc; the cross-entropy ce_bt is the MLP formula above on y_bt
 * (a step whose target row is all zeros then contributes 0 for finite logits: a task can score only some
 * steps, e.g. the last; the return scales by a constant and the ranks do not change).  Then L_b = the sum
 * of the step values over t in ascending order from 0, S = the sum of L_b over b in ascending order from 0
 * (the work item of a pair that finishes last adds them), and return = -(S / (float)(B*T*out)) for the
 * squared error, -(S / (float)(B*T)) for the cross-entropy (the integer count converted to fp32 once, an
 * IEEE divide).  No float atomics: the same bits from run to run, with or without order; sigma = 0 gives
 * every member the centre's return.  bc_plus / bc_minus receive y of the first bc_obs sequences flattened
 * in (b, t, c) order, then [:bc_dim]; the population and centre forms are those of the MLP evaluate.
 * ESTK_PREC_FP32 only, reading table (table16 is not read); a tensor-core precision, and a non-null
 * centre_return_out, are ESTK_ERR_UNSUPPORTED before any launch; T < 1, a NULL target or NULL returns,
 * and n_layers != 2 are ESTK_ERR_INVALID before any launch.  The per-sequence sums live in the context
 * workspace (pairs * 2 * B floats; ESTK_ERR_NOMEM under capture when it must grow).
 * Convolutional evaluate (bits 24-31 = n_conv, 1..7: the number of leading Conv2d layers): a policy
 * Conv2d -> act -> ... -> Conv2d -> act -> flatten -> Linear -> act -> ... -> Linear [-> out_act] over a fixed
 * batch of B images.  dims[0] = ESTK_CNN_INPUT(c, h, w) (c, h, w in 1..1023); dims[1..n_conv] =
 * ESTK_CNN_CONV(out_c, k, stride, pad), one per conv (out_c 1..4095, a square kernel k 1..63, stride 1..63,
 * symmetric zero padding 0..63 with pad < k; dilation 1, groups 1); dims[n_conv+1..n_layers] are the Linear
 * output widths, n_layers - n_conv >= 1.  The first Linear's input width is C*H*W of the last conv's output
 * flattened in torch's (c, h, w) order -- derived, never passed.  A conv's output is H' = (H + 2*pad - k) /
 * stride + 1 (and W' likewise), which must be >= 1.  Bits 0-23 keep their meaning: the hidden kind (ReLU,
 * Tanh, ELU, SiLU, LeakyReLU) follows every conv and every Linear but the last, the output is identity or
 * ESTK_ACT_OUT_TANH, the loss 0 (squared error) or ESTK_LOSS_XENT (identity output only).  The parameters
 * are in parameters_to_vector order: each conv's weight [out_c][in_c][k][k] then its bias, then each Linear's
 * weight [out][in] and bias.  obs is [B][c][h][w], target [B][out]; bc_plus / bc_minus receive
 * policy(obs[:bc_obs]).flatten()[:bc_dim]; the population and centre forms are those of the MLP evaluate.
 * Arithmetic, fp32: W = theta +- (sigma*t) with two roundings; each conv output is one fmaf chain from 0 over
 * the taps in ascending (ci, kh, kw) order (taps in the zero padding contribute nothing), then + bias, then
 * the hidden activation; each Linear output is the fp32 MLP evaluate's chain (from 0 in ascending k, + bias).
 * So a conv whose kernel covers its whole input (k = h = w, stride 1, pad 0) computes the bits of the fp32
 * MLP evaluate's first Linear on the flattened input.  The per-image value is the squared error, an fmaf
 * chain over the outputs c ascending from 0 of d*d, d = y_bc - t_bc, or the cross-entropy ce_b of the MLP
 * formula; S = the sum of the per-image values over b in ascending order from 0 (kept in the context
 * workspace, pairs * 2 * B floats; the work item of a pair that finishes last adds them), and return =
 * -(S / (float)(B*out)) for the squared error, -(S / (float)B) for the cross-entropy.  No float atomics: the
 * same bits from run to run, whatever the chunking, the schedule or order; sigma = 0 gives every member the
 * centre's bits.  ESTK_PREC_FP32 only, reading table: a tensor-core precision is ESTK_ERR_UNSUPPORTED before
 * any other check of the code, as are a non-null centre_return_out and, under ESTK_PREC_FP32, ESTK_ACTIONS or
 * a recurrent cell in bits 0-23.  n_conv > 7, undefined bits 0-23, malformed packed fields (zero channels,
 * pad >= k, a conv larger than its padded input), n_layers <= n_conv, and more than 2^30 inputs, taps or
 * outputs per image in one layer are ESTK_ERR_INVALID before any launch.  estk_eval_mlp_supported returns 0
 * for every code with bits 24-31 != 0.
 * The defined codes are, for each hidden kind h in {ESTK_ACT_RELU, ESTK_ACT_TANH, ESTK_ACT_ELU,
 * ESTK_ACT_SILU, ESTK_ACT_LEAKY_RELU}: h, h | ESTK_ACT_OUT_TANH, h | ESTK_LOSS_XENT, h | ESTK_ACTIONS
 * and h | ESTK_ACT_OUT_TANH | ESTK_ACTIONS (25 codes), and for each cell c in {ESTK_CELL_GRU,
 * ESTK_CELL_LSTM}: c | ESTK_ACTIONS and c | ESTK_ACT_OUT_TANH | ESTK_ACTIONS (4 codes; the MLP and step
 * codes, 29 in all; the sequence codes add 6: c, c | ESTK_ACT_OUT_TANH and c | ESTK_LOSS_XENT, 35 in all).
 * Loss value 2 (0x20000) is undefined.
 * ESTK_LOSS_ACCURACY (6 << 16) adds 5 codes beside them: h | ESTK_LOSS_ACCURACY for each hidden kind h.
 * 0 is ReLU hidden + identity output + squared error.  Any other value is ESTK_ERR_INVALID in
 * estk_eval_mlp with ESTK_PREC_FP32, ESTK_ERR_UNSUPPORTED with a tensor-core precision,
 * and makes estk_eval_mlp_supported return 0.
 * Arithmetic of tanh: IEEE tanhf (libdevice, ~1-2 ulp, no tanh.approx) on the fp32
 * value acc + bias.  fp32 path: the result stays fp32.  Tensor-core paths: a hidden
 * tanh is rounded ONCE to the 16-bit operand type when the activation is written back
 * (|tanh| <= 1, so the fp16 saturation never applies); the output tanh stays fp32.
 * Arithmetic of ELU / SiLU / LeakyReLU, on the fp32 value y = acc + bias: ELU y > 0 ? y :
 * expm1f(y); SiLU y / (1.0f + expf(-y)) with an IEEE divide; LeakyReLU y > 0 ? y : y * 0.01f.
 * IEEE expf / expm1f only (no __expf): SiLU(-100) = -0, ELU(-100) = -1.  fp32 path: the result
 * stays fp32.  Tensor-core paths: rounded ONCE to the 16-bit operand type when the activation
 * is written back, saturating in fp16 as ReLU does (ELU >= -1 and SiLU >= -0.28, so only their
 * positive side can saturate; LeakyReLU can saturate on both sides). */
#define ESTK_ACT_RELU 0
#define ESTK_ACT_TANH 1
#define ESTK_ACT_ELU 3
#define ESTK_ACT_SILU 4
#define ESTK_ACT_LEAKY_RELU 5
#define ESTK_CELL_GRU 8
#define ESTK_CELL_LSTM 9
#define ESTK_ACT_OUT_TANH (1 << 8)
#define ESTK_LOSS_XENT (1 << 16)
#define ESTK_ACTIONS (3 << 16)
#define ESTK_LOSS_ACCURACY (6 << 16)
/* the convolutional evaluate (above): n_conv in bits 24-31 of the activation code, packed dims */
#define ESTK_CNN_N_CONV(n) ((int32_t)((uint32_t)(n) << 24))
#define ESTK_CNN_INPUT(c, h, w) ((int32_t)((uint32_t)(c) | (uint32_t)(h) << 10 | (uint32_t)(w) << 20))
#define ESTK_CNN_CONV(out_c, k, stride, pad) \
  ((int32_t)((uint32_t)(out_c) | (uint32_t)(k) << 12 | (uint32_t)(stride) << 18 | (uint32_t)(pad) << 24))

/* Arithmetic of the evaluate kernels (estk_eval_mlp, estk_eval_conv_vbn); what each one
 * computes is stated at those functions. */
#define ESTK_PREC_FP32 0   /* CUDA cores, exact fp32 */
#define ESTK_PREC_F16 1    /* tensor cores, fp16 operands formed from fp32 sums (the default) */
#define ESTK_PREC_BF16 2   /* tensor cores, bf16 operands (opt-in, lower precision) */
#define ESTK_PREC_BF16S 3  /* tensor cores, bf16 operands from bf16 shadows (opt-in, lower precision) */
#define ESTK_PREC_F16_ANY 4 /* tensor cores, the F16 arithmetic for every MLP shape (opt-in) */
typedef struct {
  int32_t n_layers;                  /* number of Linear layers, 1..ESTK_MAX_LAYERS */
  int32_t dims[ESTK_MAX_LAYERS + 1]; /* dims[0] = obs dim, dims[n_layers] = out dim */
  int32_t activation;                /* ESTK_ACT_* bit fields above; 0 = ReLU between layers, none after the last */
} estk_mlp_desc;

/* torch.optim.Adam hyper-parameters (torch/optim/adam.py:429-545; the
 * optimizer every reference example uses, examples/cartpole_es.py:48-50).
 * The step is torch's single-tensor CPU Adam rounded as ATen rounds it: the weight-decay add,
 * lerp_ (both of its forms) and addcmul_ are one fma each, every other operation is rounded on
 * its own.  m and v are bit-exact to torch; theta is bit-exact to that form, and to torch wherever
 * torch's CPU sqrt is correctly rounded (the kernels' sqrt always is).  weight_decay is torch's L2
 * decay through the gradient; AdamW's decoupled decay (decoupled_weight_decay=True), amsgrad and
 * maximize are not implemented (the Python engine refuses them and runs torch's own optimizer). */
typedef struct {
  double lr, beta1, beta2, eps, weight_decay;
  float clamp; /* estorch.py:243 clamps the negated gradient to +-1.0; <=0 disables */
} estk_adam_desc;

ESTK_API int estk_version(void);
ESTK_API const char* estk_last_error(void);

ESTK_API int estk_ctx_create(int device, estk_ctx** out);
ESTK_API int estk_ctx_destroy(estk_ctx* ctx);
/* sm_count, compute capability of the context's device (host ints). */
ESTK_API int estk_ctx_info(estk_ctx* ctx, int* sm_count, int* cc_major, int* cc_minor);

/* ---- noise table (new-engine replacement of estorch.py:189-190's fresh
 *      Normal(0,sigma).sample per generation) ---- */

/* Fill table[0:len) with unit normals: Philox4x32-10(counter=i/4, key=seed)
 * + Box-Muller, each entry then rounded to the nearest fp16-representable value
 * (11 significant bits; still stored as fp32 here) so that the 16-bit copy made by
 * estk_shadow_f16 is exact.  len % 4 == 0.  Identical on every GPU for the same seed. */
ESTK_API int estk_fill_noise_table(estk_ctx* ctx, float* table, int64_t len, uint64_t seed,
                          void* stream);

/* offsets_out[i] = 32 * (mix64(mix64(seed ^ gen*C) + pair_begin + i) mod nslots),
 * nslots = (table_len - ceil32(n))/32 + 1.  gen = gen_host, plus state->generation
 * when `state` is non-null (device counter advanced by estk_track_best: a generation
 * replayed from a CUDA graph passes a constant gen_host -- 0, or 1 while the previous
 * generation's estk_track_best is still folded into this one -- and never a host scalar).  order_out (nullable, int32
 * [pairs]) receives the local pair indices sorted by offset (ties by index):
 * evaluating / reducing pairs in that order lets overlapping table rows hit L2.
 * pairs <= ESTK_MAX_POPULATION/2; table_len <= ESTK_MAX_TABLE_LEN.  Up to 4096 pairs one CTA sorts; more
 * take one cooperative grid-wide radix sort (workspace in the context). */
ESTK_API int estk_make_offsets(estk_ctx* ctx, uint64_t seed, const estk_state* state, int64_t gen_host,
                      int64_t pair_begin, int32_t pairs, int64_t table_len, int64_t n,
                      int64_t* offsets_out, int32_t* order_out, void* stream);

/* Materialise population rows (estorch.py:187-193 `_sample_policy`):
 * for m in [member_begin, member_begin+member_count): rows_out[m-member_begin] =
 * theta +- sigma*T[off], eps_out (nullable) = +-sigma*T[off].  P = 2*pairs. */
ESTK_API int estk_perturb_rows(estk_ctx* ctx, const float* theta, int64_t n, const float* table,
                      const int64_t* offsets, int32_t pairs, float sigma,
                      int32_t member_begin, int32_t member_count,
                      float* rows_out, float* eps_out, void* stream);

/* ---- 16-bit copies for the tensor-core evaluate ---- */

/* dst[i] = rn_f16(src[i]); inexact_count (device, nullable) += the number of entries that
 * changed.  A table made by estk_fill_noise_table comes back with 0: its fp16 copy is then
 * EXACT (every consumer converts it back to the very fp32 value the table holds), which is
 * what ESTK_PREC_F16 and the fp16-table form of estk_rank_grad* require.
 * n % 4 == 0; src 16-byte, dst 8-byte aligned. */
ESTK_API int estk_shadow_f16(estk_ctx* ctx, const float* src, uint16_t* dst, int64_t n,
                    uint64_t* inexact_count, void* stream);
/* dst[i] = rn_bf16(src[i]): the bf16 SHADOWS of theta and of the table that ESTK_PREC_BF16S
 * reads.  Same shape and alignment rules as estk_shadow_f16. */
ESTK_API int estk_shadow_bf16(estk_ctx* ctx, const float* src, uint16_t* dst, int64_t n, void* stream);

/* ---- kernel 1: population evaluate (estorch.py:195-202 `_calculate_returns`
 *      + Policy.forward examples/cartpole_es.py:14-20 + the synthetic agent
 *      return -mean((policy(obs)-target)^2), SURVEY 8d) ---- */

/* MLP policy `desc` over the observation batch obs [B, dims[0]], target [B, dims[L]] (fp32,
 * row-major).
 *
 * Population (offsets != NULL): for each local pair j, returns_plus[j] / returns_minus[j] =
 * return of theta +/- sigma*T[offsets[j]].  order (nullable) = evaluation order from
 * estk_make_offsets.  bc_plus / bc_minus (both or neither) [pairs, bc_dim] receive the
 * behaviour characteristic policy(obs[:bc_obs]).flatten()[:bc_dim] (examples/nsra_es.py:45-49).
 * centre_return_out (nullable; tensor-core precisions only, ESTK_ERR_UNSUPPORTED with FP32):
 * additionally evaluate theta itself (sigma = 0) in the same launch and write its return there
 * -- the estorch.py:182 rollout of the previous update folded into this generation's launch.
 *
 * Centre (offsets == NULL; the estorch.py:181-182 `_after_optimize` rollout): returns_plus[0] =
 * return of theta, bc_plus (nullable) [bc_dim] its behaviour characteristic.  table, table16,
 * order, pairs, sigma, returns_minus and bc_minus are not read; centre_return_out must be NULL.
 *
 * bc_obs and bc_dim must be positive when behaviour-characteristic outputs are given.
 *
 * precision -- the arithmetic, and the buffers it needs besides theta / obs / target / returns:
 *   ESTK_PREC_FP32   CUDA cores, exact fp32 with the reference's two roundings (eps = sigma*t,
 *                    then theta +- eps).  Population: table.  Any widths and any B, limited only by
 *                    device memory: shapes whose activations do not fit in shared memory, or whose
 *                    batch needs more than 64 observation chunks, stream their hidden activations
 *                    through a slab in the context workspace (grown like the other buffers above),
 *                    with the same arithmetic per element and the same bits from run to run.
 *   ESTK_PREC_F16    the default: wgmma with fp16 operands (11-bit significand, the TF32 class)
 *                    and fp32 accumulation.  Every weight is formed in fp32 from the fp32 theta
 *                    and the noise value and rounded ONCE: W16 = rn_f16(theta + s*sigma*T[off+i])
 *                    (sum in fp32, like estorch.py:192).  The noise is read from table16, the EXACT
 *                    fp16 copy of `table` (estk_shadow_f16 with inexact_count 0), so the kernel
 *                    evaluates exactly the members the gradient estimate (estk_rank_grad*) weights.
 *                    Hidden activations are rounded to fp16 when written back (saturating at
 *                    +-65504), the observations enter as x_hi + x_lo (two fp16 operands), biases and
 *                    the squared error are fp32.  Finite observations keep ~22 significant bits up
 *                    to |x| = 131008 (65504 + 65504; x_hi saturates, up to 131023 rounds to it); x_lo
 *                    does not saturate, so +-inf -- and a finite |x| >= 131024, beyond the split's
 *                    range -- enters with x_lo = +-inf and NaN as NaN: a non-finite observation gives
 *                    the non-finite outputs FP32 gives.  Population: table, table16.
 *   ESTK_PREC_BF16   opt-in, lower precision: wgmma with bf16 operands, fp32 accumulation; weights
 *                    are rounded to bf16 when the B-operand tile is formed, activations when they
 *                    are written back.  Returns agree with FP32 to ~1e-2 relative.  Population: table.
 *   ESTK_PREC_BF16S  opt-in, lower precision: as BF16, but the weights are formed from bf16
 *                    SHADOWS (estk_shadow_bf16): W = bf16(theta16 + s*sigma*table16[off+i]), half the
 *                    bytes per weight element; biases still come from the fp32 theta / table.
 *                    NOTE: it evaluates F(theta16 +- sigma16*eps16) while estk_rank_grad* weights
 *                    the fp32 eps -- the estimator multiplies a return by a noise vector that is
 *                    not exactly the one that produced it (estorch.py:177-178 uses the same eps on
 *                    both sides); F16 has no such departure.  Always: theta16.  Population: table,
 *                    table16 (the bf16 shadow of the table).
 *   ESTK_PREC_F16_ANY  opt-in: the F16 arithmetic above, per element, for every MLP shape FP32 takes
 *                    (any widths, any B >= 1, limited only by device memory).  Where F16's shape rule
 *                    below holds it runs F16's kernel, the same launch and the same bits.  Elsewhere a
 *                    streamed wgmma kernel runs: K is padded with zero weights and activations, rows
 *                    past B are masked out, hidden activations stream through a slab in the context
 *                    workspace, and the k-order per accumulator is F16's, so a pre-activation is the
 *                    same bits as F16's for the same member, row and column.  The streamed kernel
 *                    takes two launches (the observations' hi / lo split, then the evaluate), has no
 *                    folded centre (centre_return_out is ESTK_ERR_UNSUPPORTED there, before any
 *                    launch) and gives the same bits from run to run.  The kernel follows from the
 *                    shape, never from the caller.  Population: table, table16.
 *   Buffers a precision does not list are not read.
 * Tensor-core precisions (F16, F16_ANY, BF16, BF16S): theta, obs, target and the listed table / table16 /
 * theta16 must be 16-byte aligned.  F16, BF16 and BF16S: every layer input width a multiple of 64 in
 * [64,512], every output width a multiple of 32 in [32,512], B a multiple of 256, and for F16
 * dims[0] <= 256; other shapes are ESTK_ERR_UNSUPPORTED (estk_eval_mlp_supported tells in advance).
 * F16_ANY: an undefined activation code is ESTK_ERR_UNSUPPORTED.
 * Agreement with FP32 is asserted in tests/test_kernels_gpu.py and tests/test_eval_mlp_act_gpu.py. */
ESTK_API int estk_eval_mlp(estk_ctx* ctx, const estk_mlp_desc* desc, int32_t precision,
                  const float* theta, const uint16_t* theta16,
                  const float* table, const uint16_t* table16,
                  const int64_t* offsets, const int32_t* order, int32_t pairs, float sigma,
                  const float* obs, const float* target, int32_t B,
                  float* returns_plus, float* returns_minus,
                  float* bc_plus, float* bc_minus, int32_t bc_obs, int32_t bc_dim,
                  float* centre_return_out, void* stream);

/* 1 when the tensor-core `precision` (F16, BF16 or BF16S) can evaluate `desc` at batch B (the
 * shape rules above, and a defined activation code that computes a return, i.e. not ESTK_ACTIONS, and
 * no recurrent cell), else 0 -- also for a null desc and for any other precision code.  F16_ANY: 1 for
 * every desc with 1..ESTK_MAX_LAYERS layers, positive widths and a defined activation code other than
 * the ESTK_ACTIONS and recurrent-cell ones, at every B >= 1. */
ESTK_API int estk_eval_mlp_supported(const estk_mlp_desc* desc, int32_t precision, int32_t B);

/* ---- conv + VirtualBatchNorm policy of examples/atari.py:14-37 (BASELINE config 5):
 * conv1 4->16 k8 s4, VBN(16), ReLU, conv2 16->32 k4 s2, VBN(32), ReLU, fc1 2592->256,
 * ReLU, fc2 256->n_actions; VBN statistics = per-(C,H,W) mean / unbiased variance of
 * the reference batch xref [ref_batch,4,84,84] under the member's own weights
 * (estorch/modules.py:48-58).  obs [B,4,84,84], target [B,n_actions]; return =
 * -mean((policy(obs)-target)^2).
 *
 * Population (offsets != NULL): returns_plus[j] / returns_minus[j] = return of
 * theta +/- sigma*T[offsets[j]] (j = order[slot] when order is given).  Centre (offsets == NULL):
 * returns_plus[0] = return of theta; table, table16, order and returns_minus are not read.
 * scratch: caller-owned device slab of at least as many bytes as estk_eval_conv_vbn_scratch_bytes
 * returns for the same precision, ref_batch and B (it returns -1 for bad arguments or a precision
 * without a conv kernel).  Shapes: ref_batch >= 2 (unbiased variance), B >= 1, 1 <= n_actions <= 64; xref and
 * obs 16-byte aligned.
 *
 * precision:
 *   ESTK_PREC_FP32  fp32 throughout.  Population: table.
 *   ESTK_PREC_F16   conv1, conv2 and fc1 on mma.sync with fp16 operands and fp32 accumulation;
 *                   every operand -- the weights theta + s*sigma*T[off+i] (formed in fp32 from the
 *                   fp32 theta and table16, the EXACT fp16 copy of `table` made by estk_shadow_f16),
 *                   the input frames and the normalised activations (those scaled by 2^-10 first, so
 *                   values up to ~3e7 fit) -- enters as hi + lo, two fp16 values (22 significant bits), so the returns stay within 1e-5 (max-norm
 *                   relative) of the fp32 forward.  VBN statistics, normalisation, biases, fc2 and
 *                   the loss are fp32; no atomics, so the returns are the same bits run to run.
 *                   Population: table, table16.  theta, scratch and table16 16-byte aligned.
 *   any other       ESTK_ERR_UNSUPPORTED.
 *
 * Action mode (an environment population's per-step forward).  n_actions is three bit fields:
 *   bits 0-7   A, the number of actions, 1..64;
 *   bits 8-15  must be 0;
 *   bits 16-23 0 (the evaluate above) or ESTK_ACTIONS (the same macro and meaning as the loss field of
 *              estk_mlp_desc.activation): no return, each member's outputs on its OWN frames.
 * Every value refused before this mode existed is still refused.  With ESTK_ACTIONS only ESTK_PREC_FP32
 * serves (ESTK_PREC_F16 and any other precision are ESTK_ERR_UNSUPPORTED before any launch), target is not
 * read, order keeps its meaning (scheduling only), and table16, when non-null, is read INSTEAD of table (the
 * exact fp16 copy: the same values and bits at half the noise bytes).  estk_eval_conv_vbn_scratch_bytes keeps
 * its meaning (the evaluate's scratch); here scratch holds the VBN statistics of every member,
 * [members][ESTK_CONV_VBN_STATS_FLOATS] fp32 in member order (the + members of the local pairs, then their
 * mirrors; the centre has one member), so scratch_bytes >= members * ESTK_CONV_VBN_STATS_FLOATS * 4, and
 * scratch is 16-byte aligned.  A member's entry is VBN1's scale a = gamma / sqrtf(var + 1e-5f) [16*20*20],
 * then its mean [16*20*20], then VBN2's a and mean [32*9*9] each (gamma the member's perturbed parameter;
 * mean and unbiased var over xref by Welford's update in frame order, d = y - mean, mean = fmaf(d, 1/n, mean),
 * m2 = fmaf(d, y - mean, m2), var = m2/(R-1), which stays accurate where the mean is large and the variance
 * near 0, e.g. 0..255 pixels that never change).  A call
 * runs one or both phases, the stats phase first:
 *   stats phase (xref != NULL): writes every member's statistics into scratch; ref_batch >= 2.  The raw
 *              conv1 outputs of the reference batch go through a per-CTA slab of the context workspace
 *              (grown like the buffers above: ESTK_ERR_NOMEM under capture).
 *   act phase (obs != NULL): reads the statistics from scratch.  Population: obs [2*pairs][B][4][84][84]
 *              (block j the frames of the + member of local pair j, block pairs + j those of its mirror),
 *              returns_plus [pairs][B][A] receives the + members' outputs, returns_minus [pairs][B][A] the
 *              mirrors'.  Centre (offsets == NULL): obs [B][4][84][84], returns_plus [B][A] for theta.
 * A call with xref == NULL uses what an earlier stats call left in scratch; the caller must have made that
 * call for the same theta, offsets, pairs and sigma.  xref and obs both NULL is ESTK_ERR_INVALID.
 * Arithmetic, element by element that of the fp32 evaluate: W = theta +- (sigma*t) with two roundings,
 * conv1 / conv2 as fmaf chains from the bias in (ci, kh, kw) order, normalisation fmaxf(fmaf(y - mean, a, beta), 0),
 * fc1 one chain from 0 in ascending k then + bias and ReLU, fc2 one chain from the bias -- a member's
 * outputs are the bits of the outputs its ESTK_PREC_FP32 evaluate computes on the same frames.  A member's
 * outputs never depend on another member's frames; no float atomics (the same bits from run to run, with
 * or without order, from table or table16). */
#define ESTK_CONV_VBN_STATS_FLOATS 17984  /* per member: 2 * 16*20*20 + 2 * 32*9*9 */
ESTK_API int64_t estk_eval_conv_vbn_scratch_bytes(estk_ctx* ctx, int32_t precision, int32_t ref_batch, int32_t B);
ESTK_API int estk_eval_conv_vbn(estk_ctx* ctx, int32_t precision, int32_t n_actions, const float* theta,
                       const float* table, const uint16_t* table16,
                       const int64_t* offsets, const int32_t* order, int32_t pairs, float sigma,
                       const float* xref, int32_t ref_batch, const float* obs, const float* target,
                       int32_t B, float* returns_plus, float* returns_minus, void* scratch,
                       int64_t scratch_bytes, void* stream);

/* estorch.py:182-185: episode_reward = *reward; if it beats state->best_reward,
 * take it and copy theta -> best_theta (the device analogue of
 * deepcopy(state_dict())).  Also advances state->generation (estorch.py:248). */
ESTK_API int estk_track_best(estk_ctx* ctx, estk_state* state, const float* reward,
                    const float* theta, float* best_theta, int64_t n, void* stream);

/* ---- kernel 2: centred-rank transform + weighted noise reduction + Adam
 *      (estorch.py:15-39 rank_transformation, :174-179 _calculate_grad and the
 *      NS/NSR/NSRA variants :419-425/:542-549/:640-648, :236-244 negate+clamp,
 *      :245 optimizer.step -> torch Adam) ----
 *
 * Common to the three rank + gradient functions below:
 *   returns [P] (reward column), novelty [P] or NULL.  Blend row c = w_rew*c(reward) +
 *   w_nov*c(novelty) in fp32 when novelty is given (ES: novelty NULL -> c(reward)).  Ranks are
 *   bit-exact vs _compute_ranks on tie-free input (ties: stable by member index; NaN returns sort
 *   last like numpy's argsort, among themselves by index; -0 ties with +0) for any P <= ESTK_MAX_POPULATION:
 *   P <= 8192 by an all-pairs count in shared memory, larger P by a grid-wide stable radix sort in
 *   the same launch (one launch per call either way); centring in fp64 then fp32 as
 *   estorch.py:17-19,:176.  The gradient estimate is
 *     g = (1/P) * sum_j (c_j - c_{j+pairs}) * T[off_j : off_j+n]
 *   over pair j's offset offsets[j] (order, nullable = reduction order from estk_make_offsets).
 *   Every offsets[j] is a multiple of 32, as estk_make_offsets makes them, and offsets[j] + n is at most the
 *   table's length (<= ESTK_MAX_TABLE_LEN).
 *   The noise table: exactly one of `table` (fp32) and `table16` (the EXACT fp16 copy made by
 *   estk_shadow_f16: 8 noise values per 128-bit load, half the bytes per pair row, the same
 *   results because every fp16 value converts exactly to the fp32 value the table holds) is
 *   non-null; 16-byte aligned.
 *   `world` > 1 (where taken): `returns` / `novelty` are laid out RANK-MAJOR,
 *   [world][2][pairs/world] -- exactly what an in-place all-gather of each rank's
 *   (returns_plus[pairs_local], returns_minus[pairs_local]) block produces, so no re-ordering copy
 *   is needed (member j < pairs of rank r, local index i, sits at ((2r + 0) * pairs_local + i), its
 *   mirror at ((2r + 1) * pairs_local + i)); ranks_out stays in member order and ties are still
 *   broken by member index.  world must divide pairs.
 *   ranks_out / ranks2_out (nullable, int32 [P]) and grad_out (nullable, fp32 [n], the reference's
 *   un-negated estimate g) are for inspection / parity.
 *   With Adam: grad = clamp(-g), Adam(theta, m, v) in place (theta / m / v / grad_out 16-byte
 *   aligned); state->adam_step += 1. */

/* Single-GPU fused form: all P/2 pairs, member-order returns, Adam. */
ESTK_API int estk_rank_grad_adam(estk_ctx* ctx, const float* returns, const float* novelty,
                        float w_rew, float w_nov, int32_t P,
                        const float* table, const uint16_t* table16,
                        const int64_t* offsets, const int32_t* order,
                        int64_t n, float* theta, float* m, float* v, estk_state* state,
                        const estk_adam_desc* adam,
                        int32_t* ranks_out, int32_t* ranks2_out, float* grad_out, void* stream);

/* Multi-GPU form: same rank phase over all P returns (member order, or rank-major with
 * world > 1), reduction over the local pairs [pair_begin, pair_begin+pairs_local) only
 * (offsets / order index those); grad_sum_out[n] (16-byte aligned) receives the RAW partial sum
 * (no 1/P) to be all-reduced (SUM) by the caller, then estk_clamp_adam
 * (replaces the Send/Recv star of estorch.py:207-233). */
ESTK_API int estk_rank_grad(estk_ctx* ctx, const float* returns, const float* novelty,
                   float w_rew, float w_nov, int32_t P, int32_t world,
                   const float* table, const uint16_t* table16,
                   const int64_t* offsets, const int32_t* order,
                   int32_t pair_begin, int32_t pairs_local, int64_t n,
                   float* grad_sum_out, int32_t* ranks_out, int32_t* ranks2_out, void* stream);

/* ---- the same update with the cross-GPU reduction INSIDE the kernel (NVLink peer memory) ----
 * Replaces estk_rank_grad -> NCCL all-reduce -> estk_clamp_adam (the reference's gather of returns
 * on the master + one optimizer step there, estorch.py:228-245) by ONE cooperative launch per GPU:
 *   rank + partial gradient over the local pairs -> own workspace            (as estk_rank_grad)
 *   cross-GPU barrier (flags in peer memory, release/acquire at system scope)
 *   reduce-scatter: rank r sums slice r of all `world` workspaces in rank order (loads over NVLink),
 *   all-gather: and stores the sum into every rank's workspace (stores over NVLink)
 *   cross-GPU barrier
 *   negate / clamp / Adam over all n from the summed gradient (replicated: every rank applies the
 *   same bits to its own theta / m / v, so the replicas stay bit-identical).
 * The sum over ranks is taken in rank order 0..world-1 on every slice: deterministic and identical on
 * all GPUs (it differs from NCCL's order by fp32 rounding only).
 * Every rank of the job must make the same call in the same generation (like a collective).
 * Returns rank-major, 2 <= world <= ESTK_MAX_PEERS, 0 <= rank < world; the noise comes from table16,
 * the exact fp16 copy of the table.
 *
 * Workspaces: estk_peer_alloc gives zero-filled device memory plus a 64-byte handle that another
 * process on the same node turns into a device pointer with estk_peer_open (CUDA IPC; the bytes of the
 * handle travel over whatever channel the host code has, e.g. a torch.distributed all_gather_object).
 * `peer_ws` is a HOST array of `world` device pointers -- entry r = rank r's workspace as mapped in the
 * calling process, entry `rank` = the caller's own allocation -- each of estk_xr_workspace_bytes(n). */
#define ESTK_MAX_PEERS 16
#define ESTK_PEER_HANDLE_BYTES 64
ESTK_API int64_t estk_xr_workspace_bytes(int64_t n);
ESTK_API int estk_peer_alloc(estk_ctx* ctx, int64_t bytes, void** ptr_out, unsigned char* handle_out);
ESTK_API int estk_peer_open(estk_ctx* ctx, const unsigned char* handle, void** ptr_out);
ESTK_API int estk_peer_close(estk_ctx* ctx, void* ptr);
ESTK_API int estk_peer_free(estk_ctx* ctx, void* ptr);
ESTK_API int estk_rank_grad_xr_adam(estk_ctx* ctx, const float* returns, const float* novelty,
                           float w_rew, float w_nov, int32_t P, int32_t world, int32_t rank,
                           const uint16_t* table16, const int64_t* offsets, const int32_t* order,
                           int32_t pair_begin, int32_t pairs_local, int64_t n,
                           void* const* peer_ws, float* theta, float* m, float* v,
                           estk_state* state, const estk_adam_desc* adam,
                           int32_t* ranks_out, int32_t* ranks2_out, float* grad_out, void* stream);

/* Epilogue on an all-reduced raw sum: g = grad_sum / P, negate, clamp, Adam.
 * theta/m/v NULL with grad_out set = gradient only (for non-Adam optimizers:
 * grad_out then receives clamp(-g), the tensor the reference stores in .grad). */
ESTK_API int estk_clamp_adam(estk_ctx* ctx, const float* grad_sum, int32_t P, int64_t n,
                    float* theta, float* m, float* v, estk_state* state,
                    const estk_adam_desc* adam, float* grad_out, void* stream);

/* ---- novelty (estorch.py:412-417): nov[i] = sum of the k smallest euclidean
 *      distances from bc[i] to the archive rows / ||archive||_F ---- */
ESTK_API int estk_knn_novelty(estk_ctx* ctx, const float* bc, int32_t count, const float* archive,
                     int32_t archive_len, int32_t dim, int32_t k, float* novelty_out,
                     void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ESTK_H_ */
