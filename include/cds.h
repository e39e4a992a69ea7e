/* cds.h -- C ABI of the H100 diffusion-sampling engine (libcds.so).
 *
 * The reference (CleanDiffuser) has no FFI of its own: its hot path is the Python loop
 * DiscreteDiffusionSDE.sample / ContinuousDiffusionSDE.sample (cleandiffuser/diffusion/diffusionsde.py:401-606,
 * :743-952) calling model["diffusion"](x_t, t, cond) -> ATen kernels once per op.  This header is the
 * boundary a maintainer would bind instead (ctypes stub in INTEGRATION.md): the per-iteration work of that
 * loop is described ONCE as a short program of fused operators, and the engine replays the program for
 * all reverse iterations from a CUDA graph with x_t resident on the device and no host round trip.
 *
 *   operator            replaces (reference file:line)
 *   ------------------  ------------------------------------------------------------------------------
 *   CDS_OP_CONV         nn.Conv1d / ConvTranspose1d / Linear (+bias) followed by GroupNorm1d + Mish, the
 *                       time/FiLM conditioning and the residual add of a ResidualBlock / ChiResidualBlock
 *                       (nn_diffusion/jannerunet.py:21-36,52-69, chiunet.py:13-45, utils/building_blocks.py:60-76),
 *                       the Linear(+Mish/SiLU/GELU) layers of DQLMlp and DiT1d (dqlmlp.py:22-29, dit.py:25-29,43-45)
 *   CDS_OP_LNMOD        LayerNorm(no affine) + adaLN modulate (dit.py:10-11,19,21,33,35,49)
 *   CDS_OP_ATTN         nn.MultiheadAttention core softmax(QK^T/sqrt(hd))V per (trajectory, head) (dit.py:20,34)
 *   CDS_OP_PREP         consistency-model re-noise + c_in pre-scale (consistency_model.py:257,423)
 *   CDS_OP_CAST         x.permute(0,2,1) entry of the UNets (jannerunet.py:169, chiunet.py:142): layout/dtype hand-over of x_t
 *   CDS_OP_UPDATE       CFG combine, clip_prediction, eps<->x0 conversion, the 8 solver updates, fix_mask
 *                       (diffusionsde.py:202,208-223,539-592) and the CM skip/out combine (consistency_model.py:257-262)
 *   CDS_OP_MHA          the attention core of nn.TransformerDecoderLayer's causal self-attention and masked cross-attention
 *                       (chitransformer.py: decoder with tgt_mask / memory_mask), q and k|v from separate strided sources
 *   CDS_OP_STASH ..     the backward of sample(requires_grad=True) over DQLMlp (diffusionsde.py:525-594 under autograd): per-
 *   CDS_OP_WGRAD        iteration stashes, the update's backward, Linear data / weight gradients (declared further down)
 *   CDS_OP_GN ..        classifier guidance inside the loop (diffusionsde.py:153-173 with CumRewClassifier over HalfJannerUNet1d):
 *   CDS_OP_GUIDE        GroupNorm + Mish over a kept pre-norm input, its backward, and pred += s[iter] * grad (further down)
 *   CDS_OP_HEAD_GRAD    the energy head of QGPO's classifier (qgpo_classifier.py / nn_classifier/mlp.py: 10 tanh(z / 10) over
 *                       an Mlp of Linear + SiLU): z = h . w + b per row and the seed of its backward (further down)
 *   (backward modes)    classifier guidance with CumRewClassifier over HalfDiT1d (nn_classifier/half_dit.py): CDS_OP_ATTN,
 *                       CDS_OP_LNMOD and CDS_OP_STASH given an upstream gradient compute their own backward (csrc/dit_grad.cuh)
 *   (no new kind)       classifier guidance with MSEClassifier / CumRewClassifier over MLPNNClassifier (mse_classifier.py,
 *                       nn_classifier/mlp.py): CDS_OP_CONV, CDS_OP_STASH and CDS_OP_DGRAD with CDS_ACT_RELU / SILU / MISH
 *   (kind + mode)       sample(requires_grad=True) with ContinuousConsistencyModel over DQLMlp (consistency_model.py:401-426
 *                       under autograd): CDS_OP_UPDATE_BWD's kind CM and CDS_OP_PREP's backward mode (gxin != NULL)
 *   (operand)           classifier guidance with ContinuousEDM (newedm.py:217-235): CDS_OP_UPDATE's guide / guide_s add the
 *                       term to the denoised D inside the EDM update
 *
 * Conventions
 *  - every function returns 0 on success, a negative cds_status otherwise; cds_last_error() gives the
 *    message (thread local).  No C++ exception or Python object crosses this ABI.
 *  - all pointers inside operator descriptors are DEVICE pointers owned by the caller (weights are the
 *    caller's parameter storage or caller-allocated packed copies; activations live in a caller-allocated
 *    workspace).  The library never allocates device memory on the hot path and never frees caller memory.
 *  - activations are "channels last": element (b, l, c) of a (batch, L, C) tensor sits at
 *    base + b*bstride + l*lstride + c (strides in elements), which is also the reference's public (b, horizon, dim)
 *    layout, so x_t needs no permute on entry or exit.  x_t, predictions and all tables are fp32; intermediate
 *    activations are fp32 (CDS_MATH_FP32 and CDS_MATH_TF32_TC programs) or bf16 (CDS_MATH_BF16_TC programs).
 *  - "per-iteration" operands are indexed by a device-resident iteration counter, so one captured graph
 *    serves every reverse iteration:  vec(b, c) = step[iter*step_stride + c] + sample[b*sample_stride + c]
 *    (either part may be NULL = 0).
 *  - a plan is not thread safe; distinct plans may be used concurrently.  All work is enqueued on the
 *    caller's stream (e.g. torch.cuda.current_stream()) and is asynchronous.
 */
#ifndef CDS_H_
#define CDS_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CDS_ABI_VERSION 12

typedef enum cds_status {
  CDS_OK = 0,
  CDS_ERR_INVALID = -1,      /* bad argument / unsupported shape (message says which) */
  CDS_ERR_CUDA = -2,         /* a CUDA runtime call failed */
  CDS_ERR_UNSUPPORTED = -3,  /* valid request the kernels cannot serve; caller should fall back */
  CDS_ERR_STATE = -4         /* call order violated (e.g. run before finalize) */
} cds_status;

typedef enum cds_op_kind { CDS_OP_CONV = 0, CDS_OP_UPDATE = 1, CDS_OP_LNMOD = 2, CDS_OP_ATTN = 3, CDS_OP_PREP = 4,
                           CDS_OP_CAST = 5, CDS_OP_MHA = 6,
                           /* differentiable sampling (sample(requires_grad=True) over DQLMlp, csrc/grad.cuh) */
                           CDS_OP_STASH = 7, CDS_OP_UPDATE_BWD = 8, CDS_OP_DGRAD = 9, CDS_OP_WGRAD = 10,
                           /* classifier guidance (the input gradient of HalfJannerUNet1d, csrc/classifier.cuh) */
                           CDS_OP_GN = 11, CDS_OP_GN_BWD = 12, CDS_OP_GUIDE = 13,
                           /* classifier guidance (the energy head of QGPOClassifier, csrc/classifier.cuh) */
                           CDS_OP_HEAD_GRAD = 14 } cds_op_kind;
typedef enum cds_act { CDS_ACT_NONE = 0, CDS_ACT_MISH = 1, CDS_ACT_SILU = 2, CDS_ACT_GELU_TANH = 3,
                       CDS_ACT_MISH_SILU = 4 /* silu(mish(x)): DiT's map_emb tail feeding every adaLN (dit.py:26,43,71) */,
                       CDS_ACT_LEAKY_RELU = 5 /* negative slope 0.01 (nn.LeakyReLU default; pearcemlp.py:44) */,
                       CDS_ACT_GELU_ERF = 6 /* exact GELU 0.5 x (1 + erf(x / sqrt 2)) (nn.GELU default; pearcemlp.py:30) */,
                       CDS_ACT_RELU = 7 /* max(x, 0); derivative z > 0 ? 1 : 0, 0 at z == 0 like ATen's threshold_backward
                                           (nn.ReLU, MLPNNClassifier's default activation: nn_classifier/mlp.py) */ } cds_act;
/* math mode of CDS_OP_CONV:
 *   CDS_MATH_FP32     fp32 CUDA-core FMA (bit-faithful to the fp32 oracle up to summation order)
 *   CDS_MATH_BF16_TC  wgmma tensor cores, bf16 operands and bf16 inter-layer activations, fp32 accumulation
 *   CDS_MATH_TF32_TC  wgmma tensor cores (.tf32): fp32 activations and weights in memory, read by the MMA as TF32
 *                     (10-bit mantissa), fp32 accumulation -- the arithmetic of the reference's own GPU path
 *                     (torch.backends.cudnn.allow_tf32 = True is PyTorch's default for convolutions)            */
typedef enum cds_math { CDS_MATH_FP32 = 0, CDS_MATH_BF16_TC = 1, CDS_MATH_TF32_TC = 2 } cds_math;
/* element type of an activation tensor.  CDS_TF32 is fp32 STORAGE whose values are rounded to the nearest TF32 (10-bit
 * mantissa, ties away from zero, like cvt.rna.tf32.f32) when an operator writes them: wgmma .tf32 ignores the low 13
 * mantissa bits of its fp32 operands (truncation), so an operand that is already rounded is read exactly and its rounding
 * error is unbiased and half as large.  Producers honour it on store; consumers read CDS_TF32 exactly like CDS_F32. */
typedef enum cds_dtype { CDS_F32 = 0, CDS_BF16 = 1, CDS_TF32 = 2 } cds_dtype;
/* update shapes; must match cleandiffuser_b200/diffusion/solvers.py */
typedef enum cds_update_kind { CDS_UPD_DDPM = 0, CDS_UPD_DDIM = 1, CDS_UPD_EPS = 2, CDS_UPD_X = 3, CDS_UPD_X2M = 4, CDS_UPD_CM = 5,
  /* ContinuousEDM (newedm.py:142-148, :411-431).  D = K0*x + K1*net (c_skip, c_out), clipped to [x_min, x_max] when final_clip;
   *   CDS_UPD_EDM       Euler step   d = (x - D)/SIGMA;  x <- x - d*K2 (K2 = sigma_i - sigma_{i-1});  when K4 != 0 the step is
   *                     the predictor of a Heun step: the old x goes to xhat_prev and d to aux
   *   CDS_UPD_EDM_HEUN  corrector    d' = (x - D)/SIGMA (x = the predictor's result, SIGMA = sigma_{i-1});
   *                     x <- xhat_prev - (aux + d')/2 * K2                                                              */
  CDS_UPD_EDM = 6, CDS_UPD_EDM_HEUN = 7 } cds_update_kind;

/* per-iteration coefficient row (floats), one row per reverse iteration */
enum { CDS_ROW_ALPHA = 0, CDS_ROW_SIGMA = 1, CDS_ROW_K0 = 2, CDS_ROW_K1 = 3, CDS_ROW_K2 = 4, CDS_ROW_K3 = 5,
       CDS_ROW_K4 = 6, CDS_ROW_KIND = 7, CDS_ROW_NOISE = 8 /* 1 + noise slot, 0 = no draw */, CDS_ROW_T = 9,
       CDS_ROW_XW = 10, CDS_ROW_DW = 11 /* EDM kinds: when XW != 0 the slope is XW*x - DW*D (the legacy EDM archetecture's
                                           x_weight / D_weight, edm.py:152) instead of (x - D)/SIGMA */,
       CDS_ROW_FLOATS = 12 };

/* vec(b, c) = step[iter*step_stride + c] + sample[b*sample_stride + c] */
typedef struct cds_vec {
  const float* step;   int64_t step_stride;
  const float* sample; int64_t sample_stride;
} cds_vec;

/* Fused 1-D convolution / linear layer as an implicit GEMM over rows (b, l_out):
 *   acc(b,l,n)  = sum_{tap,ci} in(b, l*stride + tap - pad, ci) * w[tap][ci][n]          (zero outside [0, L_in))
 *   y = acc + bias(b,n)
 *   if groups > 0:  y = GroupNorm(y; stats over L_out x (C_out/groups) per (b, group)) * gamma + beta
 *   y = act(y)
 *   y = y * scale(b,n) + shift(b,n)                 (each optional)
 *   y += res(b,l,n)                                  (identity shortcut, optional)
 *   y += sum_ci res_in(b,l,ci) * res_w[ci][n] + res_bias[n]   (1x1-conv shortcut, optional)
 *   out(b, l*phases + n / C_out, n % C_out) = y      (phases = 2 writes a stride-2 transposed conv's two
 *                                                     output phases; N = C_out*phases columns in w)           */
typedef struct cds_conv_op {
  int32_t batch, L_in, L_out, C_in, C_out, taps, stride, pad, phases;
  int32_t in_batch_mod;            /* >0: read in() at batch index b % in_batch_mod (CFG branches share x_t) */
  const void* in;   int64_t in_bstride;  int32_t in_lstride;   /* strides in ELEMENTS of the tensor's dtype */
  const void*  w;                  /* CDS_MATH_FP32: fp32 [taps*C_in][C_out*phases] (K rows, N contiguous)
                                      CDS_MATH_BF16_TC: bf16 [taps][C_out][C_in]     (K contiguous, TMA/wgmma K-major)
                                      CDS_MATH_TF32_TC: fp32 [taps][C_out][C_in]     (same packing, fp32 elements) */
  cds_vec bias;
  int32_t groups; const float* gn_gamma; const float* gn_beta; float gn_eps;
  int32_t act;
  cds_vec scale, shift;
  const void* res; int64_t res_bstride; int32_t res_lstride; int32_t res_batch_mod;
  const void* res_in; int64_t res_in_bstride; int32_t res_in_lstride; int32_t res_C;
  const void* res_w; const float* res_bias;   /* res_w: fp32 [res_C][C_out] (FP32) or bf16 / fp32 [C_out][res_C] (TC modes), as `w` */
  void* out; int64_t out_bstride; int32_t out_lstride;
  int32_t math;                    /* cds_math: which kernel family / weight layout */
  int32_t in_dtype, out_dtype, res_dtype, res_in_dtype;   /* cds_dtype of the activation tensors */
  /* > 1: the `sample` parts of bias / scale / shift belong to row-batch index b / sample_row_div (Linear layers over a token
   * stream flattened to batch*L rows of length-1 "sequences": one vector per trajectory = per L tokens).  Tensor-core path only. */
  int32_t sample_row_div;
} cds_conv_op;

/* out(b,l,:) = LayerNorm(in(b,l,:), eps, no affine) * (1 + scale(b,:)) + shift(b,:)
 *
 * Backward mode (dout != NULL; the input gradient of HalfDiT1d): out = d in of that expression given dout, the shift unused:
 *   dy = dout(b,l,:) * (1 + scale(b,:)),   xhat = (in - mean) * rstd
 *   out = rstd * (dy - mean_c(dy) - xhat * mean_c(dy * xhat))  [+ res(b,l,:)]
 *   gated(b,l,:) = gate(b,:) * out                                    (optional: gated != NULL)
 * mean and rstd are recomputed from `in` with the forward's arithmetic (fp32, two passes: the mean, then the mean of squared
 * deviations; rstd = rsqrt(var + eps)), one warp per token row, lane-strided sums reduced by a fixed xor butterfly.  dout +
 * b*dout_bstride + l*dout_lstride (dout_lstride 0: one row per trajectory broadcast over L); res, gated dense (batch, L, C);
 * gate + b*gate_bstride; out_dtype / gated_dtype CDS_F32 or CDS_TF32.  mod_bstride and gate_bstride may be 0 (one vector for
 * every trajectory: the [gamma - 1 | beta] table of an affine LayerNorm). */
typedef struct cds_lnmod_op {
  int32_t batch, L, C; float eps;
  const float* in; void* out;                   /* dense (batch, L, C); in fp32, out of out_dtype */
  const float* shift; const float* scale; int64_t mod_bstride;   /* per-trajectory vectors */
  int32_t out_dtype;                            /* cds_dtype: bf16 feeds the tensor-core Linear that follows */
  /* backward mode */
  const float* dout; int64_t dout_bstride; int32_t dout_lstride;
  const float* res;
  const float* gate; int64_t gate_bstride; float* gated; int32_t gated_dtype;
} cds_lnmod_op;

/* qkv dense (batch, L, 3*C) with [q | k | v] column blocks, heads split C evenly; out dense (batch, L, C)
 *
 * Backward mode (dout != NULL; the input gradient of HalfDiT1d): given dout = d out (dense (batch, L, C) fp32), out = d q|k|v,
 * dense (batch, L, 3*C) in qkv's layout.  Per (trajectory, head) the softmax P = softmax(q k^T / sqrt(hd)) is recomputed from
 * q and k (the forward keeps nothing), then dV = P^T dO, dS = P * (dO V^T - rowsum(P * dO V^T)), dQ = dS K / sqrt(hd),
 * dK = dS^T Q / sqrt(hd).  qkv fp32 storage (CDS_F32 / CDS_TF32), head_dim 16, 32 or 64, L <= 128 (else CDS_ERR_UNSUPPORTED);
 * out_dtype CDS_F32 or CDS_TF32.  fp32 CUDA-core FMA, one CTA per (trajectory, head), every sum in a fixed order (no atomics):
 * two runs are bitwise equal. */
typedef struct cds_attn_op {
  int32_t batch, L, C, heads;
  const void* qkv; void* out;
  int32_t out_dtype;                            /* cds_dtype of out */
  int32_t qkv_dtype;                            /* cds_dtype of qkv: bf16 (head_dim 32, L <= 128) runs on tensor cores (mma.sync) */
  const float* dout;                            /* backward mode */
} cds_attn_op;

/* Multi-head attention with separate query and key|value sources and an optional diagonal mask:
 *   out(b, i, h) = sum_{j in vis(i)} softmax_j(q(b,i,h) . k(b,j,h) / sqrt(hd)) v(b,j,h)     (fp32 softmax and accumulation)
 *   vis(i) = { j < Lk : j <= i + diag } when masked, else every j < Lk
 * q(b, i, :)   = q[b*q_bstride + i*q_lstride + (0..C)]                   (any column offset: point q at the first channel)
 * kv(b, j, :)  = kv_step[iter*kv_step_stride + j*kv_step_lstride + (0..2C)] + kv_sample[b*kv_sample_bstride + j*kv_sample_lstride
 *                + (0..2C)]    (either part may be NULL = 0; k = channels [0, C), v = channels [C, 2C); the cds_vec convention
 *                               extended to a sequence: a per-iteration token row and per-trajectory rows feed one attention)
 * heads split C evenly; head_dim = C / heads must be a multiple of 32 up to 256, and Lq, Lk <= 64 (else CDS_ERR_UNSUPPORTED).
 * q, kv_step and kv_sample are of in_dtype (CDS_F32, CDS_TF32 -- read as fp32 -- or CDS_BF16); strides in elements.
 * A query row without a visible key (masked, i + diag < 0) is written as zeros.
 * diag = 0 is causal self-attention; diag = 1 is ChiTransformer's memory mask t >= s - 1 (chitransformer.py). */
typedef struct cds_mha_op {
  int32_t batch, Lq, Lk, C, heads;
  int32_t masked, diag;
  const void* q; int64_t q_bstride; int32_t q_lstride;
  const void* kv_step; int64_t kv_step_stride; int32_t kv_step_lstride;
  const void* kv_sample; int64_t kv_sample_bstride; int32_t kv_sample_lstride;
  void* out; int64_t out_bstride; int32_t out_lstride;
  int32_t in_dtype, out_dtype;                  /* cds_dtype */
} cds_mha_op;

/* dense fp32 (batch, L, C_in) -> dense (batch, L, C_out) of out_dtype, channels [C_in, C_out) zero: gives x_t the
 * channel-padded form the tensor-core conv reads through TMA (the UNets' first conv has C_in = obs+act dims, e.g. 14:
 * 32 bf16 channels for CDS_MATH_BF16_TC, 16 fp32 channels for CDS_MATH_TF32_TC -- rows must be multiples of 16 bytes) */
typedef struct cds_cast_op {
  int32_t batch, L, C_in, C_out;
  const float* in; void* out;
  int32_t out_dtype;             /* cds_dtype of out */
} cds_cast_op;

/* consistency model: if row.NOISE: x += K2 * noise[slot];  xin = K3 * x
 *
 * Backward mode (gxin != NULL; sample(requires_grad=True) with the consistency model, csrc/grad.cuh): x <- x + K3 * gxin, IEEE
 * fp32 multiply then add, with x holding d x (the direct part the update's backward wrote) and gxin = d xin (batch, row).  The
 * re-noise is additive, so its gradient passes through unchanged.  K3 is read from coef + iter*coef_iter_stride (a signed
 * stride: the backward program walks the forward iterations in reverse); xin and noise are unused.  Forward descriptors keep
 * gxin NULL, and their row is coef + iter*CDS_ROW_FLOATS whatever coef_iter_stride holds. */
typedef struct cds_prep_op {
  int32_t batch, row;
  float* x; float* xin; const float* noise; const float* coef;
  const float* gxin; int64_t coef_iter_stride;      /* backward mode */
} cds_prep_op;

/* One reverse-process update on x (batch, row) in place; `coef` is the [n_iters][CDS_ROW_FLOATS] table.
 *   p = w_cfg*pred + w_uncond*pred_uncond       (if pred_uncond; w_uncond = 1-w_cfg)
 *   p = clip(p)  (eps-prediction: to [(x-alpha*x_max)/sigma, (x-alpha*x_min)/sigma]; x0-prediction: [x_min,x_max])
 *   x <- solver update of kind row.KIND with noise slot row.NOISE  ;  x = x*(1-mask) + prior*mask            */
typedef struct cds_update_op {
  int32_t batch, row;
  float* x;
  const float* pred; const float* pred_uncond; float w_cfg; float w_uncond;  /* w and (1-w), both rounded from double by the host */
  const float* noise;            /* [n_slots][...] pre-drawn N(0,1): slot s of this op's rows starts at noise + s*noise_slot_stride */
  int64_t noise_slot_stride;     /* floats between slots; 0 = batch*row (the op covers the whole tape) */
  const float* prior; const float* mask;      /* mask: `row` floats or NULL */
  const float* x_min; const float* x_max;     /* `row` floats or NULL */
  float* xhat_prev;              /* (batch,row) history for the 2M solvers / the EDM Heun corrector, or NULL */
  float* aux;                    /* (batch,row) second history buffer (EDM Heun: the predictor's slope) or NULL */
  const float* coef;
  int32_t predict_noise;
  int32_t final_clip;            /* CM only: clip the combined prediction to [x_min, x_max] */
  /* optional bf16 copy of the new x_t in the channel-padded form the tensor-core UNets read (what CDS_OP_CAST produces):
   * element (r, c) of the dense (rows, cast_C_in) view of x goes to x_cast[r*cast_C_out + c]; pad channels are never
   * written (a CDS_OPF_ONCE cast zeroes them and converts the initial x_t).  NULL = no copy. */
  void* x_cast; int32_t cast_C_in; int32_t cast_C_out;
  int32_t x_cast_dtype;          /* cds_dtype of x_cast */
  /* optional classifier-guidance term of kinds CDS_UPD_EDM / CDS_UPD_EDM_HEUN (ContinuousEDM, newedm.py:217-235): between the
   * c_skip / c_out combine and the clip, D <- D + guide_s[iter] * guide(b, e), IEEE fp32 multiply then add (no FMA contraction):
   * with guide_s = w * sigma^2 of the evaluation this is bit for bit the reference's D + (w * sigma ** 2) * grad.  guide: dense
   * (batch, row) fp32, the classifier's input gradient at the raw x_t; guide_s: one float per iteration.  NULL = no term (every
   * unguided program); the other kinds ignore it. */
  const float* guide; const float* guide_s;
} cds_update_op;

/* ---- backward operators of a differentiable reverse loop ------------------------------------------------------------
 * A differentiable program keeps, per iteration n, what its backward reads in "stashes": [n_iters][...] buffers written at
 * slot iter by the forward.  Every iteration-indexed operand below is `base + iter*iter_stride` (floats) with a SIGNED stride:
 * the backward program walks the forward iterations in reverse by pointing at the last slot with a negative stride, so that
 * one captured graph serves every backward iteration like it does every forward one. */

/* dst[iter*dst_iter_stride + i] = src[i] when dst != NULL;  act_out[i] = act(src[i]) when act_out != NULL (i < n); at least one
 * of the two.  act: CDS_ACT_NONE / MISH / SILU / RELU / GELU_TANH
 * Backward mode (grad != NULL): act_out[i] = grad[i] * act'(src[i]), src the stashed pre-activation, dst NULL; act MISH, SILU,
 * RELU (act' as CDS_OP_DGRAD applies it) or GELU_TANH (ATen's gelu_backward with approximate = "tanh"). */
typedef struct cds_stash_op {
  int64_t n;
  int32_t act;
  const float* src;
  float* dst; int64_t dst_iter_stride;
  float* act_out;
  const float* grad;
} cds_stash_op;

/* Backward of CDS_OP_UPDATE for kinds DDPM, DDIM, EPS, X and CM with a single prediction (no CFG combine, no history):
 *   in:  gx = d x_{n+1} (batch, row); the forward's operands x_n and the raw prediction from their stashes
 *   out: gpred = d pred;  gx <- the direct part of d x_n (through the update and clip_prediction's x_t-dependent bounds;
 *        the part through the network is added by the operators that follow)
 * fix_mask: d out = gx * (1 - mask).  clip_prediction follows torch.clip's tensor-bound gradient: an element equal to a bound
 * is not clipped (its gradient goes to pred), a clipped element's gradient goes to the bound, and an eps-prediction bound
 * (x - alpha*x_lim)/sigma passes it to x_t divided by sigma.
 * Kind CM (the consistency model, forward final_clip = 1; x_n is the re-noised x_t that CDS_OP_PREP wrote): f = K0*x + K1*pred
 * is recomputed with the forward's fp32 ops and clipped to [x_min, x_max] under the same rule (x_min > x_max: no element
 * passes); g' = the masked gradient where f passes, else 0; gpred = K1*g', gx = K0*g'.  predict_noise is ignored.
 * The kernel has no backward for kinds X2M, EDM and EDM_HEUN: a row of such a kind makes both outputs NaN. */
typedef struct cds_update_bwd_op {
  int32_t batch, row;
  float* gx; float* gpred;
  const float* x; int64_t x_iter_stride;
  const float* pred; int64_t pred_iter_stride;
  const float* mask;                       /* `row` floats or NULL */
  const float* x_min; const float* x_max;  /* `row` floats or NULL */
  const float* coef; int64_t coef_iter_stride;   /* row of iteration iter: coef + iter*coef_iter_stride (CDS_ROW_FLOATS) */
  int32_t predict_noise;
} cds_update_bwd_op;

/* Data gradient of a Linear layer:  out(r, k) [+]= (sum_n dz(r, n) W(n, k)) * act'(z(r, k))
 * dz (rows, N) row stride ldz; W (N, K) row stride ldw (a PyTorch [out, in] weight or a column block of one);
 * z = the stashed pre-activation of the layer's input (z + iter*z_iter_stride, dense (rows, K)), required when act = MISH, SILU
 *     or RELU (act' follows ATen: mish_backward, silu_backward's sig * (1 + z * (1 - sig)), and threshold_backward's
 *     z > 0 ? 1 : 0);
 * out (rows, K) row stride ldo, overwritten (accumulate = 0) or added to (1); out_sum (dense (rows, K), optional) += result.
 * fp32 CUDA cores; deterministic (every output is one thread's fixed-order sum). */
typedef struct cds_dgrad_op {
  int32_t rows, N, K;
  const float* dz; int32_t ldz;
  const float* w; int32_t ldw;
  const float* z; int64_t z_iter_stride;
  int32_t act, accumulate;
  float* out; int32_t ldo;
  float* out_sum;
} cds_dgrad_op;

/* Weight gradient of a Linear layer:  dw(n, k) [+]= sum_r dz(r, n) act(h(r, k));  db(n) [+]= sum_r dz(r, n)
 * dz (rows, N) row stride ldz; h = h + iter*h_iter_stride, (rows, K) row stride ldh, read through act (CDS_ACT_NONE or MISH:
 * the layer input recomputed from its stashed pre-activation); dw (N, K) row stride lddw; db + iter*db_iter_stride or NULL.
 * Deterministic: each output is summed over the rows in a fixed order by one thread, no atomics, so two runs are bitwise equal. */
typedef struct cds_wgrad_op {
  int32_t rows, N, K;
  const float* dz; int32_t ldz;
  const float* h; int64_t h_iter_stride; int32_t ldh; int32_t act;
  float* dw; int32_t lddw;
  float* db; int64_t db_iter_stride;
  int32_t accumulate;
} cds_wgrad_op;

/* ---- classifier guidance inside the loop ---------------------------------------------------------------------------------
 * The classifier's forward runs its convolutions as plain CDS_OP_CONV (no GroupNorm in the epilogue) so that the pre-norm
 * activation h survives for the backward; CDS_OP_GN normalises it.  The data gradients of the convolutions are CDS_OP_CONV with
 * re-packed weights.  GroupNorm statistics: per (b, group) over L x C/groups elements, fp32, two passes (mean, then the mean of
 * squared deviations), rstd = 1/sqrt(var + eps), every sum in one fixed order (no atomics): both operators compute the same
 * mean and rstd bit for bit.  h, res and dout are fp32 storage (CDS_F32 or CDS_TF32, read alike); strides in floats. */

/* out(b,l,c) = act(xhat(b,l,c) * gamma[c] + beta[c]) [+ vec(b, c)] [+ res(b,l,c)],  xhat = (h - mean) * rstd.
 * act: CDS_ACT_NONE / MISH.  out_dtype: CDS_F32 or CDS_TF32 (rounded on store). */
typedef struct cds_gn_op {
  int32_t batch, L, C, groups; float eps; int32_t act;
  const float* h; int64_t h_bstride; int32_t h_lstride;
  const float* gamma; const float* beta;
  cds_vec vec;
  const float* res; int64_t res_bstride; int32_t res_lstride;
  float* out; int64_t out_bstride; int32_t out_lstride; int32_t out_dtype;
} cds_gn_op;

/* Backward of CDS_OP_GN with respect to h (the vec and res terms do not depend on h):
 *   dxhat = gamma * dout * act'(y),  y = xhat * gamma + beta
 *   dh    = rstd * (dxhat - mean_g(dxhat) - xhat * mean_g(dxhat * xhat))
 * dh_dtype: CDS_F32 or CDS_TF32. */
typedef struct cds_gn_bwd_op {
  int32_t batch, L, C, groups; float eps; int32_t act;
  const float* h; int64_t h_bstride; int32_t h_lstride;
  const float* gamma; const float* beta;
  const float* dout; int64_t dout_bstride; int32_t dout_lstride;
  float* dh; int64_t dh_bstride; int32_t dh_lstride; int32_t dh_dtype;
} cds_gn_bwd_op;

/* pred(b, l, c) = pred(b, l, c) + s[iter] * g(b, l, c), IEEE fp32 multiply then add (no FMA contraction): with
 * s = -(w * sigma) this is bit for bit the reference's pred - (w * sigma) * grad.  pred dense (batch, L, C); g strided (an input
 * gradient may carry padding channels). */
typedef struct cds_guide_op {
  int32_t batch, L, C;
  float* pred;
  const float* g; int64_t g_bstride; int32_t g_lstride;
  const float* s;
} cds_guide_op;

/* The energy head of QGPO's classifier, logp = scale * tanh(z / scale), z = act(h(r, :)) . w + b, and the seed of its backward:
 *   seed(r) = ((1 * scale) * (1 - tanh(z / scale)^2)) / scale        (d sum(logp) / d z in autograd's order: the product's
 *                                                                        backward, tanh_backward, then the division's)
 * h (rows, K) row stride ldh, read through act (CDS_ACT_NONE or SILU: the head's input recomputed from the last hidden layer's
 * pre-activation); w: K floats (the [1, K] weight of an out_dim-1 Linear); b: 1 float; seed: rows floats.  One warp per row,
 * lane-strided partial sums reduced by a fixed xor butterfly: two runs are bitwise equal. */
typedef struct cds_head_grad_op {
  int32_t rows, K;
  const float* h; int32_t ldh; int32_t act;
  const float* w; const float* b;
  float scale;
  float* seed;
} cds_head_grad_op;

/* cds_op.flags */
enum { CDS_OPF_ONCE = 1 /* run once per cds_plan_run, before its first iteration, instead of in every iteration */,
       CDS_OPF_BRANCH_SHIFT = 8, CDS_OPF_BRANCH_MASK = 0xff00
       /* bits 8..15: branch index.  Operators of one branch run in program order; different branches are independent
        * chains (disjoint trajectories) that the engine enqueues on parallel streams / parallel graph branches and joins at
        * the end of every iteration, so that one chain's kernel boundaries overlap with the other chain's kernels. */ };

typedef struct cds_op {
  int32_t kind;                  /* cds_op_kind */
  int32_t flags;
  union { cds_conv_op conv; cds_update_op update; cds_lnmod_op lnmod; cds_attn_op attn; cds_prep_op prep; cds_cast_op cast;
          cds_mha_op mha; cds_stash_op stash; cds_update_bwd_op update_bwd; cds_dgrad_op dgrad; cds_wgrad_op wgrad;
          cds_gn_op gn; cds_gn_bwd_op gn_bwd; cds_guide_op guide; cds_head_grad_op head_grad; } u;
} cds_op;

typedef struct cds_plan cds_plan;

int         cds_version(void);
/* sizeof(cds_op) as compiled into the library -- bindings assert their struct mirror against it */
int         cds_op_size(void);
const char* cds_last_error(void);
/* number of SMs etc. of `device`, -1 on error; used by the host to size workspaces */
int         cds_device_sm_count(int device);

/* 1 if the tensor-core kernel of op->math (CDS_MATH_BF16_TC or CDS_MATH_TF32_TC; anything else is read as BF16_TC) can run
 * `op` as described (dtypes, strides, shapes; `w` may still be NULL), else 0: the host lowering asks before choosing the
 * weight layout; ops that are not eligible run on the CUDA-core kernel with math = CDS_MATH_FP32 (which accepts fp32 or
 * bf16 activations).  Pure host logic. */
int cds_conv_tc_supported(const cds_conv_op* op);

/* kernel families of CDS_OP_CONV (cds_conv_choice info[0]) */
enum { CDS_CONV_SIMT = 0 /* fp32 CUDA cores, conv_simt.cuh */, CDS_CONV_TC = 1 /* wgmma, conv_tc.cuh */,
       CDS_CONV_PS = 2 /* wgmma, position-sliced L = 4, conv_ps.cuh */ };
/* The kernel instantiation cds_plan_append / cds_run_op would choose for `op`.  Pure host logic.  The data pointers in, out and
 * w (and res_in, gn_gamma, gn_beta, res_bias) may be NULL: only their alignment is read.  res, res_w and the step / sample
 * parts of bias, scale and shift are presence flags as well: NULL means the operand is absent, which changes the choice.
 * info[0] = family; CDS_CONV_TC: info[1..6] = KC, N (CTA tile columns), SPLIT, runtime column
 * tiles, HAS_RES (1x1 shortcut conv), TF32; CDS_CONV_PS: info[1..6] = KC, N, 1, 1, HAS_RES, TF32; CDS_CONV_SIMT: info[2] = BN.
 * Unused entries are 0.  Returns 0, or the negative cds_status with which the op would be refused. */
int cds_conv_choice(const cds_conv_op* op, int32_t info[8]);

/* kernel families of CDS_OP_ATTN (cds_attn_choice info[0]) */
enum { CDS_ATTN_F32 = 0 /* fp32 CUDA cores, attention_f32_kernel<HD> */, CDS_ATTN_BF16_MMA = 1 /* mma.sync bf16, head_dim 32 */,
       CDS_ATTN_TF32_TMA = 3 /* mma.sync tf32, head_dim 32, persistent and TMA-fed, attention_tma.cuh<NT> */ };
/* The attention kernel cds_plan_append / cds_run_op would choose for `op`.  Pure host logic: only the alignment of qkv and out
 * is read (they may be NULL).  info[0] = family; info[1] = HD (CDS_ATTN_F32), NT = ceil(L / 8) (CDS_ATTN_TF32_TMA), else 0;
 * info[2] = head_dim; info[3] = dynamic shared memory of the launch in bytes (0 for CDS_ATTN_BF16_MMA).  Returns 0, or the
 * negative cds_status with which the op would be refused. */
int cds_attn_choice(const cds_attn_op* op, int32_t info[4]);

/* The CDS_OP_MHA kernel cds_plan_append / cds_run_op would run `op` on.  Pure host logic: no pointer is dereferenced (they may
 * be NULL).  info[0] = head_dim / 32 (the template parameter HPL of mha_f32_kernel: head channels per lane), info[1] = 1 when
 * q / k / v are bf16 (else 0).  Returns 0, or the negative cds_status with which the op would be refused. */
int cds_mha_choice(const cds_mha_op* op, int32_t info[2]);

/* A plan = the per-iteration operator program for one (model, shape, option set) on one device. */
int cds_plan_create(int device, cds_plan** out);
int cds_plan_destroy(cds_plan* plan);
/* Append operators (copied).  Pointers inside must stay valid until the plan is destroyed or rebuilt. */
int cds_plan_append(cds_plan* plan, const cds_op* ops, int32_t n_ops);
/* Validate shapes, choose kernels, allocate the 4-byte device iteration counter. n_iters = rows in coef tables. */
int cds_plan_finalize(cds_plan* plan, int32_t n_iters);
/* Enqueue iterations [first, first+count) on `stream` (a cudaStream_t): CDS_OPF_ONCE operators first, then `count`
 * replays of the iteration program.  The first call captures the program into a CUDA graph; later calls replay it.
 * use_graph = 0 launches kernels directly (debug/ncu).  Consecutive tensor-core conv kernels are chained with
 * programmatic dependent launch (the next kernel's prologue and weight prefetch overlap the previous kernel's tail);
 * CDS_PDL=0 in the environment switches that off.  It is latched at each kernel instantiation's first launch: an instantiation
 * already launched ignores later changes, one first launched after a change reads the new value. */
int cds_plan_run(cds_plan* plan, int32_t first, int32_t count, void* stream, int32_t use_graph);
/* Single-step entry ("cds_step"): enqueue operators [op_first, op_first + op_count) of the program (indices into the appended
 * operator list; CDS_OPF_ONCE operators inside the range are skipped) for iteration `iter` with direct launches -- the device
 * iteration counter is set to `iter` first.  This is how a host callback is interleaved with the loop (classifier guidance,
 * diffusionsde.py:153-173: the denoiser operators run, PyTorch adds the guidance term to the prediction in place, then the
 * update operator runs); `cds_plan_run(plan, first, 0, ...)` runs the CDS_OPF_ONCE operators alone, and
 * `cds_plan_run(plan, i, 1, ...)` is the whole iteration i. */
int cds_plan_run_range(cds_plan* plan, int32_t iter, int32_t op_first, int32_t op_count, void* stream);
/* Run iteration `iter` once with direct launches, bracketing every operator with CUDA events on `stream`;
 * ms_per_op[i] receives the device time of operator i (n_ops entries; CDS_OPF_ONCE operators are run and timed first).
 * Synchronises `stream`.  For bench.py's live per-kernel roofline; note that it advances x_t like a normal iteration. */
int cds_plan_profile(cds_plan* plan, int32_t iter, void* stream, float* ms_per_op, int32_t n_ops);
/* Number of kernel launches one iteration of the program performs (for bench.py's gpu_launches). */
int cds_plan_launches_per_iter(const cds_plan* plan);

/* Debug: record a clock64 timeline (64 slots per CTA, layout in csrc/conv_tc.cuh) of the `target_launch`-th tensor-core conv
 * launch issued from now on into `device_buffer` (int64 entries); NULL switches tracing off.  Returns the grid size of the
 * launch traced since the previous call (0 if none). */
int cds_debug_trace(void* device_buffer, int64_t capacity_entries, int32_t target_launch);

/* Stand-alone operator launch (parity tests of single kernels): runs `op` once with iteration index `iter`. */
int cds_run_op(int device, const cds_op* op, int32_t iter, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* CDS_H_ */
