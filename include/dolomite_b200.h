/*
 * dolomite_b200.h -- C ABI of the H100-native (sm_90a) hot path of dolomite-engine.
 *
 * Scope: the data-parallel GPTDolomite / MoEDolomite training step (SURVEY.md section 8).  The reference
 * (ibm-granite/dolomite-engine @ 2024_08_07) is pure Python and reaches its GPU kernels through
 * torch / flash-attn / scattermoe; it has no FFI of its own.  Every entry point below therefore cites
 * the reference *call site* (file:line under dolomite_engine/) whose arithmetic it replaces.  The Python
 * host side (dolomite_engine_b200/) binds these with ctypes; INTEGRATION.md shows the stub a reference
 * maintainer would add.
 *
 * Conventions
 *   - every function returns 0 (DOLO_OK) or a negative error code; dolomite_b200_last_error() returns a
 *     thread-local human readable message for the last failure on the calling thread.
 *   - all pointers are DEVICE pointers unless the name ends in _host.  The callee never allocates, frees
 *     or retains device memory and never synchronises the stream.
 *   - `stream` is a cudaStream_t passed as void*.
 *   - results are bit-identical from run to run on the same inputs (every reduction sums in a fixed order), except
 *     for the split-K flag of dolomite_b200_gemm_bf16.
 *   - activations/weights are bf16 (uint16 storage), statistics / master weights / gradients-of-weights fp32.
 *   - row-major everywhere; `ld*` are leading dimensions in ELEMENTS.
 */
#ifndef DOLOMITE_B200_H
#define DOLOMITE_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DOLOMITE_B200_ABI_VERSION 1

#define DOLO_OK 0
#define DOLO_ERR_INVALID (-1) /* bad argument / unsupported shape */
#define DOLO_ERR_CUDA (-2)    /* CUDA runtime / driver error     */

/* library management (no reference counterpart): thread-local text of the last error, ABI version, device query */
const char* dolomite_b200_last_error(void);
int dolomite_b200_abi_version(void);
int dolomite_b200_device_info(int* sm_count, int* cc_major, int* cc_minor);
/* process-wide tuning knobs:
 *   "gemm_sm_margin"   SMs the persistent GEMM grids leave free for concurrent communication kernels
 *   "attn_head_fastest" heads per chunk of the attention CTA order (default 8: inside a chunk heads fastest + longest tiles
 *                      first, so that the last wave is short tiles; 0 = tiles fastest)
 *   "gemm_l2_hints"    1 | 0 (long-contraction GEMMs load the streamed operand evict-first and the re-used one evict-last)
 *   "gemm_tile_n"      0 (default) | 128 | 256: output tile width of the dense bf16 GEMMs (gemm_bf16 without split-K and
 *                      gemm_bf16_wgrad_multi); 0 chooses per launch (dolomite_b200_gemm_bf16_tile_n), 128 / 256 force a
 *                      width (diagnostics and tests; both widths give bit-identical results)
 * Accepted and reported back, but without effect on sm_90 (one kernel per job): "gemm_cta_pair", "gemm_dynamic",
 * "gemm_f32_tma_epilogue", "attn_fwd_split", "attn_bwd_variant", "attn_bwd_ablate". */
int dolomite_b200_set_option(const char* key, int value);
int dolomite_b200_get_option(const char* key, int* value);

/* ------------------------------------------------------------------------------------------------
 * RMSNorm  -- hf_models/modeling_utils/normalization/rmsnorm/base.py:18-25
 *   y = w * bf16( x32 * rsqrt(mean(x32^2) + eps) ), rstd saved for backward.
 *   bwd: dx (+ optional dx_add, the residual-stream gradient), dw accumulated (+=) into fp32.
 *   workspace for bwd: dolomite_b200_rmsnorm_bwd_workspace_bytes(H) bytes.
 * ------------------------------------------------------------------------------------------------ */
int dolomite_b200_rmsnorm_fwd(const void* x, const void* w, void* y, float* rstd, int64_t T, int H, float eps,
                              void* stream);
int64_t dolomite_b200_rmsnorm_bwd_workspace_bytes(int H);
int dolomite_b200_rmsnorm_bwd(const void* dy, const void* x, const void* w, const float* rstd, const void* dx_add,
                              void* dx, float* dw_accum, void* workspace, int64_t T, int H, void* stream);

/* ------------------------------------------------------------------------------------------------
 * RoPE on the packed qkv buffer, in place -- hf_models/modeling_utils/position_embedding/rope.py:104-114,
 *   call sites attention/padding_free.py:38-40; cos/sin gather gpt_dolomite/base.py:289-296.
 *   qkv rows are `n_groups` groups of (q_per_group + 2) head slots of head_dim (layouts of
 *   attention/padding_free.py:79-116: mha = nh groups x [q,k,v]; gqa = nkv groups x [q*g,k,v]; mqa = 1 group).
 *   The first q_per_group+1 slots of each group (queries and the key) are rotated.
 *   cos/sin: bf16 tables [n_positions, head_dim]; position_ids int32 or int64 [T].
 *   inverse != 0 applies the transpose rotation (backward).
 * ------------------------------------------------------------------------------------------------ */
int dolomite_b200_rope_qk_inplace(void* qkv, int64_t row_stride, int64_t T, int n_groups, int q_per_group,
                                  int head_dim, const void* cos_table, const void* sin_table, const void* position_ids,
                                  int position_ids_is_int64, int64_t n_positions, int inverse, void* stream);

/* ------------------------------------------------------------------------------------------------
 * LayerNorm -- normalization_function "layernorm" = torch.nn.LayerNorm
 * (hf_models/modeling_utils/normalization/layernorm/__init__.py): fp32 statistics, one rounding to bf16:
 *   y = bf16((x - mean) * rstd * w + b);  b may be null.  mean / rstd (fp32 [T]) are saved for backward.
 * bwd: dx = rstd * (g*w - mean(g*w) - xhat * mean(g*w*xhat)) [+ dx_add];  dw_accum += sum g*xhat;  db_accum += sum g.
 * workspace: dolomite_b200_layernorm_bwd_workspace_bytes(H) bytes, 16-byte aligned.
 * ------------------------------------------------------------------------------------------------ */
int dolomite_b200_layernorm_fwd(const void* x, const void* w, const void* b, void* y, float* mean, float* rstd, int64_t T,
                                int H, float eps, void* stream);
int64_t dolomite_b200_layernorm_bwd_workspace_bytes(int H);
int dolomite_b200_layernorm_bwd(const void* dy, const void* x, const void* w, const float* mean, const float* rstd,
                                const void* dx_add, void* dx, float* dw_accum, float* db_accum, void* workspace, int64_t T,
                                int H, void* stream);

/* ------------------------------------------------------------------------------------------------
 * MLP activations -- activation_function of gpt_dolomite/mlp.py:27-36 and moe_dolomite/moe/base.py:88-93, resolved by
 * hf_models/modeling_utils/activations/{__init__,base,glu}.py (host side: dolomite_engine_b200/activations.py).
 * Functions (torch's default constructor arguments): */
enum {
    DOLO_ACT_CELU = 0,     /* alpha 1 */
    DOLO_ACT_ELU,          /* alpha 1 */
    DOLO_ACT_GELU,         /* exact erf */
    DOLO_ACT_GELU_TANH,    /* approximate="tanh" */
    DOLO_ACT_SELU,
    DOLO_ACT_HARDSHRINK,   /* lambda 0.5 */
    DOLO_ACT_HARDSIGMOID,
    DOLO_ACT_HARDSWISH,
    DOLO_ACT_HARDTANH,     /* [-1, 1] */
    DOLO_ACT_LAPLACE,      /* transformers' LaplaceActivation, mu 0.707107, sigma 0.282095 */
    DOLO_ACT_LEAKY_RELU,   /* slope 0.01 */
    DOLO_ACT_LOG_SIGMOID,
    DOLO_ACT_MISH,
    DOLO_ACT_RELU,
    DOLO_ACT_RELU2,        /* relu(x)^2 */
    DOLO_ACT_RELU6,
    DOLO_ACT_SIGMOID,
    DOLO_ACT_SILU,
    DOLO_ACT_SOFTPLUS,     /* beta 1, threshold 20 */
    DOLO_ACT_SOFTSHRINK,   /* lambda 0.5 */
    DOLO_ACT_SOFTSIGN,
    DOLO_ACT_TANH,
    DOLO_ACT_TANHSHRINK,
    DOLO_ACT_COUNT
};
/* Forms:
 *   DOLO_ACT_PLAIN        x [T, F]:  y = f(x)
 *   DOLO_ACT_GLU          x [T, 2F] = [u | g]:  y = u * bf16(f(g))     (GLUActivation, activations/glu.py)
 *   DOLO_ACT_SIGMOID_GLU  x [T, 2F] = [u | g]:  y = u * sigmoid(g), rounded once (nn.GLU, names "glu" / "sigmoid_glu");
 *                         DOLO_ACT_SIGMOID only
 * Where the reference's eager module rounds to bf16 more than once (laplace, softsign, tanhshrink) f rounds at the same
 * points.  bwd: plain dx = dy * f'(x); both GLU forms du = dy * f(g), dg = dy * u * f'(g); f' takes torch autograd's
 * value at non-differentiable points.  dbias_accum (fp32 [F] or [2F], may be null) += column sums of the bf16 dx (bias
 * gradient of c_fc), summed in a fixed order.  F is a positive multiple of 8, pointers 16-byte aligned. */
enum { DOLO_ACT_PLAIN = 0, DOLO_ACT_GLU = 1, DOLO_ACT_SIGMOID_GLU = 2 };
int dolomite_b200_act_fwd(int act_id, int form, const void* x, void* y, int64_t T, int64_t F, void* stream);
int dolomite_b200_act_bwd(int act_id, int form, const void* dy, const void* x, void* dx, float* dbias_accum, int64_t T,
                          int64_t F, void* stream);
/* act_bwd on rows grouped into segments (MoE expert rows): segment s is rows [seg_offsets[s], seg_offsets[s+1]) (int32
 * device table of num_segments + 1 entries, e.g. the offsets_padded of moe_route), dx is written on those rows only, and
 * row s of dbias_accum (fp32 [num_segments, ld_dbias]) += the column sums of the segment's bf16 dx, in the fixed order of
 * the dense launch.  An empty segment adds exact zeros. */
int dolomite_b200_act_bwd_segmented(int act_id, int form, const void* dy, const void* x, void* dx, float* dbias_accum,
                                    int64_t ld_dbias, int64_t F, const int32_t* seg_offsets, int num_segments,
                                    void* stream);

/* ------------------------------------------------------------------------------------------------
 * tanh-GELU -- activation_function "gelu_pytorch_tanh" (hf_models/modeling_utils/activations/base.py), the non-GLU MLP
 * of gpt_dolomite/mlp.py:45-50.  bwd: dx = dy * gelu'(x); dbias_accum (fp32 [F], may be null) += column sums of the
 * bf16 dx (bias gradient of c_fc).  Same kernels as dolomite_b200_act_fwd / _bwd(DOLO_ACT_GELU_TANH, DOLO_ACT_PLAIN).
 * ------------------------------------------------------------------------------------------------ */
int dolomite_b200_gelu_fwd(const void* x, void* y, int64_t n, void* stream);
int dolomite_b200_gelu_bwd(const void* dy, const void* x, void* dx, float* dbias_accum, int64_t T, int64_t F, void* stream);

/* ------------------------------------------------------------------------------------------------
 * SwiGLU -- hf_models/modeling_utils/activations/glu.py:26-28 with gpt_dolomite/mlp.py:54-55 ordering:
 *   x = [up | gate] (first F columns up, last F gate);  y = up * silu(gate).
 *   Same kernels as dolomite_b200_act_fwd / _bwd(DOLO_ACT_SILU, DOLO_ACT_GLU).
 * ------------------------------------------------------------------------------------------------ */
int dolomite_b200_swiglu_fwd(const void* x, void* y, int64_t T, int64_t F, void* stream);
int dolomite_b200_swiglu_bwd(const void* dy, const void* x, void* dx, int64_t T, int64_t F, void* stream);
/* Same, and additionally accumulates the bias gradient of the linear layer that produced x (autograd of
 * ParameterizedLinear's `+ bias`, modeling_utils/linear.py): dbias_accum[0..2F) += column sums of the bf16 dx written. */
int dolomite_b200_swiglu_bwd_bias(const void* dy, const void* x, void* dx, float* dbias_accum, int64_t T, int64_t F,
                                  void* stream);

/* ------------------------------------------------------------------------------------------------
 * Embedding -- gpt_dolomite/base.py:351-372 (wte gather, * m_emb); bwd accumulates (+=) into fp32 dwte.
 *   ids int64 [T].  Out-of-range ids are an error on the host side (checked by the caller), the kernel clamps.
 * ------------------------------------------------------------------------------------------------ */
int dolomite_b200_embedding_fwd(const int64_t* ids, const void* wte, void* out, int64_t T, int H, int64_t V,
                                float scale, void* stream);
int dolomite_b200_embedding_bwd(const int64_t* ids, const void* dout, float* dwte, int64_t T, int H, int64_t V,
                                float scale, void* stream);
/* The gather with NEFTune noise (model_wrapper/base.py:246-267, training mode): out = bf16(wte[ids] + v) with
 * v = uniform(-mag, mag) at the rounding points of torch's CUDA uniform kernel on a bf16 tensor (bounds and range in bf16,
 * bf16(u * range + from) in fp32, a value equal to the upper bound becomes the lower one).  u in (0, 1] is a counter hash of
 * the flat element index t * H + c under (key0, key1) (kernels.dropout_keys), so a pass's noise is a pure function of
 * its keys.  mag: the reference's alpha / sqrt(numel), in fp32, > 0. */
int dolomite_b200_embedding_fwd_neft(const int64_t* ids, const void* wte, void* out, int64_t T, int H, int64_t V,
                                     uint32_t key0, uint32_t key1, float mag, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Cross entropy (mean over non-ignored tokens), fused forward + backward --
 *   model_wrapper/pretraining.py:124-125 (F.cross_entropy on [T,V]) and gpt_dolomite/main.py:185-200.
 *   logits bf16 [T, ldl]; labels int64 [T]; label == ignore_index contributes nothing.  Any V in [1, 131072] with
 *   ldl % 8 == 0 and ldl >= V: columns [V, ldl) are never read as data (they may hold anything, NaN included) and
 *   receive 0 in dlogits where the last 16-byte vector of a row straddles V.
 *   Writes per-token loss (fp32, 0 for ignored), the scalar mean loss, and overwrites dlogits (may alias
 *   logits) with (softmax - onehot) * grad_scale / n_valid in bf16.
 *   scratch: 2 floats.  logit_scale multiplies logits before the softmax (1/m_width, gpt_dolomite/main.py:155-156).
 * ------------------------------------------------------------------------------------------------ */
int dolomite_b200_cross_entropy_fwd_bwd(const void* logits, int64_t ldl, const int64_t* labels, void* dlogits,
                                        float* loss_per_token, float* loss_mean, float* scratch, int64_t T, int64_t V,
                                        int64_t ignore_index, float logit_scale, float grad_scale, void* stream);
/* The same computation in three steps, for an LM head that never materialises [T, V] (gpt_dolomite/main.py:172-177 +
 * model_wrapper/pretraining.py:107-127 fused): `_count` leaves the number of labels != ignore_index of the WHOLE batch in
 * scratch[0]; `_rows` handles any chunk of rows (logits of the chunk, its labels, its slice of loss_per_token) and may be
 * called once per chunk; `_mean` reduces loss_per_token [T] to the scalar loss.  A label outside [0, V) that is not
 * ignore_index traps (device-side assert, like torch). */
int dolomite_b200_cross_entropy_count(const int64_t* labels, int64_t T, int64_t ignore_index, float* scratch,
                                      void* stream);
int dolomite_b200_cross_entropy_rows(const void* logits, int64_t ldl, const int64_t* labels, void* dlogits,
                                     float* loss_per_token, const float* scratch, int64_t T, int64_t V,
                                     int64_t ignore_index, float logit_scale, float grad_scale, void* stream);
int dolomite_b200_cross_entropy_mean(const float* loss_per_token, int64_t T, const float* scratch, float* loss_mean,
                                     void* stream);

/* ------------------------------------------------------------------------------------------------
 * Column sum (bias gradient of nn.Linear, autograd of linear.py:5-25):  out[n] += scale * sum_t x[t, n]
 * ------------------------------------------------------------------------------------------------ */
int dolomite_b200_colsum_accum(const void* x, int64_t ldx, float* out, int64_t T, int64_t N, float scale,
                               void* stream);
/* Per-segment column sums (bias gradient of the MoE expert linears): out[s * ld_out + n] += scale * sum of x[t, n] over
 * the rows t of segment s, [seg_offsets[s], seg_offsets[s+1]) (int32 device table of num_segments + 1 entries).  Same
 * summation order per segment as colsum_accum over those rows; no float atomics; an empty segment adds exact zeros. */
int dolomite_b200_colsum_accum_segmented(const void* x, int64_t ldx, float* out, int64_t ld_out, int64_t N,
                                         const int32_t* seg_offsets, int num_segments, float scale, void* stream);
/* x[i] *= scale[0]  (bf16 in place; scale is a DEVICE scalar: the upstream gradient autograd hands to the loss when the
 * caller does anything but `loss.backward()`, train_utils.py:61-90) */
int dolomite_b200_scale_bf16_by_device_scalar(void* x, int64_t n, const float* scale, void* stream);

/* out = a + alpha * b  (bf16; residual adds of gpt_dolomite/layer.py:70-85), a/b/out may alias */
int dolomite_b200_add_scaled(const void* a, const void* b, void* out, float alpha, int64_t n, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Training-mode dropout on flat bf16 activations -- nn.Dropout at gpt_dolomite/base.py:138 (after the embeddings),
 * attention/base.py:92 + padding_free.py:75 (after the attention c_proj), gpt_dolomite/mlp.py:43-49 (after the MLP c_proj),
 * moe_dolomite/moe/base.py:106-120 -- fused with the `* m_residual` / `* m_emb` and `+ residual` that follow it
 * (gpt_dolomite/layer.py:73-86, base.py:368-371), each with the reference's own bf16 rounding:
 *   fwd: out = [residual +] bf16(bf16(x * s) * post_mul)      s = 1 / (1 - p) on kept elements, 0 on dropped ones
 *   bwd: dx  = bf16(bf16(dy * pre_mul) * s)
 * The mask is a counter-based hash of (element index, key0, key1): backward and re-computed (checkpointed) blocks regenerate
 * it from the same keys.  p in [0, 1); n % 8 == 0; residual may be NULL; out may alias x / residual, dx may alias dy.
 * ------------------------------------------------------------------------------------------------ */
int dolomite_b200_dropout_fwd(const void* x, const void* residual, void* out, int64_t n, float p, float post_mul,
                              uint32_t key0, uint32_t key1, void* stream);
int dolomite_b200_dropout_bwd(const void* dy, void* dx, int64_t n, float p, float pre_mul, uint32_t key0, uint32_t key1,
                              void* stream);

/* ------------------------------------------------------------------------------------------------
 * Optimizer-side flat-shard kernels (train_utils.py:99-106: clip_grad_norm_ + AdamW step).
 *   sumsq: out[0] += sum(g^2)  (fp32 grads), summed in a fixed order (bit-identical from run to run); workspace:
 *   dolomite_b200_sumsq_workspace_bytes() bytes, 4-byte aligned.   clip coef: coef = min(1, max_norm / (sqrt(sumsq) + 1e-6)),
 *   NaN for a NaN norm (torch.clamp); 1 when max_norm <= 0.
 *   adamw: torch.optim.AdamW semantics on fp32 master shard; also emits the bf16 copy that the next
 *   all-gather ships.  `clip_coef` is a device pointer (nullable -> 1).  step >= 1.
 * ------------------------------------------------------------------------------------------------ */
int64_t dolomite_b200_sumsq_workspace_bytes(void);
int dolomite_b200_sumsq_accum(const float* g, int64_t n, float* out, void* workspace, void* stream);
int dolomite_b200_clip_coef(const float* sumsq, float max_norm, float* coef_out, float* norm_out, void* stream);
int dolomite_b200_adamw_step(float* p, const float* g, float* m, float* v, void* p_bf16, int64_t n, float lr,
                             float beta1, float beta2, float eps, float weight_decay, int64_t step,
                             const float* clip_coef, void* stream);
/* fp32 -> bf16 cast of a flat shard (FSDP MixedPrecision param_dtype = bf16, distributed/__init__.py:34-44);
 * bf16 reduce-scatter output -> fp32 shard gradient accumulate (reduce_dtype = bf16, same table) */
int dolomite_b200_cast_f32_to_bf16(const float* src, void* dst, int64_t n, void* stream);
int dolomite_b200_accum_bf16_into_f32(const void* src, float* dst, float scale, int64_t n, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Single-query attention over a KV cache (decoding with `past_key_values`: attention/sdpa.py:11-83, attention/flash.py:16-140;
 * model_wrapper/base.py:110-136 `generate`).  One new token per sequence:
 *   qkv      bf16 [batch, row_stride]: the packed c_attn output of the new tokens (RoPE applied); only the q slots are read
 *   k_cache / v_cache  bf16 [batch, L_max, n_groups * head_dim]: keys / values by position (the new token already appended)
 *   lens     int32 [batch]: valid positions per sequence INCLUDING the new token
 *   out      bf16 [batch, n_heads * head_dim]
 * ------------------------------------------------------------------------------------------------ */
int dolomite_b200_attn_decode(const void* qkv, int64_t row_stride, const void* k_cache, const void* v_cache, const int32_t* lens,
                              void* out, int batch, int64_t L_max, int n_groups, int q_per_group, int head_dim,
                              float softmax_scale, void* stream);
/* The same with ALiBi (eager / SDPA attention of a `position_embedding_type: alibi` model decoding with a mask:
 * model_wrapper/base.py:110-136 `generate` -> gpt_dolomite/base.py:261-287 `_get_alibi_bias`, :559-598
 * `_get_maybe_causal_mask`): the score of cache position k of head h gets bias bf16(alibi_slopes[h] * k).
 *   alibi_slopes  fp32 [n_heads], the reference's slopes (modeling_utils/position_embedding/alibi.py:32-44); null is an
 *                 error. */
int dolomite_b200_attn_decode_alibi(const void* qkv, int64_t row_stride, const void* k_cache, const void* v_cache,
                                    const int32_t* lens, void* out, int batch, int64_t L_max, int n_groups, int q_per_group,
                                    int head_dim, float softmax_scale, const float* alibi_slopes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Attention of several new tokens per sequence against a KV cache (a forward with `past_key_values` and a query block of
 * n tokens: gpt_dolomite/base.py:173-257 and :300-349, the causal mask of a query block that starts past_length keys in;
 * attention/sdpa.py:11-83).  Sequence b has past[b] cached tokens and n[b] = cu_new[b+1] - cu_new[b] >= 0 new ones;
 * new token i of b attends to cache positions 0 .. past[b] + i.  fp32 online softmax, output rounded to bf16 once; no
 * dropout (inference only).  n[b] == 0: nothing is computed or written for b.
 *   qkv      bf16 [sum n, row_stride]: packed c_attn output of the new tokens (RoPE applied); only the q slots are read
 *   cu_new   int32 [batch + 1]: token rows of each sequence's new tokens in qkv / out
 *   past     int32 [batch]: cached tokens before the new ones
 *   k_cache / v_cache  bf16 [batch, L_max, n_groups * head_dim]: keys / values by position, the new tokens' already
 *            written at past[b] .. past[b] + n[b] - 1
 *   out      bf16 [sum n, n_heads * head_dim]
 *   max_new  host upper bound of n[b] (sets the grid); max_end host upper bound of past[b] + n[b], at most L_max
 *   head_dim: 16, 32, 64, 80, 96, 128, 160, 192 or 256.  qkv, the caches and out 16-byte aligned, row_stride % 8 == 0.
 * The _alibi form adds bf16(alibi_slopes[h] * k) to the logit of cache position k of head h, as attn_decode_alibi.
 * ------------------------------------------------------------------------------------------------ */
int dolomite_b200_attn_cache(const void* qkv, int64_t row_stride, const int32_t* cu_new, const int32_t* past,
                             const void* k_cache, const void* v_cache, void* out, int batch, int max_new, int max_end,
                             int64_t L_max, int n_groups, int q_per_group, int head_dim, float softmax_scale, void* stream);
int dolomite_b200_attn_cache_alibi(const void* qkv, int64_t row_stride, const int32_t* cu_new, const int32_t* past,
                                   const void* k_cache, const void* v_cache, void* out, int batch, int max_new, int max_end,
                                   int64_t L_max, int n_groups, int q_per_group, int head_dim, float softmax_scale,
                                   const float* alibi_slopes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * bf16 GEMM on Hopper tensor cores (TMA -> smem -> wgmma -> register accumulators -> epilogue), replacing the cuBLAS
 * calls behind nn.Linear (linear.py:5-25; call sites attention/base.py:100, padding_free.py:74,
 * gpt_dolomite/mlp.py:46-48, gpt_dolomite/main.py:172-177) and their autograd (dgrad / wgrad).
 *
 *   D[M,N] = alpha * (sum_k A[m,k] * B[n,k] + bias[n]) + beta * C[m,n]
 *
 *   A is logical [M,K]: a_mn_major == 0 -> stored row-major [M,K] (ld = lda);  1 -> stored [K,M] (ld = lda).
 *   B is logical [N,K]: b_mn_major == 0 -> stored row-major [N,K] (ld = ldb);  1 -> stored [K,N] (ld = ldb).
 *   D/C: row-major [M,N]; d_is_f32 selects fp32 (else bf16) for BOTH D and C.  C may be NULL (beta ignored)
 *   or alias D.  bias: bf16 [N] (4-byte aligned) or NULL.   M, N, K >= 1 of any value (an LM head of any vocabulary:
 *   N = V forward, K = V dgrad, M = V wgrad); the row strides keep 16 bytes (lda, ldb, ldd, ldc % 8 == 0 for bf16,
 *   ldd, ldc % 4 == 0 for fp32) and the bases are 16-byte aligned.  TMA zero-fills operand tails and clips D / C
 *   tails: columns of a row beyond N (or K) are never read as data.  TMA stores write whole 16-byte segments, so when
 *   N is not a multiple of 16 bytes the columns [N, round_up(N, 16 bytes)) of D receive zeros (ldd must cover them);
 *   nothing beyond that segment is written.
 *   flags: bit0 = the caller promises bf16 D and no C (checked).  With or without it, every launch stages its output
 *   tiles in shared memory and writes them with TMA stores (reduce-adds for split-K), so D and C need 16-byte aligned
 *   bases and row strides.
 * ------------------------------------------------------------------------------------------------ */
#define DOLO_GEMM_FLAG_TMA_STORE 1
/* bit1: D(fp32) += alpha*A.B^T with split-K + TMA fp32 reduce-adds (weight gradients); C must be NULL or alias D with
 * beta == 1, bias NULL.  Summation order over K splits is not deterministic (like FSDP's own reduce order). */
#define DOLO_GEMM_FLAG_SPLITK_ACCUMULATE 2
/* bit2 / bit3: force / forbid a CTA-pair kernel: accepted, no effect on sm_90 (no paired MMA). */
#define DOLO_GEMM_FLAG_CTA_PAIR 4
#define DOLO_GEMM_FLAG_NO_CTA_PAIR 8
/* bit4 / bit5: epilogue selection of other GPU generations: accepted, no effect on sm_90 (bf16 and fp32 D both take
 * the shared-memory + TMA-store epilogue). */
#define DOLO_GEMM_FLAG_DIRECT_EPILOGUE 16
#define DOLO_GEMM_FLAG_F32_TMA_EPILOGUE 32
int dolomite_b200_gemm_bf16(const void* A, int64_t lda, int a_mn_major, const void* B, int64_t ldb, int b_mn_major,
                            void* D, int64_t ldd, int d_is_f32, const void* C, int64_t ldc, float alpha, float beta,
                            const void* bias, int64_t M, int64_t N, int64_t K, int flags, void* stream);

/* Up to 4 weight gradients in ONE persistent launch (the four nn.Linear of a GPTDolomiteBlock, autograd of linear.py:5-25):
 *   dW_i[M_i, N_i] = alpha_i * dY_i^T X_i  (accumulate[i] == 0: overwrite)   or   dW_i += alpha_i * dY_i^T X_i  (!= 0)
 * dY_i bf16 [K, M_i] (ld_dy), X_i bf16 [K, N_i] (ld_x), dW_i fp32 [M_i, N_i] (ld_dw); K = token rows, common to all. */
int dolomite_b200_gemm_bf16_wgrad_multi(int n_problems, const void* const* dY, const int64_t* ld_dy, const void* const* X,
                                        const int64_t* ld_x, float* const* dW, const int64_t* ld_dw, const int64_t* M,
                                        const int64_t* N, int64_t K, const float* alpha, const int* accumulate,
                                        void* stream);

/* Output tile width (128 or 256 columns, 128 rows) that a dense launch of gemm_bf16 (without split-K) or
 * gemm_bf16_wgrad_multi over these problems takes on the current device, under the current gemm_tile_n and
 * gemm_sm_margin options.  Automatic choice: the wider tile unless its last, partly filled wave makes the launch slower,
 * i.e. 256 iff ceil(tiles_256 / SMs) * cost_256_over_128 < ceil(tiles_128 / SMs), tiles summed over the problems.
 * *cost_256_over_128 (may be NULL) receives the constant of that rule: the time of one 128x256 tile over one 128x128 tile. */
int dolomite_b200_gemm_bf16_tile_n(int n_problems, const int64_t* M, const int64_t* N, int* tile_n,
                                   float* cost_256_over_128);

/* ------------------------------------------------------------------------------------------------
 * FP8 linear layers with delayed scaling: what TransformerEngine's te.Linear computes inside
 * te.fp8_autocast(DelayedScaling(Format.HYBRID, amax_history_len=16, amax_compute_algo="max")) -- the nn.Linear swap of
 * distributed/fp8/nv_te.py:15-42 and the training forward context of pretrain.py:126-134 / finetune.py:90-98.
 * Formats: 0 = e4m3 (max 448; inputs and weights), 1 = e5m2 (max 57344; output gradients).  fp8 tensors are uint8 storage.
 *
 * gemm_fp8:  D[M,N] = alpha * (a_scale_inv * b_scale_inv * sum_k A[m,k] * B[n,k] + bias[n]) + beta * C[m,n]
 *   A fp8 row-major [M,K] (lda), B fp8 row-major [N,K] (ldb): both K-major (fp8 wgmma reads no other layout).
 *   a_scale_inv / b_scale_inv: DEVICE fp32 scalars (no host sync).  D/C/bias as in gemm_bf16.
 *   K % 16 == 0, N % 16 == 0, lda / ldb % 16 == 0, 16-byte aligned bases.
 *   split_accumulate != 0: the tensor-core accumulator is added into a separate fp32 sum once per 128-deep k-block (TE's
 *   split accumulator, dgrad / wgrad); 0 = one accumulator over the whole contraction (TE's fprop fast accumulation).
 * gemm_fp8_wgrad_multi: up to 4 weight gradients in one launch, dW_i (+)= alpha_i * dYt_i . Xt_i^T with dYt_i fp8
 *   [M_i, K] and Xt_i fp8 [N_i, K] (the transposed casts; K = token rows, K % 16 == 0), dW_i fp32.
 * ------------------------------------------------------------------------------------------------ */
int dolomite_b200_gemm_fp8(const void* A, int64_t lda, int a_fmt, const void* B, int64_t ldb, int b_fmt,
                           const float* a_scale_inv, const float* b_scale_inv, void* D, int64_t ldd, int d_is_f32,
                           const void* C, int64_t ldc, float alpha, float beta, const void* bias, int64_t M, int64_t N,
                           int64_t K, int split_accumulate, void* stream);
int dolomite_b200_gemm_fp8_wgrad_multi(int n_problems, const void* const* dYt, const int64_t* ld_dyt, const void* const* Xt,
                                       const int64_t* ld_xt, const float* const* dy_scale_inv,
                                       const float* const* x_scale_inv, float* const* dW, const int64_t* ld_dw,
                                       const int64_t* M, const int64_t* N, int64_t K, const float* alpha,
                                       const int* accumulate, int dy_fmt, int x_fmt, int split_accumulate, void* stream);
/* fp8_cast: x bf16 [rows, cols] (ldx) -> q = satfinite_rne(fp32(x) * scale[0]) as fp8 `fmt`:
 *   out   [rows, cols] contiguous (may be NULL), out_t [cols, rows] contiguous, the transpose (may be NULL; needs
 *   rows % 16 == 0); amax (may be NULL): *amax = max(*amax, max|x|) -- the amax-history row 0 entry of the tensor's slot.
 *   cols % 16 == 0, ldx % 8 == 0, 16-byte aligned pointers. */
int dolomite_b200_fp8_cast(const void* x, int64_t ldx, int64_t rows, int64_t cols, int fmt, const float* scale, void* out,
                           void* out_t, float* amax, void* stream);
/* fp8_scaling_update: DelayedScaling's amax / scale update for n_slots tensors of one format in one launch.
 *   amax_history fp32 [history_len, n_slots] (row 0 = current), scale / scale_inv fp32 [n_slots]:
 *   amax = max over the history (NaN propagates); scale = fp8_max / amax if amax is finite and > 0, else kept;
 *   scale_inv = 1 / scale; the history rolls by -1 along rows and row 0 is zeroed.  history_len <= 64. */
int dolomite_b200_fp8_scaling_update(float* amax_history, int history_len, int64_t n_slots, float* scale, float* scale_inv,
                                     float fp8_max, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Grouped GEMM for MoE experts (replaces scattermoe `parallel_linear`, moe_dolomite/moe/scatter.py:38-49, and the
 * per-expert F.linear loop of moe/base.py:12-50).  Token rows are grouped by expert, each segment padded to a
 * multiple of 256 rows (scattermoe `padded_block_indices`); m_tile_group[i] = expert of 128-row tile i (-1: unused).
 *   grouped_m:  D[rows, N] = alpha * A[rows, K] . W[g]^T      W stored [G, N, K] (b_mn_major = 0: expert forward)
 *                                                         or W stored [G, K, N] (b_mn_major = 1: expert dgrad)
 *   grouped_k:  D[g][M, N] = alpha * A_g^T B_g + beta * D[g]  (expert wgrad, fp32): A [K_max, M], B [K_max, N] row-major,
 *               contraction over the rows [group_k_offsets[g], group_k_offsets[g+1]) of expert g.  beta = 0 OVERWRITES: D need not
 *               be initialised, and the slice of an expert with an empty row range is written as zeros; beta != 0 leaves it alone.
 * Extents: N and K may take any value that keeps the row strides 16-byte aligned (lda, ldb, ldd multiples of 8 bf16 / 4
 * fp32 elements; an MN-major B, and the fused gather, need K % 8 == 0).  Every K and N tail is expert-local: TMA
 * zero-fills the last k-block of expert g from its own rows (a K-major B as one [G * N, K] map whose N tail only reaches
 * the clipped output columns >= N; an MN-major B as a rank-3 {N, K, G} map), so another expert's weights, finite or not,
 * never enter a product.  grouped_k stops every tile at row M and column N of its own group (D is a rank-3 {N, M, G}
 * map with group stride M * ldd), for the overwrite, the accumulate and the zero slices of experts without rows.
 * ------------------------------------------------------------------------------------------------ */
int dolomite_b200_gemm_bf16_grouped_m(const void* A, int64_t lda, const void* B, int64_t ldb, int b_mn_major, void* D,
                                      int64_t ldd, float alpha, int64_t M_max, int64_t N, int64_t K,
                                      const int32_t* m_tile_group, int num_groups, int flags, void* stream);
/* grouped_m with the gather fused into the operand load: A is the UNGROUPED [a_rows, K] activation matrix,
 * a_row_index[r] (int32, 16-byte aligned, M_max entries) the source row of grouped row r; W stored [G, N, K]. */
int dolomite_b200_gemm_bf16_grouped_m_gather(const void* A, int64_t lda, int64_t a_rows, const int32_t* a_row_index,
                                             const void* B, int64_t ldb, void* D, int64_t ldd, float alpha, int64_t M_max,
                                             int64_t N, int64_t K, const int32_t* m_tile_group, int num_groups, int flags,
                                             void* stream);
/* grouped_m with a per-expert bias (ParameterizedExperts with add_bias, moe/base.py:12-50):
 *   D[rows of g] = (A . W[g]^T + bias[g]) * alpha, fp32 epilogue, one rounding to bf16 (as the dense biased linear).
 * bias bf16 [G, N] with row stride ld_bias (even, >= N).  a_row_index NULL: A is grouped (as grouped_m); otherwise the
 * fused gather of grouped_m_gather (a_rows, a_row_index as there, b_mn_major must be 0). */
int dolomite_b200_gemm_bf16_grouped_m_bias(const void* A, int64_t lda, int64_t a_rows, const int32_t* a_row_index,
                                           const void* B, int64_t ldb, int b_mn_major, void* D, int64_t ldd,
                                           const void* bias, int64_t ld_bias, float alpha, int64_t M_max, int64_t N,
                                           int64_t K, const int32_t* m_tile_group, int num_groups, int flags,
                                           void* stream);
int dolomite_b200_gemm_bf16_grouped_k(const void* A, int64_t lda, const void* B, int64_t ldb, float* D, int64_t ldd,
                                      float alpha, float beta, int64_t M, int64_t N, int64_t K_max,
                                      const int32_t* group_k_offsets, int num_groups, void* stream);

/* ------------------------------------------------------------------------------------------------
 * MoE routing / dispatch (moe_dolomite/moe/base.py:108-181, moe/scatter.py:109-138); all on the device, no host sync.
 *   moe_max_rows: upper bound of padded grouped rows for T tokens (buffer sizing).
 *   moe_route: router logits bf16 [T,E] -> top-k expert ids int32 [T,k] (arg-max order), fp32 softmax weights [T,k],
 *              counts[E] (== bincount, bit exact), offsets_padded[E+1], m_tile_group[max_rows/128], cursors[E] scratch,
 *              row_of_slot[T*k] (grouped row of token-slot), slot_of_row[max_rows] (-1 = padding row),
 *              token_of_row[max_rows] (source token of a grouped row; padding rows name token 0) -- the row index of
 *              dolomite_b200_gemm_bf16_grouped_m_gather.  Segments are padded to 256 rows.
 *   moe_gather: X_g[row] = x[slot_of_row[row] / k] or 0.     moe_combine: out = c + alpha * sum_j w_j * Y_g[row_j].
 *   moe_combine_bwd / moe_token_sum / moe_router_bwd: their backward pieces.
 * Any E in [1, 256]: router logits and dlogits are contiguous [T, E] (row stride E); a caller whose GEMMs need 16-byte
 * rows (E % 8 != 0) stages them (kernels.router_logits / router_grad in the Python package).
 * ------------------------------------------------------------------------------------------------ */
int64_t dolomite_b200_moe_max_rows(int64_t T, int E, int k);
int dolomite_b200_moe_route(const void* router_logits, int64_t T, int E, int k, int32_t* sel_idx, float* sel_w,
                            int32_t* counts, int32_t* offsets_padded, int32_t* m_tile_group, int32_t* cursors,
                            int32_t* row_of_slot, int32_t* slot_of_row, int32_t* token_of_row, void* stream);
int dolomite_b200_moe_gather(const void* x, void* xg, const int32_t* slot_of_row, const int32_t* offsets_padded,
                             int64_t T, int E, int k, int H, void* stream);
int dolomite_b200_moe_combine(const void* yg, const int32_t* row_of_slot, const float* sel_w, const void* c, void* out,
                              int64_t T, int k, int H, float alpha, void* stream);
int dolomite_b200_moe_combine_bwd(const void* dy, const void* yg, const int32_t* slot_of_row,
                                  const int32_t* offsets_padded, const float* sel_w, void* dyg, float* dw, int64_t T,
                                  int E, int k, int H, float alpha, void* stream);
int dolomite_b200_moe_token_sum(const void* dxg, const int32_t* row_of_slot, void* dx, int64_t T, int k, int H,
                                void* stream);
int dolomite_b200_moe_router_bwd(const int32_t* sel_idx, const float* sel_w, const float* dw, void* dlogits, int64_t T,
                                 int E, int k, void* stream);

/* ------------------------------------------------------------------------------------------------
 * MoE load-balancing loss (moe_dolomite/base.py:24-43 -> transformers' Mixtral load_balancing_loss_func), accumulated
 * over the L MoE layers of one forward; rows t >= T_real (alignment rows) are not tokens.  With N = L * T_real:
 *   moe_aux_stats:    acc[0][e] += sum_t softmax(logits[t])_e (fp32 softmax over all E of the bf16 row),
 *                     acc[1][e] += #(t, slot) with sel_idx[t, slot] == e (exact below 2^24 per expert).  acc is [2, E]
 *                     fp32, partial is scratch of moe_aux_partial_floats(T_real, E) floats; fixed-order sums only.
 *   moe_aux_finalize: aux = E * sum_e acc[1][e] acc[0][e] / N^2, c[e] = E * acc[1][e] / N^2, and loss[0] += coef * aux
 *                     when loss != NULL (all on the device).
 *   moe_router_bwd_aux: moe_router_bwd plus, on rows t < T_real, s * p[t,e] * (c[e] - sum_j p[t,j] c[j]) with the scalar
 *                     s = *s (coef * dL/dloss + dL/daux) read on the device; dlogits rounded to bf16 once.
 * ------------------------------------------------------------------------------------------------ */
int64_t dolomite_b200_moe_aux_partial_floats(int64_t T_real, int E);
int dolomite_b200_moe_aux_stats(const void* router_logits, const int32_t* sel_idx, int64_t T, int64_t T_real, int E, int k,
                                float* partial, float* acc, void* stream);
int dolomite_b200_moe_aux_finalize(const float* acc, int E, int64_t n_tokens, float coef, float* aux, float* c,
                                   float* loss, void* stream);
int dolomite_b200_moe_router_bwd_aux(const void* router_logits, const int32_t* sel_idx, const float* sel_w,
                                     const float* dw, const float* c, const float* s, void* dlogits, int64_t T,
                                     int64_t T_real, int E, int k, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Packed var-len causal attention (replaces flash_attn_varlen_func at attention/padding_free.py:51-62).
 *   qkv: packed projection output [T, row_stride] in the slot layout described at rope_qk_inplace.
 *   out: [T, n_heads*head_dim] bf16; lse: fp32 [n_heads, T] (natural log-sum-exp of scale*s).
 *   cu_seqlens int32 [B+1] (same for q and k), causal within each document.
 *   head_dim: 16, 32, 64, 80, 96, 128, 160, 192 or 256 (the same for attn_decode); any other value returns an error.
 *   bwd: dqkv has the same layout as qkv (dq, dk, dv written into their slots; bf16).
 *   workspace sizes via the *_workspace_bytes helpers.
 * ------------------------------------------------------------------------------------------------ */
int dolomite_b200_attn_varlen_fwd(const void* qkv, int64_t row_stride, void* out, float* lse,
                                  const int32_t* cu_seqlens, int n_docs, int64_t T, int max_seqlen, int n_groups,
                                  int q_per_group, int head_dim, float softmax_scale, void* stream);
int64_t dolomite_b200_attn_varlen_bwd_workspace_bytes(int64_t T, int n_groups, int q_per_group, int head_dim);
int dolomite_b200_attn_varlen_bwd(const void* dout, const void* qkv, int64_t row_stride, const void* out,
                                  const float* lse, void* dqkv, const int32_t* cu_seqlens, int n_docs, int64_t T,
                                  int max_seqlen, int n_groups, int q_per_group, int head_dim, float softmax_scale,
                                  void* workspace, void* stream);
/* The same with attention-probability dropout (attention/base.py:252 `attn_dropout`; `dropout_p` of flash_attn_varlen_func,
 * attention/padding_free.py:49-59, training mode only): P_ij is kept with probability 1 - dropout_p and scaled by
 * 1 / (1 - dropout_p) after the softmax normaliser was taken over the undropped row.  The mask is a hash of (global query
 * token, global key token, head, key0, key1); backward must be given the keys of its forward.  dropout_p == 0: identical
 * to the functions above. */
int dolomite_b200_attn_varlen_fwd_dropout(const void* qkv, int64_t row_stride, void* out, float* lse,
                                          const int32_t* cu_seqlens, int n_docs, int64_t T, int max_seqlen, int n_groups,
                                          int q_per_group, int head_dim, float softmax_scale, float dropout_p,
                                          uint32_t key0, uint32_t key1, void* stream);
int dolomite_b200_attn_varlen_bwd_dropout(const void* dout, const void* qkv, int64_t row_stride, const void* out,
                                          const float* lse, void* dqkv, const int32_t* cu_seqlens, int n_docs, int64_t T,
                                          int max_seqlen, int n_groups, int q_per_group, int head_dim,
                                          float softmax_scale, float dropout_p, uint32_t key0, uint32_t key1,
                                          void* workspace, void* stream);
/* The same with ALiBi (position_embedding_type: alibi with eager or SDPA attention on padded batches; the reference's
 * call sites: gpt_dolomite/base.py:261-287 `_get_alibi_bias` -> modeling_utils/position_embedding/alibi.py:14-30, added to
 * the logits through the mask of `_get_maybe_causal_mask`, base.py:559-598, in attention/base.py:233-245 (eager
 * baddbmm) and attention/sdpa.py:56-64 (attn_mask of scaled_dot_product_attention)).  The logit of (query, key k) of
 * head h is softmax_scale * <q, k> + bf16(alibi_slopes[h] * kpos(k)), kpos = the key's index inside its document; the
 * softmax scale does not multiply the bias.  The logits stay fp32 (as in SDPA's fused kernels; eager rounds them to
 * bf16).  lse is the natural log-sum-exp of the biased logits; the backward must be given the slopes of its forward.
 *   alibi_slopes  fp32 [n_heads], the reference's slopes (alibi.py:32-44); null is an error.
 * dropout_p / key0 / key1 as in the *_dropout functions (dropout_p == 0: none). */
int dolomite_b200_attn_varlen_fwd_alibi(const void* qkv, int64_t row_stride, void* out, float* lse,
                                        const int32_t* cu_seqlens, int n_docs, int64_t T, int max_seqlen, int n_groups,
                                        int q_per_group, int head_dim, float softmax_scale, float dropout_p, uint32_t key0,
                                        uint32_t key1, const float* alibi_slopes, void* stream);
int dolomite_b200_attn_varlen_bwd_alibi(const void* dout, const void* qkv, int64_t row_stride, const void* out,
                                        const float* lse, void* dqkv, const int32_t* cu_seqlens, int n_docs, int64_t T,
                                        int max_seqlen, int n_groups, int q_per_group, int head_dim, float softmax_scale,
                                        float dropout_p, uint32_t key0, uint32_t key1, const float* alibi_slopes,
                                        void* workspace, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DOLOMITE_B200_H */
