/*
 * b200nlp.h — C-ABI of libb200nlp.so: hand-written sm_90a (H100) kernels for the PaddleNLP LLM decoder hot path.
 *
 * This is the drop-in boundary (SURVEY.md §8b).  Each entry point replaces one native op the reference reaches
 * through Paddle's custom-op C++ API (PD_BUILD_OP) or through a Paddle-core kernel; the reference call site is
 * cited beside each declaration (paths relative to the PaddleNLP tree).
 *
 * Conventions
 *   - plain C, no framework types: device pointers + int64 sizes + scalar attributes + cudaStream_t.
 *   - the CALLER owns every buffer (inputs, outputs, workspaces); kernels never allocate or free device memory.
 *   - all work is enqueued on `stream`; no host synchronisation inside any entry point.
 *   - return value: 0 = ok, <0 = argument error, >0 = cudaError_t of the failed launch;
 *     b200_last_error() returns a thread-local message for the last non-zero return.
 *   - bf16 tensors are `__nv_bfloat16` bit patterns (uint16), row-major, contiguous unless a leading dimension
 *     is passed.  "T" below is the token count (batch * seq).
 */
#ifndef B200NLP_H_
#define B200NLP_H_

#include <stdbool.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200NLP_ABI_VERSION 2

#ifndef __CUDA_RUNTIME_API_H__
typedef struct CUstream_st* cudaStream_t;
#endif

/* ---- plumbing ------------------------------------------------------------------------------------------ */
const char* b200_last_error(void);
int b200_abi_version(void);
/* 0 if the current device is compute capability 9.0 (H100); error otherwise. */
int b200_device_check(void);
/* Programmatic dependent launch for the GEMM kernels (returns the previous setting; NOT an error code): when enabled, a GEMM
 * may become resident while the previous kernel of the stream is still draining; it waits (griddepcontrol.wait) before
 * touching operands or outputs.  Used for the decode-step chain. */
int b200_set_pdl(int enable);
/* Kernel of b200_fa_fwd / b200_fa_fwd_flashmask (returns the previous setting; NOT an error code): 2 (default) = the wgmma
 * kernel (128-row q tiles, TMA-fed 128-row K/V tiles), 1 = the mma.sync kernel (128-row q tiles, 8 warps), kept as the
 * cross-check and as the paged prefill of b200_append_attention.  Same rounding points. */
int b200_set_fa_fwd_impl(int impl);
/* Kernel of b200_fa_bwd / b200_fa_bwd_flashmask (returns the previous setting): 2 (default) = the warp-specialised wgmma
 * kernel (128-row kv tiles, TMA-fed 64-row q tiles, TMA reduce-adds), 1 = the mma.sync kernel (64-row kv and q tiles), kept as
 * the cross-check.  Same rounding points. */
int b200_set_fa_bwd_impl(int impl);

/* ---- GEMM: replaces paddle.matmul / nn.Linear (cuBLASLt) --------------------------------------------------
 * C[M,N] (+)= op(A)[M,K] * op(B)[K,N] (+ bias[N]);  bf16 operands, fp32 accumulation in registers (wgmma), ONE rounding to bf16.
 *   a_mn_major = 0 : A is stored [M,K] row-major (lda = row stride in elements)          — activations
 *   a_mn_major = 1 : A is stored [K,M] row-major (i.e. the caller passes A^T)            — dW = X^T * dY
 *   b_mn_major = 1 : B is stored [K,N] row-major — Paddle's nn.Linear weight layout [in,out]
 *   b_mn_major = 0 : B is stored [N,K] row-major (i.e. B^T)                               — dX = dY * W^T
 *   accumulate != 0: C_new = bf16(fp32(C_old) + acc)   (gradient accumulation, cf. llm/utils/fused_layers.py:36-74)
 *   bias            : optional fp32 [N], added in fp32 before the rounding (Qwen2 q/k/v bias, qwen2/modeling.py:478-480)
 * Reference call sites: llama/modeling.py:933-935,1103 (q/k/v/o), :632-652 (gate/up/down), :1894-1921 (lm_head).
 * Requires lda, ldb, ldc multiples of 8 elements and 16-byte aligned base pointers: A, B, C and residual here, X, W, GU and
 * Mout of b200_gemm_swiglu_bf16, dY, Wdown, GU and DGU of b200_gemm_swiglu_bwd_bf16, A, B and a non-NULL C of
 * b200_gemm_bf16_splitk; any other is an argument error (M, N, K themselves are free: TMA zero-fills / clips partial tiles).
 */
int b200_gemm_bf16(const void* A, const void* B, void* C, const float* bias, int64_t M, int64_t N, int64_t K,
                   int64_t lda, int64_t ldb, int64_t ldc, int a_mn_major, int b_mn_major, int accumulate,
                   cudaStream_t stream);
/* Same with a fused residual epilogue and a limit on the persistent grid.
 *   residual (bf16 [M,N], leading dimension ldr; exclusive with accumulate):
 *       C = bf16( bf16(acc + bias) + residual )  — the Linear-output rounding followed by the decoder layer's residual
 *       add (llama/modeling.py:1212, 1218), i.e. the reference's two rounding points in one kernel.
 *   max_ctas > 0 limits the persistent grid (used to leave SMs to a concurrent kernel). */
int b200_gemm_bf16_ex(const void* A, const void* B, void* C, const float* bias, const void* residual, int64_t M,
                      int64_t N, int64_t K, int64_t lda, int64_t ldb, int64_t ldc, int64_t ldr, int a_mn_major,
                      int b_mn_major, int accumulate, int max_ctas, cudaStream_t stream);
/* Same operands, fp32 output C [M, ldc] (fp32 master gradients, amp_master_grad; cf. fused_linear_param_grad_add(...,
 * multi_precision=True), llm/utils/fused_layers.py:44-50):
 *   accumulate == 0: C = acc ;  accumulate != 0: C += acc, one fp32 add per element (TMA reduce-add in L2; a subnormal sum
 *   is flushed to zero).  No rounding to bf16 anywhere.
 * Requires lda, ldb multiples of 8, ldc a multiple of 4 and >= N, A, B and C 16-byte aligned; any other is an argument error. */
int b200_gemm_bf16_f32(const void* A, const void* B, float* C, int64_t M, int64_t N, int64_t K, int64_t lda, int64_t ldb,
                       int64_t ldc, int a_mn_major, int b_mn_major, int accumulate, cudaStream_t stream);

/* Weight-streaming GEMM for the decode step (M <= ~128 tokens): same math as b200_gemm_bf16 (C = op(A) op(B) + bias, one
 * rounding), but K is split over CTAs (split_k, 0 = auto) so that every SM streams part of the weight matrix; fp32 partial
 * tiles are summed in L2 by TMA reduce-add into `workspace` (b200_gemm_splitk_workspace_bytes; must be ZERO on entry,
 * is returned zeroed) and rounded once.  C == NULL skips the rounding pass: the consumer (b200_add_rmsnorm_f32,
 * b200_decode_rope_append_f32) reads the fp32 sums, rounds them once to bf16 and re-zeroes the workspace.
 * Replaces the cuBLASLt calls of FusedMultiTransformer's decode step (fused_transformer_layers.py:817-820, 895-896, 967-974). */
int64_t b200_gemm_splitk_workspace_bytes(int64_t M, int64_t N);
int b200_gemm_bf16_splitk(const void* A, const void* B, void* C, const float* bias, void* workspace, int64_t M, int64_t N,
                          int64_t K, int64_t lda, int64_t ldb, int64_t ldc, int a_mn_major, int b_mn_major, int split_k,
                          cudaStream_t stream);

/* ---- weight-only int8 linear layers (--quant_type weight_only_int8, llm/predict/predictor.py:86,1250): weight_quantize /
 * weight_only_linear of FusedMultiTransformerWeightOnly (fused_transformer_layers.py:1221-1440) --------------------------
 * Quantisation of a bf16 W [K, N] (Paddle's [in, out] layout, row stride ldw), one scale per output channel:
 *   a[n] = max_k |W[k, n]| (fp32, exact), scale[n] = bf16_rn(a[n] / 127.0f) (bf16 [N]),
 *   q[k, n] = clamp(rint(W[k, n] / float(scale[n])), -127, 127) (IEEE fp32 division, half to even); scale 0 gives q = 0.
 * Packed layout of q (exactly N * K bytes; this library's own, not Paddle's CUTLASS interleave): 128-byte units, one per
 * 8 output channels x 16 k, unit (g, s) at byte (g * K/16 + s) * 128 for channels 8g .. 8g+7 and k 16s .. 16s+15.  Inside a
 * unit, lane l (0..31) owns bytes 4l .. 4l+3 = q[16s + c][n], q[16s + c + 1][n], q[16s + c + 8][n], q[16s + c + 9][n] with
 * n = 8g + l/4, c = 2 (l % 4): the two bf16 pairs of the tensor-core A fragment of row l/4, so a thread reads each half of its
 * fragment with one 32-bit shared-memory load and converts it in registers.
 * Requires K % 16 == 0, N % 8 == 0, ldw >= N, Q 4-byte aligned.  Runs on the device (load time, not a hot path). */
int b200_weight_quantize_int8(const void* W, void* Q, void* scale, int64_t K, int64_t N, int64_t ldw, cudaStream_t stream);
/* y[m, n] = scale[n] * sum_k X[m, k] q[k, n] (+ bias[n]): X bf16 [M, K] (row stride ldx), Q / scale from
 * b200_weight_quantize_int8, fp32 sums (int8 -> bf16 is exact, the weights are never rounded), the scale multiplies the fp32
 * sum (or each split-K partial before it is reduced), ONE rounding to bf16 into C [M, ldc].  One kernel for every M: the
 * weights are the wgmma A operand (converted in registers), the tokens its N dimension (8 to 128 wide).
 *   split_k: 0 chooses (K is split across CTAs only when the output tiles leave SMs idle), 1 = no split, > 1 explicit.  A
 *   split needs `workspace` (b200_gemm_splitk_workspace_bytes(M, N), ZERO on entry, returned zeroed, as for
 *   b200_gemm_bf16_splitk); workspace == NULL means no split (split_k > 1 is then an argument error).
 *   bias: optional fp32 [N] (Qwen2 q/k/v bias).
 * Requires M, N, K > 0, K % 16 == 0, N % 8 == 0, ldx and ldc multiples of 8, X, Q, C and workspace 16-byte aligned; any other
 * is an argument error. */
int b200_weight_only_gemm_bf16(const void* X, const void* Q, const void* scale, const float* bias, void* C, void* workspace,
                               int64_t M, int64_t N, int64_t K, int64_t ldx, int64_t ldc, int split_k, cudaStream_t stream);
/* Same product left as fp32 sums: workspace [M, N] (contiguous, ZERO on entry) += scale[n] * sum_k X[m, k] q[k, n], by TMA
 * reduce-add of each (split-K) partial.  The consumer (b200_add_rmsnorm_f32, b200_decode_rope_append_f32, b200_swiglu_fwd_f32)
 * rounds once and re-zeroes it, as after b200_gemm_bf16_splitk with C == NULL. */
int b200_weight_only_gemm_f32(const void* X, const void* Q, const void* scale, float* workspace, int64_t M, int64_t N, int64_t K,
                              int64_t ldx, int split_k, cudaStream_t stream);

/* gate|up projection + SwiGLU in ONE kernel — LlamaMLP.forward with fuse_attention_ffn (llama/modeling.py:632-652, swiglu :38-45):
 *   GU[M, 2I] = bf16(X[M,K] * W[K,2I])  (gate columns [0,I), up columns [I,2I); kept for the backward),
 *   Mout[M, I] = bf16(silu(gate) * up)  with gate/up rounded to bf16 first (the unfused rounding points).
 * A 256-column wgmma tile is formed from 128 gate columns and the 128 up columns of the same channels, so no interleaved
 * weight layout is needed; requires I % 64 == 0 (a last tile of 64 channels leaves half of it unused).  GU == NULL: gate|up are
 * not stored (the decode step's ffn1 + fused_bias_act("swiglu"), fused_transformer_layers.py:100-168).  Bit-identical to
 * b200_gemm_bf16 followed by b200_swiglu_fwd. */
int b200_gemm_swiglu_bf16(const void* X, const void* W, void* GU, void* Mout, int64_t M, int64_t inter, int64_t K, int64_t ldx,
                          int64_t ldw, int64_t ldgu, int64_t ldm, cudaStream_t stream);
/* Backward twin: the down-projection dX GEMM with the SwiGLU backward in its epilogue.
 *   d(m) = dY[M,K] * Wdown[I,K]^T (never written);  DGU[M, 2I] = [ d(m) * up * silu'(gate) | d(m) * silu(gate) ],
 * GU = the saved gate|up projection [M, 2I].  Bit-identical to b200_gemm_bf16 (b_mn_major = 0) + b200_swiglu_bwd.  I % 64 == 0. */
int b200_gemm_swiglu_bwd_bf16(const void* dY, const void* Wdown, const void* GU, void* DGU, int64_t M, int64_t inter, int64_t K,
                              int64_t lddy, int64_t ldw, int64_t ldgu, int64_t lddgu, cudaStream_t stream);

/* ---- RMSNorm: replaces fused_ln.fused_rms_norm / fast_ln (apex-derived custom ops) --------------------------
 * fwd : y = bf16( bf16(x * rstd) * w ), rstd[row] = rsqrt(mean(x^2) + eps) in fp32 (saved for the backward).
 * bwd : dx = rstd * (dy*w - xhat * mean(dy*w*xhat)) (+ dres, the gradient arriving through the residual branch);
 *       dw (+)= sum_rows dy * bf16(xhat).   workspace: b200_rmsnorm_bwd_workspace_bytes(rows, h) bytes.
 * Reference: llama/modeling.py:352-386; fusion_ops.py:119-144; legacy/model_zoo/gpt-3/external_ops/fused_ln/
 * layer_norm_cuda.cu:47-66 (fwd), :164-183 (bwd); layer_norm_cuda.h:447-531, 1190-1260.
 */
int b200_rmsnorm_fwd(const void* x, const void* w, void* y, float* rstd, int64_t rows, int64_t h, float eps,
                     cudaStream_t stream);
int64_t b200_rmsnorm_bwd_workspace_bytes(int64_t rows, int64_t h);
int b200_rmsnorm_bwd(const void* dy, const void* x, const void* w, const float* rstd, const void* dres, void* dx,
                     void* dw, int accumulate_dw, void* workspace, int64_t rows, int64_t h, cudaStream_t stream);
/* Same, dw an fp32 gradient (16-byte aligned): dw (+)= the fp32 column sums, never rounded to bf16. */
int b200_rmsnorm_bwd_f32(const void* dy, const void* x, const void* w, const float* rstd, const void* dres, void* dx,
                         float* dw, int accumulate_dw, void* workspace, int64_t rows, int64_t h, cudaStream_t stream);

/* Column sums of a bf16 [rows, n] matrix (leading dimension ld) into a bf16 vector: bias gradients of Qwen2 q/k/v
 * (qwen2/modeling.py:478-480).  workspace: b200_colsum_workspace_bytes(rows, n). */
int64_t b200_colsum_workspace_bytes(int64_t rows, int64_t n);
int b200_colsum_bf16(const void* a, void* out, int accumulate, void* workspace, int64_t rows, int64_t n, int64_t ld,
                     cudaStream_t stream);
/* Same into an fp32 vector (16-byte aligned). */
int b200_colsum_f32(const void* a, float* out, int accumulate, void* workspace, int64_t rows, int64_t n, int64_t ld,
                    cudaStream_t stream);

/* ---- RoPE (rotate-half), in place on `num_heads` consecutive heads starting at x: replaces Paddle-core
 * fused_rotary_position_embedding(use_neox_rotary_style=False) (fusion_ops.py:57-116; llama/modeling.py:557-577).
 * cos/sin tables: fp32 [max_pos, head_dim/2]; position of token t = position_ids[t] or t %% seq_len.
 * backward != 0 applies the transposed rotation (sin -> -sin). */
int b200_rope_inplace(void* x, const float* cos_table, const float* sin_table, const int32_t* position_ids,
                      int64_t tokens, int64_t seq_len, int64_t ld, int64_t num_heads, int64_t head_dim, int backward,
                      cudaStream_t stream);

/* ---- SwiGLU on a packed [rows, 2*inter] = [gate | up] buffer: replaces Paddle-core swiglu
 * (llama/modeling.py:38-45, 648-650).  bwd writes [dgate | dup] packed the same way. */
int b200_swiglu_fwd(const void* gate_up, void* out, int64_t rows, int64_t inter, cudaStream_t stream);
/* Same, gate|up given as the fp32 split-K workspace [rows, 2*inter] of the producing GEMM (rounded to bf16 here, workspace
 * re-zeroed): the decode step's ffn1 -> fused_bias_act("swiglu") pair (fused_transformer_layers.py:100-168). */
int b200_swiglu_fwd_f32(float* gate_up_f32_ws, void* out, int64_t rows, int64_t inter, cudaStream_t stream);
int b200_swiglu_bwd(const void* gate_up, const void* dout, void* dgate_up, int64_t rows, int64_t inter,
                    cudaStream_t stream);
/* ---- Embedding gather / scatter-add (nn.Embedding, llama/modeling.py:1465-1468, 1634). ids are int64. */
int b200_embedding_fwd(const int64_t* ids, const void* table, void* out, int64_t tokens, int64_t h, int64_t vocab,
                       cudaStream_t stream);
int b200_embedding_bwd(const int64_t* ids, const void* dout, void* dtable, int64_t tokens, int64_t h, int64_t vocab,
                       cudaStream_t stream);
/* Same scatter-add into an fp32 table (16-byte aligned; dout 8-byte aligned): fp32 vector atomics, 4 columns each. */
int b200_embedding_bwd_f32(const int64_t* ids, const void* dout, float* dtable, int64_t tokens, int64_t h, int64_t vocab,
                           cudaStream_t stream);

/* ---- Flash attention, causal, GQA, head_dim 64 or 128 (anything else: argument error): replaces F.scaled_dot_product_attention(is_causal=True)
 * (fusion_ops.py:147-267; Paddle-vendored FlashAttention-2) and its gradient (csrc/gpu/flash_attn_bwd.cc:22-92).
 * q [B,S,nh,d], k/v [B,S,kvh,d], o [B,S,nh,d]; ld* = token stride in elements (the tensors may be views into a
 * packed QKV projection).  lse [B,nh,S] fp32 (natural log).  Backward workspace: b200_fa_bwd_workspace_bytes(). */
int b200_fa_fwd(const void* q, const void* k, const void* v, void* o, float* lse, int64_t B, int64_t S,
                int64_t num_heads, int64_t num_kv_heads, int64_t head_dim, int64_t ldq, int64_t ldk, int64_t ldv,
                int64_t ldo, float softmax_scale, cudaStream_t stream);
int64_t b200_fa_bwd_workspace_bytes(int64_t B, int64_t S, int64_t num_heads, int64_t head_dim);
int b200_fa_bwd(const void* q, const void* k, const void* v, const void* o, const void* dout, const float* lse,
                void* dq, void* dk, void* dv, void* workspace, int64_t B, int64_t S, int64_t num_heads,
                int64_t num_kv_heads, int64_t head_dim, int64_t ldq, int64_t ldk, int64_t ldv, int64_t ldo,
                int64_t lddo, int64_t lddq, int64_t lddk, int64_t lddv, float softmax_scale, cudaStream_t stream);
/* FlashMask, causal lower-triangular form: the same two ops with a per-key-column start row
 * (fusion_ops.py:218-231 -> F.flashmask_attention(q, k, v, startend_row_indices=..., causal=True)):
 * mask_start_rows [B, S] int32, query row i sees key column c iff c <= i < mask_start_rows[b, c].  For packed SFT samples
 * ("zero padding", llm/utils/data.py:200-204, paddlenlp/datasets/zero_padding_dataset.py:84-86) it is the end of c's document
 * and must be non-decreasing in c; kv tiles that a q tile cannot see are skipped, not just masked.  NULL = plain causal. */
int b200_fa_fwd_flashmask(const void* q, const void* k, const void* v, void* o, float* lse, const int32_t* mask_start_rows,
                          int64_t B, int64_t S, int64_t num_heads, int64_t num_kv_heads, int64_t head_dim, int64_t ldq,
                          int64_t ldk, int64_t ldv, int64_t ldo, float softmax_scale, cudaStream_t stream);
int b200_fa_bwd_flashmask(const void* q, const void* k, const void* v, const void* o, const void* dout, const float* lse,
                          const int32_t* mask_start_rows, void* dq, void* dk, void* dv, void* workspace, int64_t B, int64_t S,
                          int64_t num_heads, int64_t num_kv_heads, int64_t head_dim, int64_t ldq, int64_t ldk, int64_t ldv,
                          int64_t ldo, int64_t lddo, int64_t lddq, int64_t lddk, int64_t lddv, float softmax_scale,
                          cudaStream_t stream);

/* ---- Criterion: LlamaPretrainingCriterion (llama/modeling.py:1799-1825) on bf16 logits [tokens, vocab] (ld).
 * fwd : loss_tok[i] = fp32 CE (0 for ignore_index), lse[i]; loss_out[0] = sum(l_i [l_i>0]) / count, loss_out[1] = count.
 * bwd : logits are overwritten by dlogits = (softmax - onehot) * [l_i>0] * grad_scale / count (bf16);
 *       grad_scale_dev (optional device scalar) multiplies grad_scale, so an upstream gradient that lives on the
 *       device (loss / gradient_accumulation_steps, trainer.py:2237-2238) needs no host synchronisation. */
int b200_ce_fwd(const void* logits, const int64_t* labels, float* loss_tok, float* lse, float* loss_out, int64_t tokens,
                int64_t vocab, int64_t ld, int64_t ignore_index, cudaStream_t stream);
int b200_ce_bwd(void* logits_inout, const int64_t* labels, const float* loss_tok, const float* lse,
                const float* loss_out, float grad_scale, const float* grad_scale_dev, int64_t tokens, int64_t vocab,
                int64_t ld, cudaStream_t stream);
/* Evaluation row pass over rows [row0, row0 + rows): `logits` points at row row0 (row stride ld); labels, loss_tok and pred
 * are indexed by absolute row.  One read of each row gives loss_tok (bit-identical to b200_ce_fwd's) and, when pred is not
 * null, pred (bit-identical to b200_argmax_bf16's).  No lse, no reduction: b200_ce_reduce then gives b200_ce_fwd's
 * loss_out over all rows, so the logits can be produced and consumed a chunk of rows at a time. */
int b200_ce_rows_fwd(const void* logits, const int64_t* labels, float* loss_tok, int64_t* pred, int64_t row0, int64_t rows,
                     int64_t vocab, int64_t ld, int64_t ignore_index, cudaStream_t stream);
int b200_ce_reduce(const float* loss_tok, float* loss_out, int64_t tokens, cudaStream_t stream);
/* Greedy token choice: first maximal index of each bf16 row (generation_utils.py:291-363 with top_p = 0). */
int b200_argmax_bf16(const void* logits, int64_t* out, int64_t rows, int64_t vocab, int64_t ld, cudaStream_t stream);

/* ---- Optimizer on the flat parameter buffer: ClipGradByGlobalNorm + AdamW(multi_precision)
 * (trainer.py:1717-1750; SURVEY.md A.4).  Elements [0, decay_end) receive weight decay.
 * grad_sqnorm: out[0] = || scale * g ||^2 ; adamw: g_eff = g * grad_scale * max_norm / max(||.||, max_norm). */
int64_t b200_grad_sqnorm_workspace_bytes(void);
int b200_grad_sqnorm(const void* grads, float* out, void* workspace, int64_t n, float scale, cudaStream_t stream);
int b200_adamw_step(void* params_bf16, const void* grads_bf16, float* master, float* exp_avg, float* exp_avg_sq,
                    const float* grad_sqnorm, int64_t n, int64_t decay_end, float lr, float beta1, float beta2, float eps,
                    float weight_decay, int64_t step, float grad_scale, float max_grad_norm, cudaStream_t stream);
/* The same two ops on an fp32 gradient buffer (fp32 master gradients; 16-byte aligned).  The arithmetic is the bf16 forms':
 * those convert each gradient to fp32 first, so a buffer of bf16-representable values gives the same bits. */
int b200_grad_sqnorm_f32(const float* grads, float* out, void* workspace, int64_t n, float scale, cudaStream_t stream);
int b200_adamw_step_f32(void* params_bf16, const float* grads, float* master, float* exp_avg, float* exp_avg_sq,
                        const float* grad_sqnorm, int64_t n, int64_t decay_end, float lr, float beta1, float beta2, float eps,
                        float weight_decay, int64_t step, float grad_scale, float max_grad_norm, cudaStream_t stream);
int b200_bf16_to_f32(const void* src, float* dst, int64_t n, cudaStream_t stream);

/* ======================================================================================================================
 * Generation path (FusedMultiTransformer / paddlenlp_ops, bf16 non-quantised subset; SURVEY.md §8 rows a16-a21)
 * ====================================================================================================================== */

/* Fused residual add + RMSNorm: r = bf16(x + residual) (residual may be NULL), normed = RMSNorm(r) * w.
 * normed or residual_out may be NULL (last layer: residual add only).  Replaces Paddle-core
 * fused_rms_norm(x, w, ..., residual=) -> (out, residual_out) as called by
 * experimental/transformers/fused_transformer_layers.py:799-805, 937-949, 976-999. */
int b200_add_rmsnorm(const void* x, const void* residual, const void* w, void* normed, void* residual_out, int64_t rows,
                     int64_t h, float eps, cudaStream_t stream);
/* Same, x given as the fp32 split-K workspace [rows, h] of the producing GEMM (rounded to bf16 here, workspace re-zeroed). */
int b200_add_rmsnorm_f32(float* x_f32_ws, const void* residual, const void* w, void* normed, void* residual_out,
                         int64_t rows, int64_t h, float eps, cudaStream_t stream);

/* KV cache tensor: bf16 [2, B, kvh, max_len, d] (K then V), the shape the reference predictor allocates
 * (llm/predict/predictor.py:697-706; experimental/transformers/llama/modeling.py:1768-1794).
 * Prefill: copy rotated K and V rows of the packed [B*S, ld] QKV projection for positions s < seq_lens[b]
 * (seq_lens may be NULL = all S).  Replaces write_cache_kv (csrc/gpu/write_cache_kv.cu:23-99). */
int b200_write_cache_kv(const void* qkv, void* cache, const int32_t* seq_lens, int64_t B, int64_t S, int64_t num_heads,
                        int64_t num_kv_heads, int64_t head_dim, int64_t max_len, int64_t ld, cudaStream_t stream);
/* Decode: rotate-half RoPE of the new token's q,k at position seq_lens[b] (in place in qkv [B, ld]) and append k,v to
 * the cache.  Replaces the RoPE + cache-write half of masked_multihead_attention
 * (fused_transformer_layers.py:884-893) / append_attn/decoder_write_cache_with_rope_kernel.cu:47-390. */
int b200_decode_rope_append(void* qkv, void* cache, const float* cos_table, const float* sin_table, const int32_t* seq_lens,
                            int64_t B, int64_t num_heads, int64_t num_kv_heads, int64_t head_dim, int64_t max_len,
                            int64_t ld, cudaStream_t stream);
/* Same, the QKV projection given as the fp32 split-K workspace [B, (nh+2kvh)*d] (+ optional fp32 bias): rounded to bf16
 * into qkv first, workspace re-zeroed. */
int b200_decode_rope_append_f32(void* qkv, float* acc_f32_ws, const float* bias, void* cache, const float* cos_table,
                                const float* sin_table, const int32_t* seq_lens, int64_t B, int64_t num_heads,
                                int64_t num_kv_heads, int64_t head_dim, int64_t max_len, int64_t ld, cudaStream_t stream);
/* Decode attention of one query token per sequence over cache positions [0, seq_lens[b]] (GQA, head_dim 64 or 128);
 * out [B, nh*d].  num_splits > 1 splits each sequence's cache range over that many CTAs (split-KV, merged by a second
 * kernel through `workspace`), as the reference's append_attention does (append_attention_c16_impl.cuh:826-1000).
 * Replaces the attention half of masked_multihead_attention / append_attention decode
 * (csrc/gpu/append_attn/append_attention_c16_impl.cuh:377-744). */
int64_t b200_decode_attention_workspace_bytes(int64_t B, int64_t num_heads, int64_t num_splits);
int b200_decode_attention(const void* qkv, const void* cache, const int32_t* seq_lens, void* out, void* workspace, int64_t B,
                          int64_t num_heads, int64_t num_kv_heads, int64_t head_dim, int64_t max_len, int64_t ld,
                          float softmax_scale, int64_t num_splits, cudaStream_t stream);
/* Same contract, Hopper streaming kernel: a producer warp moves 8 KB K/V chunks (32 rows at d = 128, 64 at d = 64) with
 * cp.async.bulk into a 4-stage shared-memory ring on mbarriers, four consumer warps compute (d / 8 lanes per cache row, the G
 * heads of a group sharing each row); GQA group size 1 to 8.  Split-KV partial rows are 132 floats at either head_dim.
 * Cache rows past the sequence length must hold finite values (zero-filled allocation, as the reference's paddle.zeros). */
int b200_decode_attention_tc(const void* qkv, const void* cache, const int32_t* seq_lens, void* out, void* workspace, int64_t B,
                             int64_t num_heads, int64_t num_kv_heads, int64_t head_dim, int64_t max_len, int64_t ld,
                             float softmax_scale, int64_t num_splits, cudaStream_t stream);

/* Paged ("block") KV cache of FusedBlockMultiTransformer / append_attention (fused_transformer_layers.py:2192-2354,
 * csrc/gpu/append_attention.cu:428-851): key_cache / value_cache [num_blocks, kvh, block_size, head_dim] bf16,
 * block_tables [B, max_blocks_per_seq] int32 (logical block -> physical block).  Same math as the dense entry points above:
 * prefill cache fill, decode RoPE + append (acc_f32_ws / bias optional as in b200_decode_rope_append_f32), decode attention
 * (the streaming kernel reads each cache row through the block table).  Every paged entry point, b200_append_attention
 * included, requires block_size 32, 64 or 128 and max_blocks_per_seq > 0 and returns an argument error otherwise, so a cache
 * that one of them fills can be read by all of them. */
int b200_write_cache_kv_paged(const void* qkv, void* key_cache, void* value_cache, const int32_t* block_tables,
                              const int32_t* seq_lens, int64_t B, int64_t S, int64_t num_heads, int64_t num_kv_heads,
                              int64_t head_dim, int64_t block_size, int64_t max_blocks_per_seq, int64_t ld, cudaStream_t stream);
int b200_decode_rope_append_paged(void* qkv, float* acc_f32_ws, const float* bias, void* key_cache, void* value_cache,
                                  const int32_t* block_tables, const float* cos_table, const float* sin_table,
                                  const int32_t* seq_lens, int64_t B, int64_t num_heads, int64_t num_kv_heads, int64_t head_dim,
                                  int64_t block_size, int64_t max_blocks_per_seq, int64_t ld, cudaStream_t stream);
int b200_decode_attention_paged(const void* qkv, const void* key_cache, const void* value_cache, const int32_t* block_tables,
                                const int32_t* seq_lens, void* out, void* workspace, int64_t B, int64_t num_heads,
                                int64_t num_kv_heads, int64_t head_dim, int64_t num_blocks, int64_t block_size,
                                int64_t max_blocks_per_seq, int64_t ld, float softmax_scale, int64_t num_splits,
                                cudaStream_t stream);

/* Bookkeeping ops, same semantics as the reference custom ops (file:line beside each). bool = 1-byte flags. */
/* get_padding_offset_v2 (+ remove padding): csrc/gpu/get_padding_offset_v2.cu:17-80 */
int b200_get_padding_offset(const int64_t* input_ids, const int32_t* cum_offsets, const int32_t* seq_lens,
                            int64_t* x_remove_padding, int32_t* padding_offset, int32_t* cum_offsets_out,
                            int32_t* cu_seqlens_q, int32_t* cu_seqlens_k, int64_t bsz, int64_t max_seq_len,
                            cudaStream_t stream);
/* rebuild_padding_v2: csrc/gpu/rebuild_padding_v2.cu:18-69 (one row per sequence = its last valid token) */
int b200_rebuild_padding(const void* tmp_out, const int32_t* cum_offsets, const int32_t* seq_lens_decoder,
                         const int32_t* seq_lens_encoder, void* out, int64_t bsz, int64_t max_len, int64_t dim,
                         cudaStream_t stream);
/* set_value_by_flags_and_idx: csrc/gpu/set_value_by_flags.cu:17-35 ; _v2: csrc/gpu/set_value_by_flags_v2.cu */
int b200_set_value_by_flags_and_idx(const bool* stop_flags, int64_t* pre_ids_all, const int64_t* pre_ids_now,
                                    const int64_t* step_idx, int64_t bs, int64_t length, cudaStream_t stream);
int b200_set_value_by_flags_and_idx_v2(const bool* stop_flags, int64_t* pre_ids_all, const int64_t* input_ids,
                                       const int32_t* seq_lens_encoder, const int32_t* seq_lens_decoder,
                                       const int64_t* step_idx, int64_t bs, int64_t length, int64_t length_input_ids,
                                       cudaStream_t stream);
/* get_token_penalty_multi_scores(_v2): csrc/gpu/token_penalty_multi_scores_v2.cu:19-139 (CPU twin
 * csrc/cpu/src/token_penalty_multi_scores.cc:18-85).  In place on fp32 logits [bs, length]; temperatures / bad_tokens may
 * be NULL (v1 op); workspace = bs*length int32. */
int b200_token_penalty_multi_scores(const int64_t* pre_ids, float* logits, const float* penalty_scores,
                                    const float* frequency_scores, const float* presence_scores, const float* temperatures,
                                    const int64_t* bad_tokens, const int64_t* cur_len, const int64_t* min_len,
                                    const int64_t* eos_token_id, int32_t* workspace, int64_t bs, int64_t length,
                                    int64_t length_id, int64_t bad_len, int64_t eos_len, cudaStream_t stream);
/* set_stop_value_multi_ends: v1 mode 2 csrc/gpu/stop_generation_multi_ends.cu:45-56 ; v2 …_v2.cu:35-59 */
int b200_set_stop_value_multi_ends(bool* stop_flags, int64_t* topk_ids, int64_t* next_tokens, const int64_t* end_ids,
                                   const int32_t* seq_lens, int64_t bs, int64_t end_length, int v2, cudaStream_t stream);
/* fused_get_rotary_embedding(input_ids, position_ids, head_dim_shape_tensor, prompt_num, theta, use_neox):
 * csrc/gpu/fused_get_rope.cu:40-223, called experimental/transformers/llama/modeling.py:799-803.
 * position_ids int64 [bsz, max_position_seq_length]; rope_embedding fp32 [2, bsz, 1, max_seq_length, head_dim] (cos, sin) with
 * angle = position_ids[b, s + prompt_num] * powf(theta, -2j/head_dim); use_neox != 0: value j at columns j and j + head_dim/2
 * (rotate-half, Llama/Qwen2), use_neox == 0: at columns 2j, 2j+1.  max_seq_length is input_ids.shape[1] in the reference. */
int b200_fused_get_rotary_embedding(const int64_t* position_ids, float* rope_embedding, int64_t bsz, int64_t max_seq_length,
                                    int64_t max_position_seq_length, int64_t head_dim, int64_t prompt_num, float theta,
                                    int use_neox, cudaStream_t stream);

/* step_paddle: csrc/gpu/step.cu:19-283 (free_and_dispatch_block + recover_block) — continuous-batching block bookkeeping of the
 * paged KV cache, called once per decode step: finished sequences return their decoder blocks to free_list; running sequences
 * that step into an unallocated block get one (pre-empting the largest holders into step_block_list when the list runs dry);
 * parked sequences are recovered when blocks are available again (lengths / stop flag / input_ids rebuilt from pre_ids).
 * All arguments are updated in place like the reference op (every tensor is an input aliased to an output there).  Sizes:
 * bsz = seq_lens_this_time.shape[0] (<= 1024), block_num_per_seq = block_tables.shape[1], length = input_ids.shape[1],
 * pre_id_length = pre_ids.shape[1]; the reference attribute `encoder_decoder_block_num` is unused by its kernels and omitted.
 * ONE launch, no host synchronisation (the reference copies recover_lens to the host between its two kernels); list order
 * is by sequence index (deterministic; the reference's atomics leave it timing dependent). */
int b200_step_paddle(bool* stop_flags, int32_t* seq_lens_this_time, const int32_t* ori_seq_lens_encoder,
                     int32_t* seq_lens_encoder, int32_t* seq_lens_decoder, int32_t* block_tables, int32_t* encoder_block_lens,
                     bool* is_block_step, int32_t* step_block_list, int32_t* step_lens, int32_t* recover_block_list,
                     int32_t* recover_lens, int32_t* need_block_list, int32_t* need_block_len, int32_t* used_list_len,
                     int32_t* free_list, int32_t* free_list_len, int64_t* input_ids, const int64_t* pre_ids,
                     const int64_t* step_idx, const int64_t* next_tokens, int64_t bsz, int64_t block_size,
                     int64_t block_num_per_seq, int64_t length, int64_t pre_id_length, int64_t first_token_id,
                     cudaStream_t stream);

/* retire_admit: the continuous-batching step step_paddle leaves to its caller (the reference's serving stack does it on the
 * host); call it right after b200_step_paddle on the same state, with a device-resident request queue: prompt_ids int64 packed,
 * prompt_offsets int32 [num_requests + 1], req_max_dec_len / req_min_dec_len int64 [num_requests], *cursor = next request.
 *   - a slot step_paddle recovered this step gets input_ids[b, 0] = its prompt's first token back;
 *   - a parked slot (is_block_step) returns its encoder blocks to free_list and adds them to used_list_len, so that
 *     step_paddle's recovery re-attaches all of its pages from position 0;
 *   - a stopped, not parked slot with slot_request[b] = r >= 0 retires: out_ids[r, :n] = pre_ids[b, 1:n] + next_tokens[b] with
 *     n = step_idx[b], out_lens[r] = n, the encoder blocks left in its row (step_paddle freed the decoder blocks and zeroed
 *     encoder_block_lens) back to free_list, slot_request = -1;
 *   - while no slot is parked (*step_lens == 0), empty slots take requests FIFO, in slot order, while the free list holds
 *     ceil(prompt / block_size) blocks for the head request (popped from its tail): input_ids row, seq_lens_this_time =
 *     seq_lens_encoder = ori_seq_lens_encoder = prompt, seq_lens_decoder = step_idx = 0, stop flag cleared, pre_ids row = -1,
 *     max/min_dec_len, slot_request;
 *   - header (int32 [B200_RA_HEADER_INTS], pinned device-mapped host memory, zeroed before the first call) receives the next
 *     step's token_num / max_q_len and the counters below.
 * One CTA (bsz <= 1024), list positions by prefix sums in slot order, no host synchronisation, graph-replayable.
 * max_prompt_len / max_seq_len = the queue's longest prompt / prompt + max_dec_len (host bounds, checked against the table
 * and input_ids widths); out_stride >= every max_dec_len, pre_id_length >= out_stride. */
enum {
  B200_RA_TOKEN_NUM = 0,    /* sum of seq_lens_this_time: rows of the next step */
  B200_RA_MAX_Q_LEN = 1,    /* max of seq_lens_this_time (1: a decode-only step) */
  B200_RA_RUNNING = 2,      /* slots with seq_lens_this_time > 0 */
  B200_RA_PENDING = 3,      /* requests not yet admitted */
  B200_RA_PARKED = 4,       /* *step_lens */
  B200_RA_DONE = 5,         /* 1 once every request has retired */
  B200_RA_FREE_BLOCKS = 6,  /* *free_list_len */
  B200_RA_PREEMPTIONS = 7,  /* cumulative over the calls since the header was zeroed */
  B200_RA_RECOVERIES = 8,   /* cumulative */
  B200_RA_ADMITTED = 9,     /* this call */
  B200_RA_RETIRED = 10,     /* this call */
  B200_RA_HEADER_INTS = 16
};
int b200_retire_admit(bool* stop_flags, bool* is_block_step, int32_t* seq_lens_this_time, int32_t* seq_lens_encoder,
                      int32_t* ori_seq_lens_encoder, int32_t* seq_lens_decoder, int64_t* step_idx, int64_t* pre_ids,
                      const int64_t* next_tokens, int64_t* input_ids, int32_t* block_tables, int32_t* encoder_block_lens,
                      int32_t* used_list_len, int32_t* free_list, int32_t* free_list_len, const int32_t* step_lens,
                      int64_t* max_dec_len, int64_t* min_dec_len, int32_t* slot_request, const int64_t* prompt_ids,
                      const int32_t* prompt_offsets, const int64_t* req_max_dec_len, const int64_t* req_min_dec_len,
                      int32_t* cursor, int64_t* out_ids, int32_t* out_lens, int32_t* header, int64_t bsz, int64_t block_size,
                      int64_t block_num_per_seq, int64_t length, int64_t pre_id_length, int64_t num_requests,
                      int64_t out_stride, int64_t max_prompt_len, int64_t max_seq_len, cudaStream_t stream);

/* save_output(x, not_need_stop, rank_id) replacement: csrc/gpu/save_with_output_msg.cc:28-52 (producer) / csrc/gpu/get_output.cc
 * (consumer), reader loop paddlenlp/utils/llm_utils.py:753-776.  Writes the step's message {flag, bsz, tokens...} (flag 1 =
 * running, -1 = finished: *stop_count >= bs or step >= last_step) into slot (step % num_slots) of `ring`, an int32 buffer of
 * num_slots x slot_stride in pinned device-mapped host memory, and publishes it by storing step + 1 into the slot's first word
 * last; `step_counter` (device int64) is the running step and is incremented.  No host synchronisation; graph-replayable. */
int b200_save_output_stream(const int64_t* next_tokens, const int32_t* stop_count, int32_t* ring, int64_t slot_stride,
                            int64_t num_slots, int64_t* step_counter, int64_t last_step, int64_t bs, cudaStream_t stream);

/* append_attention(qkv, key_cache, value_cache, seq_lens_encoder, seq_lens_decoder, seq_lens_this_time, padding_offsets,
 * cum_offsets, block_tables, ..., rotary_embs, ...): csrc/gpu/append_attention.cu:428-851, called
 * fused_transformer_layers.py:2215-2262 (FusedBlockMultiTransformer.compute_attn with config.append_attn).  ONE entry point for a
 * mixed batch over the paged KV cache: sequence b contributes seq_lens_this_time[b] rows of the packed projection
 * qkv [token_num, ldq] (rows cu_seqlens_q[b] ..), at absolute positions seq_lens_decoder[b] + i.  RoPE (rotate-half, tables
 * [rope_positions, 64] fp32) is applied to q and k in place, k and v are appended to the pages, and every row attends to cache
 * positions [0, its own]: prompts and prompt CHUNKS on top of a cached prefix (seq_lens_encoder[b] > 0 or more than one row)
 * through the flash kernel with page-gathered K/V, single decode rows through the decode kernel.  out [token_num, ldo].
 * max_q_len >= max(seq_lens_this_time) (host bound for the grid; the reference passes max_enc_len_this_time the same way).
 * cu_seqlens_q replaces padding_offsets / cum_offsets (same information; get_padding_offset produces it).
 * No host synchronisation.  Workspace: b200_append_attention_workspace_bytes(). */
int64_t b200_append_attention_workspace_bytes(int64_t B, int64_t num_heads, int64_t num_kv_heads, int64_t head_dim,
                                              int64_t num_splits);
int b200_append_attention(void* qkv, void* key_cache, void* value_cache, const int32_t* seq_lens_encoder,
                          const int32_t* seq_lens_decoder, const int32_t* seq_lens_this_time, const int32_t* cu_seqlens_q,
                          const int32_t* block_tables, const float* cos_table, const float* sin_table, void* out, void* workspace,
                          int64_t B, int64_t token_num, int64_t max_q_len, int64_t num_heads, int64_t num_kv_heads,
                          int64_t head_dim, int64_t num_blocks, int64_t block_size, int64_t max_blocks_per_seq,
                          int64_t rope_positions, int64_t ldq, int64_t ldo, float softmax_scale, int64_t num_splits,
                          cudaStream_t stream);

/* int8 paged KV cache (cachekv_int8_type="static"; append_attention's cache_int8 mode, append_attention_kernel.h:224).
 * key_cache / value_cache: uint8 [num_blocks, kvh, block_size, head_dim], the bf16 cache's shape and row formula with 1-byte
 * elements.  Per kv head a quantise scale s (cache_k_scale / cache_v_scale) and a dequantise scale o = 1 / s
 * (cache_k_out_scale / cache_v_out_scale), each bf16 [kvh].  A cache byte holds
 *     u = clamp(rne(bf16(s * x)), -127, 127) + 128
 * of the post-RoPE bf16 value x that the bf16 cache would hold (bf16 product, then round to nearest integer with ties to
 * even), for prompt and decode rows alike, and reads back as (u - 128) * o.  The attention kernels apply o once per kv head:
 * o_k on the softmax scale, o_v on the output; a dequantised value is never rounded to bf16.  Each entry point mirrors its bf16
 * twin above; a null scale array, an unsupported shape or an unsupported block size is an argument error before any launch.
 * head_dim must also be a multiple of 16.  The writers take the quantise scales, decode attention the dequantise scales,
 * b200_append_attention_c8 (which writes and reads) all four.  Workspaces are the bf16 twins'. */
int b200_write_cache_kv_paged_c8(const void* qkv, void* key_cache, void* value_cache, const int32_t* block_tables,
                                 const void* cache_k_scale, const void* cache_v_scale, const int32_t* seq_lens, int64_t B,
                                 int64_t S, int64_t num_heads, int64_t num_kv_heads, int64_t head_dim, int64_t block_size,
                                 int64_t max_blocks_per_seq, int64_t ld, cudaStream_t stream);
int b200_decode_rope_append_paged_c8(void* qkv, float* acc_f32_ws, const float* bias, void* key_cache, void* value_cache,
                                     const int32_t* block_tables, const void* cache_k_scale, const void* cache_v_scale,
                                     const float* cos_table, const float* sin_table, const int32_t* seq_lens, int64_t B,
                                     int64_t num_heads, int64_t num_kv_heads, int64_t head_dim, int64_t block_size,
                                     int64_t max_blocks_per_seq, int64_t ld, cudaStream_t stream);
int b200_decode_attention_paged_c8(const void* qkv, const void* key_cache, const void* value_cache, const int32_t* block_tables,
                                   const void* cache_k_out_scale, const void* cache_v_out_scale, const int32_t* seq_lens,
                                   void* out, void* workspace, int64_t B, int64_t num_heads, int64_t num_kv_heads,
                                   int64_t head_dim, int64_t num_blocks, int64_t block_size, int64_t max_blocks_per_seq,
                                   int64_t ld, float softmax_scale, int64_t num_splits, cudaStream_t stream);
int b200_append_attention_c8(void* qkv, void* key_cache, void* value_cache, const void* cache_k_scale, const void* cache_v_scale,
                             const void* cache_k_out_scale, const void* cache_v_out_scale, const int32_t* seq_lens_encoder,
                             const int32_t* seq_lens_decoder, const int32_t* seq_lens_this_time, const int32_t* cu_seqlens_q,
                             const int32_t* block_tables, const float* cos_table, const float* sin_table, void* out,
                             void* workspace, int64_t B, int64_t token_num, int64_t max_q_len, int64_t num_heads,
                             int64_t num_kv_heads, int64_t head_dim, int64_t num_blocks, int64_t block_size,
                             int64_t max_blocks_per_seq, int64_t rope_positions, int64_t ldq, int64_t ldo, float softmax_scale,
                             int64_t num_splits, cudaStream_t stream);

/* update_inputs: csrc/gpu/update_inputs.cu:18-82 */
int b200_update_inputs(bool* not_need_stop, int32_t* seq_lens_this_time, int32_t* seq_lens_encoder,
                       int32_t* seq_lens_decoder, int64_t* input_ids, const int64_t* stop_nums, const bool* stop_flags,
                       const bool* is_block_step, const int64_t* next_tokens, int64_t bsz, int64_t max_bsz,
                       int64_t input_ids_stride, cudaStream_t stream);
/* One fused state update per decode step of the dense-cache generate loop
 * (update_model_kwargs_for_generation, experimental/transformers/generation_utils.py:185-260): step_idx, length stop,
 * EOS stop, pre_ids history, seq_len_decoder, next/tgt ids, optional token log (column out_col, or *out_col_dev which is
 * then incremented on the device so that the step is CUDA-graph replayable), stop_count = number of stopped rows. */
int b200_generate_step_update(int64_t* next_tokens, bool* stop_flags, int64_t* step_idx, const int64_t* max_dec_len,
                              int32_t* seq_len_decoder, int64_t* pre_ids, int64_t pre_len, const int64_t* eos_ids,
                              int64_t eos_len, int64_t* out_tokens, int64_t out_stride, int64_t out_col,
                              int64_t* out_col_dev, int32_t* stop_count, int64_t bs, cudaStream_t stream);
int b200_argmax_f32(const float* logits, int64_t* out, int64_t rows, int64_t vocab, int64_t ld, cudaStream_t stream);
int b200_bf16_rows_to_f32(const void* src, float* dst, int64_t rows, int64_t cols, int64_t ld, cudaStream_t stream);
/* In-place fp32 softmax over each row of logits [rows, vocab] (row stride ld): `probs = F.softmax(logits)`,
 * experimental/transformers/generation_utils.py:327. */
int b200_softmax_f32(float* logits, int64_t rows, int64_t vocab, int64_t ld, cudaStream_t stream);
/* top_p_sampling_reject (csrc/gpu/sample_kernels/top_p_sampling_reject.cu:18-60, sampling.cuh:197-376): rejection sampling
 * of one token per row from probs [bs, vocab] restricted to the top-p nucleus; top_p [bs]; uniform [max_rounds, bs] are
 * the U(0,1) draws (the reference draws max_rounds = 32 per row from its generator inside the op); out [bs] int64.
 * top_p == 0 selects the arg max. */
int b200_top_p_sampling_reject(const float* probs, const float* top_p, const float* uniform, int64_t* out, int64_t bs,
                               int64_t vocab, int64_t ld, int64_t max_rounds, cudaStream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* B200NLP_H_ */
