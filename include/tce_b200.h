/*
 * tce_b200.h -- C ABI of libtce_b200.so: the H100 (sm_90a) implementation of TinyChatEngine's quantized-linear
 * hot path (W4A16 AWQ GEMV/GEMM, W8A8 SmoothQuant GEMM, per-token KV-cache attention).
 *
 * Boundary contract (SURVEY.md 8(b)): plain pointers and sizes, no C++/torch types.  Every data pointer is a
 * DEVICE-accessible pointer (cudaMalloc or cudaMallocManaged, which is what the reference allocates,
 * llm/src/nn_modules/cuda/utils.cu:93-96) unless the function name ends in `_host`.  The caller owns all data
 * buffers; the library owns only its context workspaces.  All calls are asynchronous on the context's stream
 * (like the reference's default-stream kernels) except `_host` calls, which return after their D2H copy.
 * Return value: 0 on success, negative tce_status otherwise; tce_last_error() gives the message.
 * There is NO CPU fallback: without a CUDA device every compute entry point fails with TCE_ERR_CUDA.
 *
 * Each entry point names the reference interface it replaces (file:line under the reference tree).
 */
#ifndef TCE_B200_H
#define TCE_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TCE_API __attribute__((visibility("default")))

typedef enum tce_status {
    TCE_OK = 0,
    TCE_ERR_INVALID = -1,     /* bad shape / null pointer / unsupported group size (reference: assert / exit(1)) */
    TCE_ERR_UNSUPPORTED = -2,
    TCE_ERR_CUDA = -3
} tce_status;

typedef struct tce_ctx tce_ctx;

/* ---- context ------------------------------------------------------------------------------------------ */
TCE_API int tce_version(void);
TCE_API const char *tce_last_error(void);
TCE_API int tce_ctx_create(int device, tce_ctx **out);
TCE_API int tce_ctx_destroy(tce_ctx *ctx);
/* cudaStream_t as void*; NULL = legacy default stream (what the reference launches on) */
TCE_API int tce_ctx_set_stream(tce_ctx *ctx, void *cuda_stream);
TCE_API int tce_ctx_synchronize(tce_ctx *ctx);
/* knobs: "gemv_impl" (0 simple / 1 tma+mma), "gemv_ctas_per_sm", "use_pdl", "attn_chunk" */
TCE_API int tce_ctx_set_option(tce_ctx *ctx, const char *name, int value);
TCE_API int tce_ctx_num_sms(tce_ctx *ctx);
/* measurement aid (option "gemv_debug" = 1): per-CTA phase timestamps of the last W4A16 GEMV launch, 8 x u64
 * globaltimer ns per CTA: entry, first TMA issued, activations staged, first stage landed, consumers done,
 * epilogue done, first tile flushed.  Returns the number of CTAs copied.                                       */
TCE_API int tce_ctx_read_gemv_timing(tce_ctx *ctx, unsigned long long *host_out, int max_ctas);

/* ---- W4A16, QM_CUDA layout ------------------------------------------------------------------------------
 * Replaces MatmulOperator::gemv_forward_cuda (kernels/cuda/gemv_cuda.cu:213-260), called by
 * Linear_half_int4::forward (llm/src/ops/cuda/linear.cu:5-40).
 *   x half[M][IC], w uint32[OC][IC/8], zeros uint32[OC][zeros_w], scales half[OC][zeros_w*8], y half[M][OC]
 *   zeros_w = tce_zeros_width(IC, group); group 128 (QK under QM_CUDA, llm/include/common.h:17-21) or 64 (gemv_kernel_g64,
 *   kernels/cuda/gemv_cuda.cu:68-123: GEMV only; the GEMM entry point takes 128).
 * Any M: M <= 8 is one pass over the weights, larger M loops in blocks of 8 rows.                        */
TCE_API int tce_zeros_width(int in_features, int group_size);
TCE_API int tce_w4a16_gemv(tce_ctx *ctx, const void *x, const void *w, const void *zeros, const void *scales, void *y,
                           int M, int IC, int OC, int group_size);
/* Same contract; the slot of the reference's declared-but-undefined prefill GEMM
 * MatmulOperator::gemm_forward_cuda (kernels/matmul.h:142-145).                                            */
TCE_API int tce_w4a16_gemm(tce_ctx *ctx, const void *x, const void *w, const void *zeros, const void *scales, void *y,
                           int M, int IC, int OC, int group_size);

/* fp16-accumulate reference of the AWQ-GEMM layout, replaces MatmulOperator::naive_mat_mul_fp16_int4
 * (kernels/cuda/matmul_int4.cu:8-48, call site Linear_FP16_int4_ref::forward_ref llm/src/ops/cuda/linear.cu:43-76):
 * A half[M][IC], B int32[IC][OC/8] nibble order 0 2 4 6 1 3 5 7, scales half[IC/block][OC], zero 8, C half[M][OC].
 * Bit-identical to the host reference (float op + round to half, serial k).                                   */
TCE_API int tce_naive_fp16_int4(tce_ctx *ctx, const void *A, const void *B, const void *scales, void *C, int M, int IC, int OC,
                                int block_size);
/* fp32 C[M][N] = A[M][K] * B[N][K]^T, serial k, no FMA: MatmulOperator::mat_mul_accelerator_transposed_fastover_column
 * of the CUDA build (kernels/cuda/matmul_ref_fp32.cc:11-34).                                                   */
TCE_API int tce_f32_matmul_transposed(tce_ctx *ctx, const float *A, const float *B, float *C, int M, int N, int K);

/* ---- W8A8 family -----------------------------------------------------------------------------------------
 * Replaces MatmulOperator::mat_mul_accelerator_int8_fast_* (kernels/ref/matmul_ref_int8.cc:11-192).
 * variant: 0 bias int8 -> int8 out (2x2_32unroll / 32unroll_over_column), 1 nobias -> int8 (…_nobias),
 *          2 bias fp32 -> fp32 out (…_bfp32_ofp32[_over_column]), 3 nobias -> fp32 (…_nobias_ofp32)
 * batch != 0: row i of A uses slab B[i][N][K] (…_nobias_batch / …_nobias_ofp32_batch; variants 1 and 3 only)
 * A int8[M][K], B int8[N][K], bias int8[N] | float[N] | NULL, C int8[M][N] | float[M][N].  Bit-exact.   */
TCE_API int tce_w8a8_matmul(tce_ctx *ctx, int variant, int batch, const void *A, const void *B, const void *bias,
                            void *C, int M, int N, int K, float alpha, float beta, int q_min, int q_max);

/* int8 attention core of Int8OPTAttention::forward (llm/src/nn_modules/Int8OPTAttention.cc:183-284): everything between the
 * q/k/v projections and out_proj -- shape(), cat_past_keys_values, BMM_S8T_S8N_F32T(qk_alpha), batch_Add(mask), softmax,
 * round(p*127), transpose_1_2idx, BMM_S8T_S8N_S8T(pv_alpha), unshape().  Bit-identical to the CPU reference.
 *   q8,k8,v8 int8 [sqlen][H*hd] (the three projections' outputs);  attn_out int8 [sqlen][H*hd]
 *   past_k/past_v int8 [H][past][hd] with `past_head_stride` bytes between heads (ignored when past == 0)
 *   final_k/final_v int8 [H][past+sqlen][hd] with `final_head_stride` between heads (Int8OPTAttention_output::past_key_value).
 *     Passing final == past with equal strides (>= (past+sqlen)*hd) updates a preallocated cache in place: only the new rows
 *     are written.
 *   mask fp32 [sqlen][past+sqlen] (Int8OPTAttention_input::attention_mask) or NULL for the causal mask.
 * hd % 4 == 0, hd <= 512.                                                                                                     */
TCE_API int tce_opt_int8_attention(tce_ctx *ctx, const void *q8, const void *k8, const void *v8, const void *past_k, const void *past_v,
                                   long long past_head_stride, void *final_k, void *final_v, long long final_head_stride, const float *mask,
                                   float qk_alpha, float pv_alpha, int sqlen, int past, int num_heads, int head_dim, void *attn_out);

/* ---- per-token KV-cache attention (fp16, GQA) ------------------------------------------------------------
 * Replaces the body of Int4llamaAttention::forward between qkv_proj and o_proj
 * (llm/src/nn_modules/cuda/Int4llamaAttention.cu:128-217; GQA mapping non_cuda/Int4llamaAttention.cc:166-184).
 *   qkv   half[(H + 2*KVH)*head_dim]  current token's q|k|v projections (pre-RoPE)
 *   k_cache, v_cache half[KVH][max_ctx][head_dim]  appended in place at *pos
 *   cos, sin float[max_ctx][head_dim]  (rotary_emb/cos_cached layout)
 *   pos   device int: index of the current token == number of tokens already cached
 *   out   half[H*head_dim]
 * The split workspace belongs to the context: the first call, and a call with a larger shape than any before it, allocates it, which
 * synchronises the device (so such a call cannot run inside a stream capture).                                                */
TCE_API int tce_attn_decode(tce_ctx *ctx, const void *qkv, void *k_cache, void *v_cache, const float *cos,
                            const float *sin, const int *pos, void *out, float alpha, int num_heads, int num_kv_heads,
                            int head_dim, int max_ctx);

/* Same module for sqlen = n > 1 (prompt processing): qkv half[n][(H + 2*KVH)*head_dim] holds the fused projections of n tokens at
 * positions pos0..pos0+n-1; q is rotated IN PLACE, rotated k and v are appended to the caches, out half[n][H*head_dim] receives
 * causal attention over cache rows 0..pos0+i for token i.  One flash kernel (mma.sync m16n8k16, fp32 softmax), no [n][T] score
 * tensor in HBM.  head_dim == 128.                                                                                            */
TCE_API int tce_attn_prefill(tce_ctx *ctx, void *qkv, void *k_cache, void *v_cache, const float *cos, const float *sin, void *out, float alpha,
                             int n, int pos0, int num_heads, int num_kv_heads, int head_dim, int max_ctx);

/* Same module for n <= 8 consecutive tokens of ONE sequence (the span step's attention): qkv half[n][(H + 2*KVH)*head_dim] holds the
 * projections of the tokens at positions pos0..pos0+n-1 (pre-RoPE, not modified); rotated k and v are appended to the caches at those rows,
 * out half[n][H*head_dim] receives causal attention over cache rows 0..pos0+i for token i.  A CTA reads each cached row of its context split
 * once for all n * H/KVH query rows.  The split is the context's "attn_chunk", lowered to the largest multiple of 16 whose CTA fits shared
 * memory.  Workspace as tce_attn_decode.  head_dim == 128; 1 <= n <= 8, 0 <= pos0 <= max_ctx - n.                                      */
TCE_API int tce_attn_span(tce_ctx *ctx, const void *qkv, void *k_cache, void *v_cache, const float *cos, const float *sin, void *out, float alpha,
                          int n, int pos0, int num_heads, int num_kv_heads, int head_dim, int max_ctx);

/* ---- small ops either side of the path -------------------------------------------------------------------
 * LlamaRMSNorm_cuda::forward (llm/src/ops/cuda/LlamaRMSNorm.cu:96-115): half in/out, fp32 gamma             */
TCE_API int tce_rmsnorm_f16(tce_ctx *ctx, const void *x, const float *gamma, void *y, int rows, int dim, float eps);
/* device int *out = index of the first maximum of device float x[n] (arg_max.cc); an input with no value greater than -inf (all -inf
 * or NaN) gives 0 */
TCE_API int tce_argmax_f32(tce_ctx *ctx, const float *x, int n, int *out);
/* LayerNormQ::forward (llm/src/ops/LayerNormQ.cc:12-52): fp32 [rows][dim] -> int8 [rows][dim], eps 1e-5, std::round.  Bit-exact: the two
 * row sums run serially in the reference's order (the int8 result depends on their last bit near rounding ties).            */
TCE_API int tce_layernorm_q(tce_ctx *ctx, const float *x, const float *weight, const float *bias, void *out_int8, int rows, int dim);
/* out = a + b (fp32): the residual add of Int8OPTDecoderLayer::forward (llm/src/nn_modules/Int8OPTDecoderLayer.cc:10-22,38,56) */
TCE_API int tce_add_f32(tce_ctx *ctx, const float *a, const float *b, float *out, long long n);

/* ---- fused Llama decode step -----------------------------------------------------------------------------
 * The call sites of the path: Int4llamaDecoderLayer::forward / Int4llamaDecoder::forward /
 * Int4LlamaForCausalLM::forward (llm/src/nn_modules/cuda/Int4llama{DecoderLayer,Decoder,ForCausalLM}.cu)
 * restated as one CUDA graph per token: embedding -> L x [RMSNorm+QKV GEMV, RoPE+KV-append+attention,
 * o_proj GEMV (+residual), RMSNorm+gate/up GEMV (+SiLU*mul), down GEMV (+residual)] -> RMSNorm+lm_head.  */
typedef struct tce_w4_tensor {
    const void *w;      /* uint32[oc][ic/8]    */
    const void *zeros;  /* uint32[oc][zeros_w] */
    const void *scales; /* half[oc][zeros_w*8] */
    int oc, ic;
} tce_w4_tensor;

typedef struct tce_llama_layer {
    tce_w4_tensor q, k, v, o, gate, up, down;
    const float *input_norm; /* fp32 gamma[embed_dim] */
    const float *post_norm;
} tce_llama_layer;

typedef struct tce_llama_config {
    int num_layers, num_heads, num_kv_heads, head_dim, embed_dim, hidden_dim, vocab_size, max_ctx;
    float rms_eps, rope_theta, qk_alpha;
    /* tensor parallel shard of this process: heads/hidden are the LOCAL sizes when tp_size > 1 */
    int tp_rank, tp_size;
} tce_llama_config;

typedef struct tce_llama_weights {
    const void *embed_f16;          /* half[vocab][embed_dim] */
    const tce_llama_layer *layers;  /* [num_layers] */
    const float *final_norm;
    tce_w4_tensor lm_head;
    const float *rope_cos, *rope_sin; /* float[max_ctx][head_dim] or NULL: computed from rope_theta */
} tce_llama_weights;

typedef struct tce_llama tce_llama;

TCE_API int tce_llama_create(tce_ctx *ctx, const tce_llama_config *cfg, const tce_llama_weights *w, tce_llama **out);
TCE_API int tce_llama_destroy(tce_llama *m);
/* ---- loading the reference's model zoo format (SURVEY.md 8(f)2) --------------------------------------------------------------------
 * Build the model from a parameter tree on disk, as the reference's constructors do (Int4LlamaForCausalLM(param_path, config),
 * llm/src/nn_modules/cuda/Int4llamaForCausalLM.cu:7-15 and below): <dir>/decoder/{embed_tokens,norm,layer<i>/...}, <dir>/lm_head, INT4 ops
 * in the QM_CUDA flavour (weight_int4.bin / scaling_factor_int4.bin / zero_point_int4.bin, llm/tools/model_quantizer.py:35-66), q|k|v either
 * merged (self_attn/qkv_proj, llm/tools/llama_qkv_merger.py) or separate.  cfg gives the geometry (the reference's model_config); file
 * sizes are checked against it.  The model owns its device copies.  Single GPU.                                                    */
TCE_API int tce_llama_load_dir(tce_ctx *ctx, const char *dir, const tce_llama_config *cfg, tce_llama **out);
/* QM_x86 op (llm/tools/quantize_methods.py:188-243: uint8 [oc][ic/2] with byte e of each 64-weight run = w[e] | w[32+e] << 4, fp32 scales
 * [oc][ic/32], zero point 8) -> QM_CUDA op arrays (w uint32 [oc][ic/8], scales fp16 [oc][zeros_w*8], zeros uint32 [oc][zeros_w]) on the HOST:
 * exact dequantisation followed by the QM_CUDA quantisation rule (group 128).  Lossy by construction (32- vs 128-channel scales).  */
TCE_API int tce_w4_import_x86(const void *qs_u8, const float *scales_f32, int oc, int ic, void *w_out, void *scales_f16_out, void *zeros_out);
/* inputs resident: tokpos = device int[2] {token id, position}; logits stay on the device.  The pair is range-checked on the device, on
 * the persistent kernel and on the kernel-per-op step alike: a token or position out of range is refused and writes no KV row. */
TCE_API int tce_llama_decode(tce_llama *m, const int *tokpos_dev);
/* end to end: token/pos from the host, fp32 logits[vocab] copied back to `logits_host` (may be NULL) and the
 * greedy arg-max to *next_token (may be NULL); returns after the copies have completed */
TCE_API int tce_llama_decode_host(tce_llama *m, int token, int pos, float *logits_host, int *next_token);
/* Prompt processing (the reference's Int4LlamaForCausalLM::forward with sqlen = n > 1, cuda/Int4llamaForCausalLM.cu:20-47): n host
 * token ids at positions pos0..pos0+n-1 in one pass -- KV cache rows written, logits of the LAST position (the only row the
 * sampler reads, LLaMAGenerate.cu:160-166) copied to logits_host (may be NULL), greedy token to next_token (may be NULL).
 * Linears run as wgmma GEMMs, attention as a causal flash kernel.  Synchronous.  Single GPU (tp_size == 1).                */
TCE_API int tce_llama_prefill(tce_llama *m, const int *tokens_host, int n, int pos0, float *logits_host, int *next_token);
/* ---- sampling + generate loop on the device (SURVEY.md 8(f)3) -------------------------------------------------------------
 * The reference copies n_vocab logits to the host every token and samples there (llm/src/nn_modules/cuda/LLaMAGenerate.cu:112-166 with
 * llm/src/Generate.cc:14-136,304-327: repetition / frequency / presence penalties over the last `repeat_last_n` tokens, then greedy when
 * temp <= 0, else top-k -> top-p -> temperature -> softmax -> one draw).  Same chain, same order, one kernel next to the logits.
 * Fields as in the reference's opt_params (llm/include/Generate.h:48-72); tail-free / typical / mirostat are not offered (identity at
 * the reference's defaults).  temp > 0 needs 1 <= top_k <= 1024 (TCE_ERR_UNSUPPORTED otherwise).  The draw is an inverse-CDF lookup with
 * a counter-based uniform of (seed, draw index).                                                                                  */
typedef struct tce_sampling {
    int top_k;
    float top_p, temp, repeat_penalty, frequency_penalty, presence_penalty;
    int repeat_last_n; /* < 0: the whole window */
    unsigned long long seed;
} tce_sampling;
/* one sampling step: logits_dev float[n_vocab] (penalised IN PLACE), window_host = the recent tokens, oldest first (may be NULL/0).
 * Returns the token in *token_host and, when the three cand_* pointers are given, the surviving candidates (logit-descending) with their
 * final probabilities (cand_* arrays must hold max(1, top_k) entries).  Synchronous.                                            */
TCE_API int tce_sample(tce_ctx *ctx, float *logits_dev, int n_vocab, const int *window_host, int n_window, const tce_sampling *cfg,
                       unsigned long long draw_index, int *token_host, int *cand_ids_host, float *cand_probs_host, int *cand_count_host);
/* generate loop: decode `first_token` at position pos0, sample, feed the sample back, ... for at most n_predict tokens or until eos_id
 * is drawn or the context is full.  history_host (n_history recent tokens, oldest first) seeds the penalty window.  Only the generated
 * ids (4 bytes each) cross PCIe.  Single GPU (tp_size == 1).  It is the loop of tce_llama_generate_batch on one sequence in slot 0, with
 * the single-sequence step: on return slot 0 holds exactly *n_out new rows, at pos0 .. pos0 + *n_out - 1 (the last id is not decoded),
 * whether it stopped at eos_id, at n_predict or at max_ctx.  TCE_ERR_INVALID, before anything is enqueued, for a bad first_token or pos0,
 * n_predict < 0, n_history outside [0, max_ctx], a NULL history with n_history > 0, or a NULL output.                                 */
TCE_API int tce_llama_generate(tce_llama *m, int first_token, int pos0, int n_predict, const tce_sampling *cfg, const int *history_host,
                               int n_history, int eos_id, int *out_tokens_host, int *n_out);
/* ---- batched decode: up to TCE_LLAMA_MAX_BATCH sequences per step, each in its own KV-cache slot -------------------------------------
 * One step streams the weights once for the whole batch (a batch-1 step's bytes are almost all weights).  A slot is one sequence's cache,
 * half[L][2][KVH][max_ctx][hd]; slot 0 is the cache of the single-sequence entry points above.  Single GPU: with tp_size > 1 every entry
 * point of this block returns TCE_ERR_UNSUPPORTED.  The batched step is one kernel per op (4 W4A16 GEMVs per layer + lm_head, each reading
 * its weights once for all rows), not the persistent kernel.                                                                          */
#define TCE_LLAMA_MAX_BATCH 8
/* grow the number of slots to n_slots (never shrinks; new slots are zeroed).  Slot 0 always exists.  Invalidates captured batch graphs. */
TCE_API int tce_llama_reserve_slots(tce_llama *m, int n_slots);
/* half[KVH][max_ctx][hd] of (slot, layer, which: 0 K, 1 V), or NULL */
TCE_API void *tce_llama_kv_cache_slot(tce_llama *m, int slot, int layer, int which);
/* tce_llama_prefill into the cache of `slot`; slot 0 is exactly tce_llama_prefill */
TCE_API int tce_llama_prefill_slot(tce_llama *m, int slot, const int *tokens_host, int n, int pos0, float *logits_host, int *next_token);
/* inputs resident: req_dev = device int[batch][3] {token, position, slot}, 1 <= batch <= TCE_LLAMA_MAX_BATCH.  The logits land in
 * tce_llama_batch_logits(m).  Entries are range-checked on the device: an entry with a token, position or slot out of range writes no KV row
 * in any slot (its logits row is meaningless) and the other entries proceed.  Two entries naming the same slot are the caller's error:
 * both append to that slot in an unspecified order.                                                                                       */
TCE_API int tce_llama_decode_batch(tce_llama *m, int batch, const int *req_dev);
/* end to end: batch host entries; logits_host float[batch][vocab] and next_tokens int[batch] (greedy) may be NULL.  TCE_ERR_INVALID, before
 * anything is enqueued, for a batch outside [1, TCE_LLAMA_MAX_BATCH], a slot >= the reserved count or named twice, a position outside
 * [0, max_ctx) or a token outside [0, vocab).  Returns after the copies have completed.                                                  */
TCE_API int tce_llama_decode_batch_host(tce_llama *m, int batch, const int *tokens, const int *positions, const int *slots, float *logits_host,
                                        int *next_tokens);
TCE_API const float *tce_llama_batch_logits(tce_llama *m);    /* device float[TCE_LLAMA_MAX_BATCH][vocab] */
/* Prompt processing of n_seqs prompts, 1 <= n_seqs <= TCE_LLAMA_MAX_BATCH, in ONE pass over the weights (the int4 weights are expanded to
 * fp16 once for all of them).  tokens_host = the prompts concatenated; prompt s has lengths[s] >= 1 tokens at positions pos0s[s].. in slot
 * slots[s].  logits_host float[n_seqs][vocab] (last position of each prompt) and next_tokens int[n_seqs] (greedy) may be NULL.
 * TCE_ERR_INVALID, before anything is enqueued, for n_seqs outside [1, TCE_LLAMA_MAX_BATCH], a length < 1, pos0 + length > max_ctx, a slot
 * >= the reserved count or named twice, or a token outside [0, vocab).  Synchronous.                                                   */
TCE_API int tce_llama_prefill_batch(tce_llama *m, int n_seqs, const int *tokens_host, const int *lengths, const int *pos0s, const int *slots,
                                    float *logits_host, int *next_tokens);
/* Teacher-forced scoring: the prompt pass of tce_llama_prefill_batch (same prompts, slots, positions, checks, and the same KV rows written),
 * plus the lm_head over EVERY row.  n = sum of lengths.  targets_host int[n]: the token whose log-probability row i reports, -1 for none;
 * NULL = the next token of the same prompt, and -1 on each prompt's last row.  Outputs, each may be NULL:
 *   logprobs_host float[n]  log_softmax(logits_i)[target_i], NaN where the target is -1
 *   greedy_host int[n]      arg-max of logits_i (lowest id on ties)
 *   greedy_logprobs_host float[n]
 *   logits_dev              device float[n][vocab] receiving every row's logits (the reference's logits[1][sqlen][vocab]); NULL = none are stored
 * The logits come from the fp16-expanded lm_head on the tensor cores (not the decode GEMV), and each row's results are bit-identical
 * whatever other prompts share the call.  TCE_ERR_INVALID, before anything is enqueued, for everything tce_llama_prefill_batch refuses
 * and for a target outside [-1, vocab); TCE_ERR_UNSUPPORTED with tp_size > 1.  Synchronous.                                             */
TCE_API int tce_llama_score_batch(tce_llama *m, int n_seqs, const int *tokens_host, const int *lengths, const int *pos0s, const int *slots,
                                  const int *targets_host, float *logprobs_host, int *greedy_host, float *greedy_logprobs_host, float *logits_dev);
typedef struct tce_gen_request {
    int first_token, pos0, slot;   /* decode first_token at pos0 in slot, as tce_llama_generate does for slot 0 */
    int n_predict, eos_id;         /* per-sequence budget and stop id (-1: none) */
    const int *history;            /* host, oldest first, may be NULL */
    int n_history;
    tce_sampling sampling;         /* per-sequence chain and seed */
} tce_gen_request;
/* Generate loop of `batch` sequences, 1 <= batch <= TCE_LLAMA_MAX_BATCH: per token one batched step and one device sampler launch (a block
 * per sequence, each with its own chain, seed, history window, EOS and budget).  A sequence stops when it draws its eos_id, when it has
 * n_predict ids (clamped to max_ctx - pos0, as tce_llama_generate clamps) or when its next position would be max_ctx; from then on it
 * appends no KV row.  On return slot s holds exactly n_out[s] new rows, at pos0 .. pos0 + n_out[s] - 1 (the last id is not decoded).
 * out_tokens_host int[batch][out_stride], n_out int[batch].  Only ids cross PCIe.  TCE_ERR_INVALID, before anything is enqueued, for a bad
 * batch, slot (unreserved or repeated), first_token, pos0, n_predict < 0, n_history outside [0, max_ctx], out_stride below a clamped
 * n_predict or a NULL pointer; TCE_ERR_UNSUPPORTED for temp > 0 without 1 <= top_k <= 1024.                                           */
TCE_API int tce_llama_generate_batch(tce_llama *m, int batch, const tce_gen_request *reqs, int *out_tokens_host, int out_stride, int *n_out);
/* ---- span step and greedy speculative decoding -------------------------------------------------------------------------------------------
 * Span step: tokens_host[0..n) at positions pos0 .. pos0 + n - 1 of ONE slot in one pass over the weights (the batched step's GEMVs at
 * M = n, then a causal multi-query attention that reads the slot's context once for all n rows).  logits_host float[n][vocab] (row i: the
 * logits after tokens_host[i]) and next_tokens int[n] (greedy) may be NULL.  Writes KV rows pos0 .. pos0 + n - 1 of the slot and no other
 * row of any slot.  TCE_ERR_INVALID, before anything is enqueued, for n outside [1, TCE_LLAMA_MAX_BATCH], pos0 < 0, pos0 + n > max_ctx, an
 * unreserved slot or a token outside [0, vocab); TCE_ERR_UNSUPPORTED with tp_size > 1, or when no context split of the span attention
 * fits the device's shared memory at this model's query heads per KV head (never on an H100 up to 8).  Returns after the copies.         */
TCE_API int tce_llama_decode_span_host(tce_llama *m, int slot, int pos0, int n, const int *tokens_host, float *logits_host, int *next_tokens);
typedef struct tce_lookup {
    int max_draft;            /* 0..7 drafts per step; 0 = the plain greedy loop */
    int ngram_min, ngram_max; /* 1 <= ngram_min <= ngram_max */
} tce_lookup;
typedef struct tce_lookup_stats {
    int steps;    /* passes over the weights */
    int drafted;  /* draft tokens verified */
    int accepted; /* emitted ids that were drafts */
} tce_lookup_stats;
/* Greedy generation on slot 0 with prompt-lookup drafts: the ids tce_llama_generate gives at temp <= 0 (penalties over the last
 * repeat_last_n ids of history + ids, then arg-max, lowest id on ties), up to rounding, in fewer passes over the weights.
 * Drafter, before each step: S = corpus ++ history ++ [first_token] ++ ids so far, d = min(max_draft, n_predict - |ids| - 1,
 * max_ctx - pos - 1) where pos is the position of S's last token.  For n = ngram_max down to ngram_min: take the last n tokens of S and
 * find their most recent earlier occurrence S[p .. p + n) with p + n < |S| (at least one token after it); the draft is S[p + n ..
 * min(p + n + d, |S|)).  The first n that matches wins; none (or d <= 0): no draft.
 * Step: without a draft, the single-sequence decode step; with d drafts, the span step on [last id, drafts] at M = d + 1.  Row j is then
 * sampled with the penalty window the one-token loop would have had after emitting drafts 0 .. j-1; drafts are accepted while row j's id
 * equals draft j, and the step emits the accepted drafts plus the id of the first rejected row (of row d when all were accepted), cut at
 * eos_id (inclusive) and at n_predict (clamped to max_ctx - pos0).  The host reads each step's ids back to draft the next one.
 * KV rows of slot 0: rows pos0 .. pos0 + *n_out - 1 hold first_token and ids[0 .. *n_out - 2] (the last id is not decoded); rows
 * pos0 + *n_out .. min(max_ctx, pos0 + *n_out + max_draft) - 1 may hold rows of rejected drafts; no other row of any slot changes.
 * stats may be NULL.  TCE_ERR_INVALID, before anything is enqueued, for a bad first_token or pos0, n_predict < 0, n_history outside
 * [0, max_ctx], n_corpus < 0, a NULL array with a non-zero count, NULL n_out (or out_tokens with n_predict > 0), max_draft outside [0, 7],
 * ngram_min < 1 or ngram_min > ngram_max; TCE_ERR_UNSUPPORTED for temp > 0, tp_size > 1, or max_draft > 0 on a model the span step
 * refuses as unsupported.                                                                                                              */
TCE_API int tce_llama_generate_lookup(tce_llama *m, int first_token, int pos0, int n_predict, const tce_sampling *cfg, const int *history_host,
                                      int n_history, const int *corpus_host, int n_corpus, const tce_lookup *lk, int eos_id, int *out_tokens_host,
                                      int *n_out, tce_lookup_stats *stats);
/* ---- speculative sampling (any temp) --------------------------------------------------------------------------------------------------
 * Acceptance rule of one step (speculative sampling, Leviathan et al. 2023 / Chen et al. 2023, with a one-hot draft distribution).  Inputs:
 * the penalty sequence so far (h entries), d drafts x_0 .. x_{d-1}, and d + 1 logits rows, row j = the logits after [last, x_0 .. x_{j-1}].
 * For each row j:
 *   1. the chain of tce_sample (penalties over the last repeat_last_n entries of sequence ++ x_{<j}, top-k, top-p, temperature, softmax)
 *      gives candidates c_j with probabilities p_j;
 *   2. q_j = p_j[i*] when j < d and x_j = c_j[i*], else 0 (x_j cut by top-k / top-p; the last row: q_d = 0);
 *   3. u_j = the uniform of draw index h + j (the one tce_llama_generate uses for its (h + j)-th id), and a_j = the uniform of the same
 *      index in the stream of seed ^ TCE_SPEC_ACCEPT_STREAM;
 *   4. r_j: with q_j = 0 the plain inverse-CDF draw with u_j (bit for bit tce_sample's); otherwise, with S = the sum of p_j[i] over i != i*
 *      (candidate order, fp32) and t = u_j * S (one fp32 multiply), the first i != i* whose running sum over i != i* exceeds t (the last
 *      i != i* if none).  S = 0: the row counts as accepted.
 * k = the first j < d whose draft is not accepted (a_j < q_j is false), d if every draft is.  The step emits x_0 .. x_{k-1}, then r_k, cut
 * at eos_id (inclusive) and at the budget; accepted = min(k, emitted).  At temp <= 0 this is the greedy rule: q_j = 1 exactly when x_j is
 * the arg-max, and r_k is the arg-max.  Without drafts it is the plain sampled step.                                                     */
#define TCE_SPEC_ACCEPT_STREAM 0xD1B54A32D192ED03ull
/* The rule alone, on a caller's logits: logits_dev float[rows][ld] (row j: n_vocab floats, penalised IN PLACE), 1 <= rows <= 8,
 * drafts_host int[rows - 1] (may be NULL when rows == 1), window_host = the penalty sequence, oldest first (may be NULL/0; entries before it
 * read as 0), draw_index = h.  ids_host int[rows] receives the emitted ids, *n_out their count, *n_accepted the drafts among them, *stop 1
 * when eos_id was emitted; q_host float[rows] (may be NULL) receives q_0 .. q_{rows-1}.  TCE_ERR_INVALID for a bad argument, budget < 1 or
 * ld < n_vocab; TCE_ERR_UNSUPPORTED for temp > 0 without 1 <= top_k <= 1024 when n_vocab > 1024.  Synchronous.                          */
TCE_API int tce_spec_accept(tce_ctx *ctx, float *logits_dev, int rows, long long ld, int n_vocab, const int *drafts_host, const int *window_host,
                            int n_window, const tce_sampling *cfg, unsigned long long draw_index, int eos_id, int budget, int *ids_host, int *n_out,
                            int *n_accepted, int *stop, float *q_host);
/* tce_llama_generate_lookup at any temp: the same arguments, drafter, steps, stop rules, KV rows, stats and refusals, except that temp > 0
 * is accepted (it needs 1 <= top_k <= 1024 when vocab > 1024, TCE_ERR_UNSUPPORTED otherwise), and each step applies the rule above with
 * h = n_history + ids so far.  The emitted ids have the distribution of tce_llama_generate's with the same fields, but are not its ids,
 * except at max_draft = 0 or temp <= 0, where they are.                                                                                  */
TCE_API int tce_llama_sample_lookup(tce_llama *m, int first_token, int pos0, int n_predict, const tce_sampling *cfg, const int *history_host,
                                    int n_history, const int *corpus_host, int n_corpus, const tce_lookup *lk, int eos_id, int *out_tokens_host,
                                    int *n_out, tce_lookup_stats *stats);
/* KV-cache row copy: rows src_pos .. src_pos + n - 1 of slot src_slot to rows dst_pos_host[i] .. dst_pos_host[i] + n - 1 of slot
 * dst_slots_host[i], for each of the n_dst destinations, in every layer, K and V, every KV head.  The source rows are read once for all
 * destinations.  The cache holds keys after RoPE, so a K row that moves by d = dst_pos - src_pos is rotated by d: rotate-half (dim j with
 * j + 64, as the prompt pass applies it) with c = cos[|d|], s = sign(d) * sin[|d|] from the model's own tables (generated from rope_theta,
 * the caller's, or the loaded tree's): r_j = x_j c_j - x_{j+64} s_j, r_{j+64} = x_{j+64} c_{j+64} + x_j s_{j+64}, every product and sum
 * rounded on its own in fp32 (no FMA), then rounded to fp16.  V rows, and K rows with d = 0, are copied bit for bit.  With one destination
 * in the source slot the ranges may overlap, in either direction: the result is that of copying through a temporary (memmove).  No other
 * row of any slot changes.  n = 0 does nothing.  Forking a prompt into other slots is d = 0; the context shift of a full slot (keep rows
 * [0, n_keep), drop the next n_discard, move the rest down) is one copy inside the slot with d = -n_discard.  Asynchronous on the context's
 * stream, ordered with the decode steps and generate loops; the slot table does not change, so no captured graph is dropped.
 * TCE_ERR_INVALID, before anything is enqueued, for n_dst outside [1, TCE_LLAMA_MAX_BATCH], n < 0, an unreserved slot, a source or
 * destination range outside [0, max_ctx), two destinations whose ranges overlap in the same slot, or a destination that overlaps the source
 * while n_dst > 1; TCE_ERR_UNSUPPORTED with tp_size > 1.                                                                                   */
TCE_API int tce_llama_kv_copy(tce_llama *m, int src_slot, int src_pos, int n, int n_dst, const int *dst_slots_host, const int *dst_pos_host);
TCE_API const float *tce_llama_logits(tce_llama *m);          /* device float[vocab] */
TCE_API void *tce_llama_kv_cache(tce_llama *m, int layer, int which); /* which: 0 K, 1 V; half[KVH][max_ctx][hd] */
TCE_API int tce_llama_kernels_per_step(tce_llama *m);
/* ---- tensor-parallel decode across the GPUs of one box (one process per GPU) --------------------------------
 * cfg.tp_size = P > 1: heads / kv heads / hidden_dim / vocab_size in tce_llama_config are the LOCAL (1/P) sizes and the
 * weights are the local shards (q,k,v,gate,up,lm_head: row shards; o,down: column (input-channel) shards repacked as
 * [E][IC/P]).  The all-reduce after o_proj and down_proj runs over NVLink peer memory inside the persistent decode kernel, so
 * tensor parallelism needs that kernel: tce_llama_create refuses tp_size > 1 with TCE_PERSISTENT=0, and tce_llama_tp_connect returns
 * TCE_ERR_UNSUPPORTED, with the reason, for a local shard outside the kernel's envelope.
 * Setup: every rank exports a 64-byte IPC handle, the host exchanges them (e.g. torch.distributed.all_gather) and
 * every rank connects with the P handles in rank order.  tce_llama_decode_host then returns the local logits shard
 * (float[vocab_local]) and the GLOBAL greedy token; all ranks must call it with the same token/pos sequence.   */
TCE_API int tce_llama_tp_handle(tce_llama *m, void *handle_out_64_bytes);
TCE_API int tce_llama_tp_connect(tce_llama *m, const void *handles_P_times_64_bytes);
/* debugging aid: device pointers of the batched step's intermediate buffers, TCE_LLAMA_MAX_BATCH rows each (row b = request b of the last
 * batched or span step; the kernel-per-op single-sequence step, TCE_PERSISTENT=0, writes row 0): 0 residual float[E], 1 qkv
 * half[(H+2KVH)*hd], 2 attention output half[H*hd], 3 SiLU(gate)*up half[F] (values of the LAST layer after a step); NULL until those
 * buffers exist (the persistent kernel keeps its intermediates on chip).  4: the persistent kernel's phase timestamps (TCE_PK_DEBUG=1). */
TCE_API void *tce_llama_debug_buffer(tce_llama *m, int which);
/* measurement aid: enqueue only the W4A16 GEMV launches of one decode step (4 per layer + lm_head, the same fused
 * kernels with the same arguments) so the dominant kernel can be timed with CUDA events; returns the launch count */
TCE_API int tce_llama_enqueue_gemvs(tce_llama *m);

#ifdef __cplusplus
}
#endif
#endif /* TCE_B200_H */
