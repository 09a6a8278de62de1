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
 *   out   half[H*head_dim]                                                                                 */
TCE_API int tce_attn_decode(tce_ctx *ctx, const void *qkv, void *k_cache, void *v_cache, const float *cos,
                            const float *sin, const int *pos, void *out, float alpha, int num_heads, int num_kv_heads,
                            int head_dim, int max_ctx);

/* Same module for sqlen = n > 1 (prompt processing): qkv half[n][(H + 2*KVH)*head_dim] holds the fused projections of n tokens at
 * positions pos0..pos0+n-1; q is rotated IN PLACE, rotated k and v are appended to the caches, out half[n][H*head_dim] receives
 * causal attention over cache rows 0..pos0+i for token i.  One flash kernel (mma.sync m16n8k16, fp32 softmax), no [n][T] score
 * tensor in HBM.  head_dim == 128.                                                                                            */
TCE_API int tce_attn_prefill(tce_ctx *ctx, void *qkv, void *k_cache, void *v_cache, const float *cos, const float *sin, void *out, float alpha,
                             int n, int pos0, int num_heads, int num_kv_heads, int head_dim, int max_ctx);

/* ---- small ops either side of the path -------------------------------------------------------------------
 * LlamaRMSNorm_cuda::forward (llm/src/ops/cuda/LlamaRMSNorm.cu:96-115): half in/out, fp32 gamma             */
TCE_API int tce_rmsnorm_f16(tce_ctx *ctx, const void *x, const float *gamma, void *y, int rows, int dim, float eps);
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
/* inputs resident: tokpos = device int[2] {token id, position}; logits stay on the device */
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
 * ids (4 bytes each) cross PCIe.  Single GPU (tp_size == 1).                                                                       */
TCE_API int tce_llama_generate(tce_llama *m, int first_token, int pos0, int n_predict, const tce_sampling *cfg, const int *history_host,
                               int n_history, int eos_id, int *out_tokens_host, int *n_out);
TCE_API const float *tce_llama_logits(tce_llama *m);          /* device float[vocab] */
TCE_API void *tce_llama_kv_cache(tce_llama *m, int layer, int which); /* which: 0 K, 1 V; half[KVH][max_ctx][hd] */
TCE_API int tce_llama_kernels_per_step(tce_llama *m);
/* ---- tensor-parallel decode across the GPUs of one box (one process per GPU) --------------------------------
 * cfg.tp_size = P > 1: heads / kv heads / hidden_dim / vocab_size in tce_llama_config are the LOCAL (1/P) sizes and the
 * weights are the local shards (q,k,v,gate,up,lm_head: row shards; o,down: column (input-channel) shards repacked as
 * [E][IC/P]).  The all-reduce after o_proj and down_proj runs over NVLink peer memory inside the GEMV kernels.
 * Setup: every rank exports a 64-byte IPC handle, the host exchanges them (e.g. torch.distributed.all_gather) and
 * every rank connects with the P handles in rank order.  tce_llama_decode_host then returns the local logits shard
 * (float[vocab_local]) and the GLOBAL greedy token; all ranks must call it with the same token/pos sequence.   */
TCE_API int tce_llama_tp_handle(tce_llama *m, void *handle_out_64_bytes);
TCE_API int tce_llama_tp_connect(tce_llama *m, const void *handles_P_times_64_bytes);
/* debugging aid: device pointers of the step's intermediate buffers: 0 residual float[E], 1 qkv half[(H+2KVH)*hd],
 * 2 attention output half[H*hd], 3 SiLU(gate)*up half[F] (values of the LAST layer after a step) */
TCE_API void *tce_llama_debug_buffer(tce_llama *m, int which);
/* measurement aid: enqueue only the W4A16 GEMV launches of one decode step (4 per layer + lm_head, the same fused
 * kernels with the same arguments) so the dominant kernel can be timed with CUDA events; returns the launch count */
TCE_API int tce_llama_enqueue_gemvs(tce_llama *m);

#ifdef __cplusplus
}
#endif
#endif /* TCE_B200_H */
