// kernels_attn.h -- launch interface of the decode attention / small fused ops (internal).
#pragma once
#include "kernels.h"

namespace tce {

struct AttnDecodeArgs {
    const __half *qkv;   // [(H + 2*KVH) * head_dim] projections of the current token (q | k | v), pre-RoPE
    __half *k_cache;     // [KVH][max_ctx][head_dim]
    __half *v_cache;     // [KVH][max_ctx][head_dim]
    const float *cos;    // [max_ctx][head_dim]  (reference rotary_emb/cos_cached layout)
    const float *sin;    // [max_ctx][head_dim]
    const int *pos;      // device scalar: index of the token being decoded (= number of cached tokens)
    __half *out;         // [H * head_dim]
    float alpha;         // qk_bmm alpha (1/sqrt(head_dim))
    int num_heads, num_kv_heads, head_dim, max_ctx;
    int chunk;           // cached positions per CTA
    int nsplit_max;      // filled by the launcher
    float *ws;           // filled by the launcher
    unsigned *counters;  // filled by the launcher
};
cudaError_t launch_attn_decode(Ctx *ctx, AttnDecodeArgs a, bool pdl);

// prompt processing (sqlen = n > 1): RoPE + KV append for rows pos0..pos0+n-1, causal attention over the cache
struct AttnPrefillArgs {
    __half *qkv;         // [n][(H + 2*KVH) * head_dim]; q is rotated in place
    __half *k_cache;     // [KVH][max_ctx][head_dim]
    __half *v_cache;
    const float *cos, *sin;
    __half *out;         // [n][H * head_dim]
    float alpha;
    int n, pos0, num_heads, num_kv_heads, head_dim, max_ctx;
};
cudaError_t launch_attn_prefill(Ctx *ctx, const AttnPrefillArgs &a);
cudaError_t launch_embedding_rows(Ctx *ctx, const __half *table, const int *tokens, float *resid, int n, int E);
cudaError_t launch_rmsnorm_rows_f32(Ctx *ctx, const float *x, const float *gamma, __half *y, int rows, int dim, float eps);

// resid_f32[E] = (float) table[token][:]   (reference: CPU Embedding + float2half, cuda/Int4llamaDecoder.cu:62-69)
cudaError_t launch_embedding(Ctx *ctx, const __half *table, const int *token, float *resid, int E, bool pdl, int rows = 0, int max_ctx = 0, int *safe = nullptr);
// argmax over fp32 logits -> int (first index of the maximum, like arg_max.cc)
cudaError_t launch_argmax(Ctx *ctx, const float *logits, int n, int *out, bool pdl);

// device sampler (sampling.cu): llm/src/Generate.cc:14-136, 304-327 in the order of LLaMAGenerate.cu:112-166
struct SampleArgs {
    float *logits;            // [n_vocab], penalties are applied in place
    int n_vocab;
    int top_k;                // <= 0: whole vocabulary (temp > 0 needs top_k <= 1024)
    float top_p, temp, repeat_penalty, frequency_penalty, presence_penalty;
    int repeat_last_n;        // < 0: the whole history ring
    unsigned long long seed, draw_index;
    int *hist = nullptr;      // ring of recent tokens [hist_cap]; entries before the first real token read as 0
    int *hist_head = nullptr; // tokens written so far (device); with a fixed window pass hist + a head equal to the window length
    int hist_cap = 0;
    int eos_id = -1;
    int *out_token = nullptr; // the sampled id
    int *tokpos = nullptr;    // {token, position} of the next decode step: token <- id, position <- position + 1
    int *out_list = nullptr;  // generated ids
    int *out_count = nullptr;
    int out_cap = 0;
    int *stop = nullptr;      // set to 1 when eos_id is drawn; a set flag turns the kernel into a no-op
    int *dbg_ids = nullptr;   // optional: surviving candidates (sorted) and their final probabilities
    float *dbg_probs = nullptr;
    int *dbg_size = nullptr;
};
cudaError_t launch_sample(Ctx *ctx, const SampleArgs &a, cudaStream_t stream);
// standalone RMSNorm fp16 -> fp16 with fp32 gamma (reference LlamaRMSNorm_cuda, ops/cuda/LlamaRMSNorm.cu:68-115)
cudaError_t launch_rmsnorm_f16(Ctx *ctx, const __half *x, const float *gamma, __half *y, int rows, int dim, float eps);
// LayerNormQ::forward (llm/src/ops/LayerNormQ.cc:12-52), bit-exact (serial fp32 sums in the reference's order)
cudaError_t launch_layernorm_q(Ctx *ctx, const float *x, const float *weight, const float *bias, int8_t *out, int rows, int dim);
cudaError_t launch_add_f32(Ctx *ctx, const float *a, const float *b, float *out, long long n);

}  // namespace tce
