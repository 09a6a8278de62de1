// kernels_attn.h -- launch interface of the decode attention / small fused ops (internal).
#pragma once
#include "kernels.h"

struct tce_sampling;  // include/tce_b200.h

namespace tce {

// Decode attention (attention.cu) of `seqs` sequences of n consecutive rows each: sequence s is grid.z = s and owns rows s * n .. s * n + n - 1
// of qkv / out, and row s * n + i is its position pos0_s + i.  The kernel rotates and appends the n new K / V rows of each sequence, then runs
// causal attention: row i sees cache rows 0..pos0_s + i.  Every row has its own split records and every sequence its own split counters in
// the workspace.  n = 1 is the per-token step of `seqs` sequences; seqs = 1, n > 1 is the span step of one sequence.
constexpr int kMaxSpan = 8;
struct AttnDecodeArgs {
    const __half *qkv;   // [seqs * n][qkv_stride]: the (H + 2*KVH) * head_dim projections of each row (q | k | v), pre-RoPE
    __half *out;         // [seqs * n][out_stride]: H * head_dim
    int qkv_stride, out_stride;  // elements between consecutive rows
    const float *cos;    // [max_ctx][head_dim]  (reference rotary_emb/cos_cached layout)
    const float *sin;    // [max_ctx][head_dim]
    float alpha;         // qk_bmm alpha (1/sqrt(head_dim))
    int num_heads, num_kv_heads, head_dim, max_ctx;
    int chunk;           // cached positions per CTA (<= 0: the default)
    int nsplit_max;      // filled by the launcher
    float *ws;           // split records: seqs * n * attn_decode_ws_floats(...) are used
    size_t ws_floats;    // capacity of ws
    unsigned *counters;  // zero-initialised split arrival counters (the last split re-arms them): seqs * num_kv_heads are used
    size_t n_counters;   // capacity of counters
    // with a request table (the batched and span steps): row s * n gives sequence s's slot and first position; the other rows of a span
    // name the same slot at consecutive positions (host-checked)
    const int *req;          // device int[seqs * n][4] {token, position, slot, valid} (launch_embedding_batch), 16-byte aligned; valid = 0: the CTA writes nothing
    __half *const *slots;    // device table of slot bases, each [L][2][KVH][max_ctx][head_dim]
    long long k_off, v_off;  // elements from a slot's base to this layer's K / V slab
    // without one (req == nullptr, seqs 1): the cache and first position of the one sequence
    __half *k_cache;     // [KVH][max_ctx][head_dim]
    __half *v_cache;     // [KVH][max_ctx][head_dim]
    const int *pos;      // device scalar: the position of row 0 (= number of cached tokens); nullptr: pos0
    int pos0;            // host value of the position of row 0 when pos is nullptr
};
// returns cudaErrorNotSupported for a head_dim or a query-heads-per-KV-head ratio the kernel does not cover, cudaErrorInvalidValue for n outside
// 1..kMaxSpan or a workspace too small, cudaErrorInvalidConfiguration when the CTA of the chunk does not fit shared memory
cudaError_t launch_attn_decode(Ctx *ctx, const AttnDecodeArgs &a, int seqs, int n, bool pdl);
// floats of split workspace the kernel needs per row
size_t attn_decode_ws_floats(int num_heads, int max_ctx, int chunk);
// the largest multiple of 16 rows <= chunk (<= 0: the default) whose CTA, at n = kMaxSpan, fits smem_optin bytes of shared memory; 0 when
// none does.  At 8 query heads per KV head the 256-row default does not fit an H100's 227 KiB: the span runs 224-row splits.
int attn_span_chunk(int num_heads, int num_kv_heads, int chunk, int smem_optin);

// prompt processing (sqlen = n > 1): RoPE + KV append for rows pos0..pos0+n-1, causal attention over the cache.  Up to
// kMaxPrefillSeqs prompts in one launch: their rows are concatenated, and each has its own positions and KV cache.
constexpr int kMaxPrefillSeqs = 8;
struct AttnPrefillSeq {
    int row0, n, pos0;   // rows row0..row0+n-1 of qkv / out are positions pos0..pos0+n-1 of this sequence
    __half *k_cache;     // [KVH][max_ctx][head_dim]
    __half *v_cache;
};
struct AttnPrefillArgs {
    __half *qkv;         // [rows][(H + 2*KVH) * head_dim]; q is rotated in place
    const float *cos, *sin;
    __half *out;         // [rows][H * head_dim]
    float alpha;
    int num_heads, num_kv_heads, head_dim, max_ctx;
    int n_seqs;          // 1..kMaxPrefillSeqs; seq[s + 1].row0 == seq[s].row0 + seq[s].n, seq[0].row0 == 0
    AttnPrefillSeq seq[kMaxPrefillSeqs];
};
cudaError_t launch_attn_prefill(Ctx *ctx, const AttnPrefillArgs &a);
// KV-cache row copy (kv_copy.cu): rows src_pos..src_pos+n-1 of every (layer, K|V, head) slab of slot `src` to rows dst_pos[i].. of the same
// slab of slot dst[i], for every destination.  K rows are rotated by d = dst_pos[i] - src_pos (rotate-half RoPE with cos[|d|] and
// sign(d) * sin[|d|], fp32 without contraction, then round to fp16); V rows and K rows with d = 0 are byte copies.  head_dim 128, host-checked
// arguments: the destinations do not overlap each other, and a destination overlaps the source only when it is the only one (in_place).
constexpr int kMaxKvCopyDst = 8;
struct KvCopyArgs {
    const __half *src;              // slot base, [L][2][KVH][max_ctx][128]
    __half *dst[kMaxKvCopyDst];     // slot bases
    int dst_pos[kMaxKvCopyDst];
    int n_dst, src_pos, n;
    int num_kv_heads, max_ctx;
    const float *cos, *sin;         // [max_ctx][128]
    int in_place;                   // the one destination overlaps the source in its slot: memmove order, one CTA per slab
    int reverse;                    // with in_place: the rows move up (d > 0), so the tiles run from the last one down
};
// n_slabs = L * 2 * KVH; n = 0 launches nothing
cudaError_t launch_kv_copy(Ctx *ctx, const KvCopyArgs &a, int n_slabs);
cudaError_t launch_embedding_rows(Ctx *ctx, const __half *table, const int *tokens, float *resid, int n, int E);
cudaError_t launch_rmsnorm_rows_f32(Ctx *ctx, const float *x, const float *gamma, __half *y, int rows, int dim, float eps);

// decode step prologue (reference: CPU Embedding + float2half, cuda/Int4llamaDecoder.cu:62-69): resid[b][E] = table[token_b] for req = device int[batch][3] {token, position, slot}.  Every entry is
// range-checked (token < rows, position < max_ctx, slot < n_slots) and published as safe[b] = {token, position, slot, valid}; a refused
// entry (valid = 0) embeds row 0 and the attention kernels skip it, so it writes no KV row in any slot
cudaError_t launch_embedding_batch(Ctx *ctx, const __half *table, const int *req, float *resid, int E, int batch, int rows, int max_ctx, int n_slots,
                                   int *safe, bool pdl);
// out[b] = argmax over logits[b][0..n) for b < rows (first index of the maximum, like arg_max.cc; 0 when no value exceeds -inf)
cudaError_t launch_argmax_rows(Ctx *ctx, const float *logits, int rows, int n, int *out, bool pdl);

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
    int out_limit = 0;        // > 0: also stop once *out_count reaches it
    int pos_limit = 0;        // > 0: also stop when the next position reaches it; on stopping, tokpos[1] is set to pos_limit
    int *dbg_ids = nullptr;   // optional: surviving candidates (sorted) and their final probabilities
    float *dbg_probs = nullptr;
    int *dbg_size = nullptr;
};
// the sampler arguments of one chain: the fields of tce_sampling, draw index 0, no history, outputs or limits
SampleArgs sample_args(const tce_sampling &sc, float *logits, int n_vocab);
// temp > 0 over a vocabulary of more than 1024 ids needs 1 <= top_k <= 1024
bool sampling_supported(float temp, int top_k, int n_vocab);
// one row (tce_sample, the single-sequence generate loop); rows_dev = device SampleArgs[rows]: row b is sampled by block b (the batched
// generate loop).  Host-checked arguments, including sampling_supported.
cudaError_t launch_sample(const SampleArgs &a, cudaStream_t stream);
cudaError_t launch_sample_rows(const SampleArgs *rows_dev, int rows, cudaStream_t stream);
// acceptance of a speculative step (sampling.cu, the rule of tce_spec_accept): rows = 1 + drafts logits rows at pitch ld, verified in one
// launch (a block per row)
constexpr int kMaxDrafts = 7;
struct AcceptArgs {
    SampleArgs chain;          // the chain (any temp); logits = row 0; hist / hist_head / hist_cap = the history ring; row j draws with
                               // index draw_index + *hist_head + j
    size_t ld;                 // floats between logits rows
    int rows;                  // 1 + number of drafts
    int drafts[kMaxDrafts];    // draft j is verified by row j
    int eos_id, budget;        // stop id (-1: none); ids the step may emit (>= 1)
    int *repl;                 // device int[kMaxDrafts + 1] scratch: r_j
    float *q;                  // device float[kMaxDrafts + 1]: q_j, the probability of draft j under row j's chain (0 for the last row)
    unsigned *arrive;          // device counter, zero between launches
    int *result;               // device int[3 + kMaxDrafts + 1]: {emitted, stop (eos emitted), drafts among them, ids...}
};
// cudaErrorNotSupported where sampling_supported refuses the chain
cudaError_t launch_accept(const AcceptArgs &a, cudaStream_t stream);
// standalone RMSNorm fp16 -> fp16 with fp32 gamma (reference LlamaRMSNorm_cuda, ops/cuda/LlamaRMSNorm.cu:68-115)
cudaError_t launch_rmsnorm_f16(Ctx *ctx, const __half *x, const float *gamma, __half *y, int rows, int dim, float eps);
// LayerNormQ::forward (llm/src/ops/LayerNormQ.cc:12-52), bit-exact (serial fp32 sums in the reference's order)
cudaError_t launch_layernorm_q(Ctx *ctx, const float *x, const float *weight, const float *bias, int8_t *out, int rows, int dim);
cudaError_t launch_add_f32(Ctx *ctx, const float *a, const float *b, float *out, long long n);

}  // namespace tce
