// llama_decoder.h -- host-side runner of the fused Llama decode step (one CUDA graph per token).
#pragma once
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <tuple>
#include <vector>

#include "../../include/tce_b200.h"
#include "kernels.h"
#include "kernels_attn.h"
#include "persistent.h"

namespace tce {

// owners of cudaMalloc / cudaMallocHost memory; the allocation helpers leave the owner empty when the call fails
struct CudaFree {
    void operator()(void *p) const { cudaFree(p); }
};
struct CudaFreeHost {
    void operator()(void *p) const { cudaFreeHost(p); }
};
template <typename T> using DevPtr = std::unique_ptr<T, CudaFree>;
template <typename T> using HostPtr = std::unique_ptr<T, CudaFreeHost>;
template <typename T> cudaError_t dev_alloc(DevPtr<T> &p, size_t count) {
    T *q = nullptr;
    const cudaError_t e = cudaMalloc((void **)&q, count * sizeof(T));
    p.reset(e == cudaSuccess ? q : nullptr);
    return e;
}
template <typename T> cudaError_t host_alloc(HostPtr<T> &p, size_t count) {
    T *q = nullptr;
    const cudaError_t e = cudaMallocHost((void **)&q, count * sizeof(T));
    p.reset(e == cudaSuccess ? q : nullptr);
    return e;
}

// an executable graph and what it was captured for: the pointer it reads its request from and the context's option generation
struct CachedGraph {
    cudaGraphExec_t exec = nullptr;
    const void *key = nullptr;
    unsigned gen = 0;
    CachedGraph() = default;
    CachedGraph(const CachedGraph &) = delete;
    CachedGraph &operator=(const CachedGraph &) = delete;
    ~CachedGraph() { reset(); }
    void reset() {
        if (exec) cudaGraphExecDestroy(exec);
        exec = nullptr;
    }
};

// the request and read-back buffers of a decode step of up to `rows` rows
struct StepIO {
    int V = 0;
    HostPtr<int> h_req;       // [rows][3] {token, position, slot} staged for the host entry points
    DevPtr<int> req;          // [rows][3]
    DevPtr<float> logits;     // [rows][V]
    DevPtr<int> next;         // [rows] greedy arg-max
    HostPtr<float> h_logits;  // [rows][V]
    HostPtr<int> h_next;      // [rows]
    cudaError_t alloc(int rows, int V);  // zeroed requests and logits
    void stage(int slot, int pos0, int n, const int *tokens);  // h_req rows 0..n-1 = {tokens[i], pos0 + i, slot}
    // what a host round trip copies back: nothing, the greedy ids, or the logits and then the ids
    enum ReadBack { kNone, kIds, kLogitsIds };
    static ReadBack wanted(const float *logits_host) { return logits_host ? kLogitsIds : kIds; }
    // D2H of the first n rows' logits and / or greedy ids
    cudaError_t read_back(int n, ReadBack r, cudaStream_t s);
    // synchronise s, then copy the read-back out (either pointer may be null)
    cudaError_t copy_out(int n, float *logits_host, int *next_host, cudaStream_t s) const;
};

class LlamaDecoder {
   public:
    static LlamaDecoder *create(Ctx *ctx, int attn_chunk, const tce_llama_config &cfg, const tce_llama_weights &w, std::string *err);
    ~LlamaDecoder();
    cudaError_t decode_device(const int *tokpos_dev, std::string *err);
    cudaError_t decode_host(int token, int pos, float *logits_host, int *next_token, std::string *err);
    cudaError_t generate(int first_token, int pos0, int n_predict, const tce_sampling &sc, const int *history_host, int n_history, int eos_id,
                         int *out_tokens_host, int *n_out, std::string *err);
    // prompt processing: n tokens at positions pos0..pos0+n-1 in one pass (tensor-core GEMMs + causal flash attention)
    cudaError_t prefill(const int *tokens_host, int n, int pos0, float *logits_host, int *next_token, std::string *err, int slot = 0);
    // n_seqs prompts (concatenated in tokens_host) into their own slots in one pass over the weights; logits / greedy token of each last row
    cudaError_t prefill_batch(int n_seqs, const int *tokens_host, const int *lengths, const int *pos0s, const int *slots, float *logits_host,
                              int *next_tokens, std::string *err);
    // teacher-forced scoring: the prompt pass of prefill_batch plus the lm_head over every row, reduced to log-probabilities in the GEMM
    // epilogue (tce_llama_score_batch)
    cudaError_t score_batch(int n_seqs, const int *tokens_host, const int *lengths, const int *pos0s, const int *slots, const int *targets_host,
                            float *logprobs_host, int *greedy_host, float *greedy_logprobs_host, float *logits_dev, std::string *err);
    const float *logits() const { return io1_.logits.get(); }
    void *kv_cache(int layer, int which) const { return kv_cache_slot(0, layer, which); }
    // batched decode: up to TCE_LLAMA_MAX_BATCH sequences per step, each in its own KV-cache slot (slot 0 = d_kv_)
    bool tensor_parallel() const { return tp_ > 1; }
    int n_slots() const { return 1 + (int)slot_kv_.size(); }
    cudaError_t reserve_slots(int n, std::string *err);
    void *kv_cache_slot(int slot, int layer, int which) const;
    cudaError_t decode_batch_device(int batch, const int *req_dev, std::string *err);
    cudaError_t decode_batch_host(int batch, const int *tokens, const int *positions, const int *slots, float *logits_host, int *next_tokens,
                                  std::string *err);
    const float *batch_logits();
    // span step: tokens[0..n) at positions pos0..pos0+n-1 of one slot in one pass (tce_llama_decode_span_host)
    cudaError_t decode_span_host(int slot, int pos0, int n, const int *tokens, float *logits_host, int *next_tokens, std::string *err);
    // speculative loop on slot 0 with prompt-lookup drafts verified by the span step and the acceptance rule of tce_spec_accept
    // (tce_llama_sample_lookup; tce_llama_generate_lookup at temp <= 0)
    cudaError_t generate_lookup(int first_token, int pos0, int n_predict, const tce_sampling &sc, const int *history, int n_history, const int *corpus,
                                int n_corpus, const tce_lookup &lk, int eos_id, int *out_tokens, int *n_out, tce_lookup_stats *stats, std::string *err);
    // generate loop of up to TCE_LLAMA_MAX_BATCH sequences: one batched step + one sampler launch (a block per row) per token
    cudaError_t generate_batch(int batch, const tce_gen_request *reqs, int *out_tokens_host, int out_stride, int *n_out, std::string *err);
    // rows src_pos..src_pos+n-1 of src_slot to rows dst_pos[i].. of dst_slots[i] (every layer, K and V, K re-rotated by the position change):
    // host-checked, then one launch on the context's stream (tce_llama_kv_copy)
    cudaError_t kv_copy(int src_slot, int src_pos, int n, int n_dst, const int *dst_slots, const int *dst_pos, std::string *err);
    int kernels_per_step() const { return persistent_ ? 1 : 1 + 5 * cfg_.num_layers + 2; }
    // 0..3: the batched step's buffers, TCE_LLAMA_MAX_BATCH rows each (null until they exist)
    void *debug_buffer(int which) const {
        switch (which) {
            case 0: return bs_ ? bs_->resid.get() : nullptr;
            case 1: return bs_ ? bs_->qkv.get() : nullptr;
            case 2: return bs_ ? bs_->attn.get() : nullptr;
            case 3: return bs_ ? bs_->act.get() : nullptr;
            case 4: return pargs_.dbg;  // persistent-kernel phase timestamps (TCE_PK_DEBUG=1), [#CTAs][5 * layers + 1][4] u64 ns
            case 5: return pargs_.qkv_ll;  // persistent-kernel hand-off words {payload, tag} (null until it exists): q|k|v, attention
                                           // output, SiLU*up, split partials, o_proj / down_proj outputs, laid out as build_persistent cuts them
            default: return nullptr;
        }
    }
    cudaError_t enqueue_gemvs(int *count);
    cudaError_t tp_handle(void *out64);
    cudaError_t tp_connect(const void *handles, std::string *err);  // cudaErrorNotSupported (+ *err): the persistent kernel refuses the shard
    // a cudaMalloc allocation freed with the model (loader.cu)
    void adopt(void *device_allocation) { pk_allocs_.emplace_back(static_cast<uint8_t *>(device_allocation)); }

   private:
    LlamaDecoder() = default;
    cudaError_t prefill_reserve(int n);
    cudaError_t prefill_linear(int j, const __half *x, void *C, long long ldc, int n, EpiMode epi);
    // slots[0..n) name existing slots, none twice (the batched requests and prompts)
    bool slots_ok(int n, const int *slots) const;
    // the checks of a batch of prompts (prefill, prefill_batch, score_batch): cudaErrorInvalidValue, or the total row count in *n
    cudaError_t check_prompts(int n_seqs, const int *tokens_host, const int *lengths, const int *pos0s, const int *slots, int *n) const;
    // the prompt pass over n_seqs concatenated prompts (host-checked arguments); leaves the final residual rows in pf_.x.  With score, the
    // expansion of the first lm_head chunk is queued behind the last down_proj GEMM.
    cudaError_t prefill_rows(int n_seqs, const int *tokens_host, const int *lengths, const int *pos0s, const int *slots, bool score = false);
    // after prefill_rows: the last row of each prompt through the final RMSNorm + lm_head GEMV into logits[n_seqs][V], greedy ids into next
    cudaError_t prompt_logits(int n_seqs, const int *lengths, float *logits, int *next);
    // the final RMSNorm + lm_head GEMV over rows of x (pitch E) into rows of y (pitch V)
    W4GemvParams lm_head_gemv(const float *x, float *y) const;
    // the decode steps: single = one sequence on slot 0 (the persistent kernel, or the batched step at batch 1), batch = the batched step,
    // span = the batched step over consecutive tokens of one slot
    enum class Step { single, batch, span };
    // the buffers of a kind's step: io1_ for single, bs_->io for the others
    StepIO &io(Step k) { return k == Step::single ? io1_ : bs_->io; }
    // allocates what a kind's step needs (batch_alloc unless it runs on the persistent kernel); cudaErrorNotSupported (+ *err) where it
    // does not run
    cudaError_t step_ready(Step k, std::string *err);
    // one step of `rows` requests at device req, logits and greedy ids into io(k)
    cudaError_t enqueue(Step k, int rows, const int *req, cudaStream_t s, bool pdl);
    // one single-sequence step on device {token, position}: the persistent kernel, or the batched step at batch 1 on slot 0
    cudaError_t enqueue_step(const int *tokpos, cudaStream_t s, bool pdl);
    // runs body(stream, pdl) through the graph cached in g for `key`: replays it when it is current, otherwise runs body eagerly on the
    // context's stream and captures it for the next call (PDL edges first, plain edges if refused); graphs off: eager only
    cudaError_t run_graphed(CachedGraph &g, const void *key, const std::function<cudaError_t(cudaStream_t, bool)> &body);
    // the first half of a host round trip: the `rows` requests staged in io(k).h_req through the host-entry graph {H2D, step, the D2H
    // copies of r}; io(k).copy_out is the second half
    cudaError_t run_host(Step k, int rows, StepIO::ReadBack r);
    cudaError_t build_persistent(std::string *err);
    // the batched step's buffers and parameters; cudaErrorNotSupported (+ *err) for a model the batched step does not cover
    cudaError_t batch_alloc(std::string *err);
    // raw kernel sequence of one batched step on req = device int[batch][3]; lm_head rows into logits[batch][V], greedy ids into next
    // span: the rows are consecutive tokens of one slot (the attention runs them as one sequence of `batch` rows, at the span chunk)
    cudaError_t enqueue_batch(int batch, const int *req, float *logits, int *next, cudaStream_t s, bool pdl, bool span = false);
    // the generate loop of `rows` requests on kind k (single: one request on slot 0), checked before anything is enqueued
    cudaError_t generate_rows(Step k, int rows, const tce_gen_request *reqs, int *out_tokens_host, int out_stride, int *n_out, std::string *err);
    bool span_ok(int slot, int pos0, int n, const int *tokens) const;
    cudaError_t span_supported(std::string *err) const;  // cudaErrorNotSupported (+ *err) when no span split fits shared memory

    // tensor parallel state (the persistent kernel's hand-off buffers)
    int tp_ = 1;
    bool tp_connected_ = false;
    DevPtr<uint8_t> tp_buf_;             // peer-visible allocation of this rank
    size_t tp_bytes_ = 0;
    uint8_t *tp_peer_[kMaxTP] = {};      // every rank's allocation as mapped into this process
    // persistent decode kernel (default; TCE_PERSISTENT=0 selects the batched step at batch 1, one kernel per op inside a CUDA graph)
    bool persistent_ = false;
    pk::Args pargs_{};
    std::vector<DevPtr<uint8_t>> pk_allocs_;  // repacked scales|zeros, tensor maps, layer table, counters; adopted loader copies

    Ctx *ctx_ = nullptr;
    int attn_chunk_ = 128;
    tce_llama_config cfg_{};
    std::vector<tce_llama_layer> layers_;
    tce_llama_weights w_{};
    // device state
    DevPtr<__half> d_kv_;           // [L][2][KVH][max_ctx][hd]
    StepIO io1_;                    // the single-sequence step's request {token, pos, slot = 0}, logits and greedy id
    const float *d_cos_ = nullptr, *d_sin_ = nullptr;  // the caller's RoPE tables, or the halves of rope_
    DevPtr<float> rope_;            // [2][max_ctx][hd] cos | sin, when the caller gives none
    // prompt-processing activations, [cap] rows each (allocated on first use)
    struct PromptBufs {
        int cap = 0;
        DevPtr<float> x;            // fp32 residual stream [n][E]
        DevPtr<__half> xn;          // RMSNorm output [n][E]
        DevPtr<__half> qkv;         // [n][(H+2KVH)*hd]
        DevPtr<__half> att;         // [n][H*hd]
        DevPtr<__half> act;         // [n][F] SiLU(gate) * up
        DevPtr<int> tok;
    } pf_;
    // the int4 -> fp16 expansion of the NEXT linear runs on a side stream into the other half of a double-buffered scratch while the
    // tensor cores work on the current one (the expansion is HBM-bound, the GEMM tensor-bound)
    DevPtr<__half> pf_w16_[2];
    cudaStream_t pf_side_ = nullptr;
    cudaEvent_t pf_expanded_[2] = {nullptr, nullptr}, pf_consumed_[2] = {nullptr, nullptr};
    // one job per linear of the prompt pass, in launch order: job 4 * layer + {0: q|k|v, 1: o, 2: gate|up, 3: down}, then the lm_head in
    // chunks of pf_lm_chunk_ rows (scoring only); job j expands rows r0[i] .. r0[i] + rows[i] - 1 of each of its tensors, stacked
    struct PfJob { const tce_w4_tensor *ts[3]; int count; int r0[3], rows[3]; };
    std::vector<PfJob> pf_jobs_;
    int pf_njobs_ = 0;      // jobs the current pass runs: 4 * layers, or all of them when it scores
    int pf_lm_chunk_ = 0;   // lm_head rows per chunk: whole 256-row blocks that fit one scratch half
    cudaError_t pf_setup();
    cudaError_t pf_expand_job(int j);
    cudaError_t pf_job_begin(int j, const __half **w16);  // queues job j + 1's expansion, then waits for job j's weights
    // scoring buffers, [cap] rows each (allocated on first use): one chunk's records, the running state across chunks, the targets and
    // their logits, the outputs {logprob, greedy id, greedy logprob}
    struct ScoreBufs {
        int cap = 0;
        DevPtr<LmStat> rec;         // [n][pf_lm_chunk_ / 128]
        DevPtr<LmStat> state;       // [n]
        DevPtr<int> target;         // [n]
        DevPtr<float> tgt;          // [n]
        DevPtr<float> out;          // [3][n]
    } sc_;
    cudaError_t score_reserve(int n);
    // graphs: one per (entry, kind, rows, read-back).  The host entry replays run_host's work, the device entry a step on the
    // caller's request pointer (its key), the loop entry a step and the row sampler.  All are dropped when the slot table changes.
    enum Entry { kHost, kDevice, kLoop };
    std::map<std::tuple<Entry, Step, int, StepIO::ReadBack>, CachedGraph> graphs_;
    cudaStream_t cap_stream_ = nullptr;
    // batched decode state (allocated on first use; also the kernel-per-op single-sequence step): the step's buffers hold
    // TCE_LLAMA_MAX_BATCH rows each
    std::vector<DevPtr<__half>> slot_kv_;  // KV-cache slots 1.. ([L][2][KVH][max_ctx][hd] each)
    struct BatchState {
        DevPtr<__half *> slot_table;  // device table of every slot's base, slot 0 = d_kv_
        DevPtr<float> resid;          // [8][E]
        DevPtr<__half> qkv;           // [8][(H+2KVH)*hd]
        DevPtr<__half> attn;          // [8][H*hd]
        DevPtr<__half> act;           // [8][F]
        StepIO io;                    // 8 rows
        DevPtr<int> safe;             // [8][4] {token, position, slot, valid} after the device-side range check
        DevPtr<float> attn_ws;        // attention split records of 8 sequences at this model's max_ctx
        size_t attn_ws_floats = 0;
        int span_chunk = 0;           // cached rows per CTA of the span attention (attn_span_chunk), 0: the span step is not supported
        DevPtr<unsigned> attn_counters;  // [8][KVH] split arrival counters
        size_t n_counters = 0;
        // the step's parameters on these buffers: GEMV 4 * layer + {0: q|k|v, 1: o, 2: gate|up, 3: down} (M = 1), then the lm_head;
        // the attention of each layer (its slot table is read at launch)
        std::vector<W4GemvParams> gemv_ops;
        std::vector<AttnDecodeArgs> attn_ops;
    };
    std::unique_ptr<BatchState> bs_;  // non-null: every buffer of the batched step exists
    // both generate loops (allocated whole on the first call of either, never reallocated: captured graphs hold these pointers): [8][4]
    // control words {history head, output count, stop flag, unused}, then [8][max_ctx] history rings and [8][max_ctx] output lists; the
    // sampler arguments of each row
    struct LoopState {
        DevPtr<int> words;
        DevPtr<SampleArgs> sample;
    };
    std::unique_ptr<LoopState> loop_;
    // speculative loop: device {counter, step result, greedy ids, history ring [max_ctx]} and the pinned read-back of one step's result
    DevPtr<int> d_spec_;
    HostPtr<int> h_spec_;
    bool use_graphs_ = true;
    bool atomic_residual_ = true;  // o_proj/down_proj partial tiles use RED.ADD (TCE_DETERMINISTIC=1 turns it off)
};

// loader.cu: the reference's on-disk INT4 tree -> a model that owns its device copies
LlamaDecoder *load_llama_dir(Ctx *ctx, int attn_chunk, const char *dir, tce_llama_config cfg, std::string *err);
int import_x86(const uint8_t *qs, const float *scales_f32, int oc, int ic, uint32_t *w_out, __half *scales_out, uint32_t *zeros_out);

}  // namespace tce
