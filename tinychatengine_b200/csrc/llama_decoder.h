// llama_decoder.h -- host-side runner of the fused Llama decode step (one CUDA graph per token).
#pragma once
#include <string>
#include <vector>

#include "../../include/tce_b200.h"
#include "kernels.h"
#include "kernels_attn.h"
#include "kernels_tp.h"
#include "persistent.h"

namespace tce {

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
    const float *logits() const { return d_logits_; }
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
    // generate loop of up to TCE_LLAMA_MAX_BATCH sequences: one batched step + one sampler launch (a block per row) per token
    cudaError_t generate_batch(int batch, const tce_gen_request *reqs, int *out_tokens_host, int out_stride, int *n_out, std::string *err);
    int kernels_per_step() const { return kernels_per_step_; }
    void *debug_buffer(int which) const {
        switch (which) {
            case 0: return d_resid_;
            case 1: return d_qkv_;
            case 2: return d_attn_;
            case 3: return d_act_;
            case 4: return pargs_.dbg;  // persistent-kernel phase timestamps (TCE_PK_DEBUG=1), [#CTAs][5 * layers + 1][4] u64 ns
            default: return nullptr;
        }
    }
    cudaError_t enqueue_gemvs(int *count);
    cudaError_t tp_handle(void *out64);
    cudaError_t tp_connect(const void *handles);
    void adopt(void *device_allocation) { pk_allocs_.push_back(device_allocation); }  // freed with the model (loader.cu)

   private:
    LlamaDecoder() = default;
    cudaError_t prefill_reserve(int n);
    cudaError_t prefill_linear(int j, const __half *x, void *C, long long ldc, int n, EpiMode epi);
    // the checks of a batch of prompts (prefill_batch, score_batch): cudaErrorInvalidValue, or the total row count in *n
    cudaError_t check_prompts(int n_seqs, const int *tokens_host, const int *lengths, const int *pos0s, const int *slots, int *n) const;
    // the prompt pass over n_seqs concatenated prompts (host-checked arguments); leaves the final residual rows in pf_x_.  With score, the
    // expansion of the first lm_head chunk is queued behind the last down_proj GEMM.
    cudaError_t prefill_rows(int n_seqs, const int *tokens_host, const int *lengths, const int *pos0s, const int *slots, bool score = false);
    cudaError_t enqueue_step(const int *tokpos, cudaStream_t s, bool pdl, bool gemv_only = false);  // raw kernel sequence
    cudaError_t build_graphs(std::string *err);
    void build_ops();
    cudaError_t build_persistent(std::string *err);
    cudaError_t batch_alloc(std::string *err);  // cudaErrorNotSupported (+ *err) for a model the batched step does not cover
    cudaError_t enqueue_batch(int batch, const int *req, cudaStream_t s, bool pdl);  // raw kernel sequence of one batched step
    void drop_batch_graphs();

    enum OpType { OP_EMBED, OP_GEMV, OP_ATTN, OP_ARGMAX, OP_TP_SIGNAL, OP_TP_ARGMAX_SCATTER, OP_TP_ARGMAX_FINISH };
    struct StepOp {
        OpType type;
        W4GemvParams g;
        AttnDecodeArgs at;
        TpSignalArgs sig;
        TpArgmaxArgs am;
        TpArgmaxFinishArgs amf;
    };
    // tensor parallel state
    int tp_ = 1;
    bool tp_connected_ = false;
    uint8_t *tp_buf_ = nullptr;          // peer-visible allocation of this rank
    size_t tp_bytes_ = 0, tp_gather_floats_ = 0;
    uint8_t *tp_peer_[kMaxTP] = {};      // every rank's allocation as mapped into this process
    int step_index_ = 0;
    std::vector<StepOp> ops_;
    // persistent decode kernel (default; TCE_PERSISTENT=0 selects one kernel per op inside a CUDA graph)
    bool persistent_ = false;
    pk::Args pargs_{};
    std::vector<void *> pk_allocs_;     // repacked scales|zeros, tensor maps, layer table, counters

    Ctx *ctx_ = nullptr;
    int attn_chunk_ = 128;
    tce_llama_config cfg_{};
    std::vector<tce_llama_layer> layers_;
    tce_llama_weights w_{};
    // device state
    __half *d_kv_ = nullptr;        // [L][2][KVH][max_ctx][hd]
    float *d_resid_ = nullptr;      // fp32 residual stream [E]
    __half *d_qkv_ = nullptr;       // [(H+2KVH)*hd]
    __half *d_attn_ = nullptr;      // [H*hd]
    __half *d_act_ = nullptr;       // [F] SiLU(gate)*up
    float *d_logits_ = nullptr;     // [V]
    int *d_tokpos_ = nullptr;       // {token, pos} staged for the host entry point
    int *d_next_ = nullptr;         // greedy arg-max
    int *d_gen_ = nullptr;          // generate loop: [0] history head, [1] output count, [2] stop flag, then history ring [max_ctx], output list [max_ctx]
    float *d_cos_ = nullptr, *d_sin_ = nullptr;
    bool own_rope_ = false;
    // prompt-processing activations, [pf_cap_] rows each (allocated on first use)
    int pf_cap_ = 0;
    float *pf_x_ = nullptr;         // fp32 residual stream [n][E]
    __half *pf_xn_ = nullptr;       // RMSNorm output [n][E]
    __half *pf_qkv_ = nullptr;      // [n][(H+2KVH)*hd]
    __half *pf_att_ = nullptr;      // [n][H*hd]
    __half *pf_act_ = nullptr;      // [n][F] SiLU(gate) * up
    int *pf_tok_ = nullptr;
    // the int4 -> fp16 expansion of the NEXT linear runs on a side stream into the other half of a double-buffered scratch while the
    // tensor cores work on the current one (the expansion is HBM-bound, the GEMM tensor-bound)
    __half *pf_w16_[2] = {nullptr, nullptr};
    size_t pf_w16_elems_ = 0;
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
    // scoring buffers, [sc_cap_] rows each (allocated on first use): one chunk's records, the running state across chunks, the targets and
    // their logits, the outputs {logprob, greedy id, greedy logprob}
    int sc_cap_ = 0;
    LmStat *sc_rec_ = nullptr;      // [n][pf_lm_chunk_ / 128]
    LmStat *sc_state_ = nullptr;    // [n]
    int *sc_target_ = nullptr;      // [n]
    float *sc_tgt_ = nullptr;       // [n]
    float *sc_out_ = nullptr;       // [3][n]
    cudaError_t score_reserve(int n);
    // pinned host staging for the end-to-end entry point
    int *h_tokpos_ = nullptr;
    float *h_logits_ = nullptr;
    int *h_next_ = nullptr;
    // graphs
    cudaStream_t cap_stream_ = nullptr;
    cudaGraphExec_t g_host_ = nullptr;    // H2D(tokpos) + step + argmax + D2H(logits,next)
    cudaGraphExec_t g_dev_ = nullptr;     // copy tokpos (D2D) + step
    const int *g_dev_src_ = nullptr;
    bool graphs_ok_ = false;
    unsigned graphs_gen_ = 0, g_dev_gen_ = 0;       // ctx_->option_gen at capture time
    int *d_tokpos_safe_ = nullptr;  // kernel-per-op path: {token, position} after the device-side range check (+ [2] unused, [3] TP step counter alias)
    // batched decode state (allocated on first use): the step's buffers hold TCE_LLAMA_MAX_BATCH rows each
    std::vector<__half *> slot_kv_;    // KV-cache slots 1.. ([L][2][KVH][max_ctx][hd] each)
    __half **d_slot_table_ = nullptr;  // device table of every slot's base, slot 0 = d_kv_
    float *d_bresid_ = nullptr;        // [8][E]
    __half *d_bqkv_ = nullptr;         // [8][(H+2KVH)*hd]
    __half *d_battn_ = nullptr;        // [8][H*hd]
    __half *d_bact_ = nullptr;         // [8][F]
    float *d_blogits_ = nullptr;       // [8][V]
    int *d_breq_ = nullptr;            // [8][3] {token, position, slot} staged for the host entry point
    int *d_bsafe_ = nullptr;           // [8][4] {token, position, slot, valid} after the device-side range check
    int *d_bnext_ = nullptr;           // [8] greedy arg-max
    float *d_battn_ws_ = nullptr;      // attention split records of 8 sequences at this model's max_ctx
    size_t battn_ws_floats_ = 0;
    unsigned *d_battn_counters_ = nullptr;  // [8][KVH] split arrival counters
    size_t battn_counters_ = 0;
    int *h_breq_ = nullptr, *h_bnext_ = nullptr;
    float *h_blogits_ = nullptr;
    // batched generate loop: [8][4] control words {history head, output count, stop flag, unused}, then [8][max_ctx] history rings and
    // [8][max_ctx] output lists; the sampler arguments of each row
    int *d_bgen_ = nullptr;
    SampleArgs *d_bsample_ = nullptr;
    // one graph per batch size: host entry (with / without the logits copy) and device entry (for one request pointer)
    cudaGraphExec_t g_bhost_[2][TCE_LLAMA_MAX_BATCH + 1] = {};
    unsigned g_bhost_gen_[2][TCE_LLAMA_MAX_BATCH + 1] = {};
    cudaGraphExec_t g_bdev_[TCE_LLAMA_MAX_BATCH + 1] = {};
    const int *g_bdev_src_[TCE_LLAMA_MAX_BATCH + 1] = {};
    unsigned g_bdev_gen_[TCE_LLAMA_MAX_BATCH + 1] = {};
    cudaGraphExec_t g_bgen_[TCE_LLAMA_MAX_BATCH + 1] = {};  // generate loop: one batched step on d_breq_ + the row sampler
    unsigned g_bgen_gen_[TCE_LLAMA_MAX_BATCH + 1] = {};
    bool use_graphs_ = true;
    bool atomic_residual_ = true;  // o_proj/down_proj partial tiles use RED.ADD (TCE_DETERMINISTIC=1 turns it off)
    int kernels_per_step_ = 0;
};

// loader.cu: the reference's on-disk INT4 tree -> a model that owns its device copies
LlamaDecoder *load_llama_dir(Ctx *ctx, int attn_chunk, const char *dir, tce_llama_config cfg, std::string *err);
int import_x86(const uint8_t *qs, const float *scales_f32, int oc, int ic, uint32_t *w_out, __half *scales_out, uint32_t *zeros_out);

}  // namespace tce
