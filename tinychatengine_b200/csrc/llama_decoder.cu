// llama_decoder.cu -- one-token decode of an AWQ-INT4 Llama as a single CUDA graph.
//
// Call sites restated (reference, CUDA build): Int4LlamaForCausalLM::forward (cuda/Int4llamaForCausalLM.cu:17-50)
// -> Int4llamaDecoder::forward (cuda/Int4llamaDecoder.cu:57-112) -> 32 x Int4llamaDecoderLayer::forward
// (cuda/Int4llamaDecoderLayer.cu:73-115) -> Int4llamaAttention::forward (cuda/Int4llamaAttention.cu:116-229).
// The reference issues ~19 kernels + 128 memcpys per layer on stream 0; here a layer is 5 kernels
// (RMSNorm+QKV GEMV | RoPE+append+attention | o_proj+residual | RMSNorm+gate/up+SiLU*mul | down+residual),
// chained with programmatic dependent launch so each GEMV prefetches its weights while its predecessor drains.
// The residual stream is kept in fp32 (the reference's CUDA build keeps it in fp16, its CPU build in fp32).
#include "llama_decoder.h"

#include "persistent.h"

#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

namespace tce {

#define DCK(call)                              \
    do {                                       \
        cudaError_t e__ = (call);              \
        if (e__ != cudaSuccess) return e__;    \
    } while (0)

static bool w4_ok(const tce_w4_tensor &t, int oc, int ic) { return t.w && t.zeros && t.scales && t.oc == oc && t.ic == ic; }

LlamaDecoder *LlamaDecoder::create(Ctx *ctx, int attn_chunk, const tce_llama_config &cfg, const tce_llama_weights &w, std::string *err) {
    auto bad = [&](const char *m) {
        *err = m;
        return (LlamaDecoder *)nullptr;
    };
    if (cfg.head_dim != 128) return bad("head_dim must be 128");
    if (cfg.num_layers < 1 || cfg.num_heads < 1 || cfg.num_kv_heads < 1 || cfg.num_heads % cfg.num_kv_heads) return bad("bad head configuration");
    if (cfg.embed_dim % 128 || cfg.hidden_dim % 128) return bad("embed_dim / hidden_dim must be multiples of the 128 group");
    if (cfg.tp_size > kMaxTP || cfg.tp_size < 0 || (cfg.tp_size > 1 && (cfg.tp_rank < 0 || cfg.tp_rank >= cfg.tp_size))) return bad("bad tensor-parallel rank/size");
    const bool persistent = getenv("TCE_PERSISTENT") ? atoi(getenv("TCE_PERSISTENT")) != 0 : true;
    if (cfg.tp_size > 1 && !persistent) return bad("tensor parallelism runs on the persistent decode kernel only (TCE_PERSISTENT=0 turns it off)");
    const int E = cfg.embed_dim, F = cfg.hidden_dim, H = cfg.num_heads, KVH = cfg.num_kv_heads, hd = cfg.head_dim, V = cfg.vocab_size;
    if (!w.embed_f16 || !w.layers || !w.final_norm) return bad("missing weights");
    if (!w4_ok(w.lm_head, V, E) || V % 16) return bad("lm_head shape");
    for (int l = 0; l < cfg.num_layers; l++) {
        const tce_llama_layer &L = w.layers[l];
        if (!w4_ok(L.q, H * hd, E) || !w4_ok(L.k, KVH * hd, E) || !w4_ok(L.v, KVH * hd, E) || !w4_ok(L.o, E, H * hd) || !w4_ok(L.gate, F, E) ||
            !w4_ok(L.up, F, E) || !w4_ok(L.down, E, F) || !L.input_norm || !L.post_norm)
            return bad("layer weight shape");
    }
    LlamaDecoder *d = new LlamaDecoder();
    d->ctx_ = ctx;
    d->attn_chunk_ = attn_chunk;
    d->cfg_ = cfg;
    d->w_ = w;
    d->layers_.assign(w.layers, w.layers + cfg.num_layers);
    d->w_.layers = d->layers_.data();
    d->use_graphs_ = getenv("TCE_NO_GRAPH") == nullptr;
    d->atomic_residual_ = getenv("TCE_DETERMINISTIC") == nullptr;
    const size_t kv_elems = (size_t)cfg.num_layers * 2 * KVH * cfg.max_ctx * hd;
    cudaError_t e = cudaSuccess;
    auto A = [&](auto &p, size_t count) {
        if (e == cudaSuccess) e = dev_alloc(p, count);
    };
    A(d->d_kv_, kv_elems);
    if (e == cudaSuccess) e = cudaMemset(d->d_kv_.get(), 0, kv_elems * sizeof(__half));
    if (e == cudaSuccess) e = d->io1_.alloc(1, V);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&d->cap_stream_, cudaStreamNonBlocking);
    if (e == cudaSuccess) {
        if (w.rope_cos && w.rope_sin) {
            d->d_cos_ = w.rope_cos;
            d->d_sin_ = w.rope_sin;
        } else {
            // HF rotate-half tables: cos/sin(pos * theta^(-2i/hd)) duplicated over both halves
            std::vector<float> hc((size_t)cfg.max_ctx * hd), hs((size_t)cfg.max_ctx * hd);
            const double theta = cfg.rope_theta > 0 ? cfg.rope_theta : 10000.0;
            for (int p = 0; p < cfg.max_ctx; p++)
                for (int i = 0; i < hd / 2; i++) {
                    const double inv = 1.0 / pow(theta, (2.0 * i) / hd);
                    const double ang = p * inv;
                    hc[(size_t)p * hd + i] = hc[(size_t)p * hd + i + hd / 2] = (float)cos(ang);
                    hs[(size_t)p * hd + i] = hs[(size_t)p * hd + i + hd / 2] = (float)sin(ang);
                }
            A(d->rope_, 2 * hc.size());
            if (e == cudaSuccess) e = cudaMemcpy(d->rope_.get(), hc.data(), hc.size() * sizeof(float), cudaMemcpyHostToDevice);
            if (e == cudaSuccess) e = cudaMemcpy(d->rope_.get() + hc.size(), hs.data(), hs.size() * sizeof(float), cudaMemcpyHostToDevice);
            d->d_cos_ = d->rope_.get();
            d->d_sin_ = d->rope_.get() + hc.size();
        }
    }
    if (e != cudaSuccess) {
        *err = std::string("allocation failed: ") + cudaGetErrorString(e);
        delete d;
        return nullptr;
    }
    d->persistent_ = persistent;
    d->tp_ = cfg.tp_size > 1 ? cfg.tp_size : 1;
    if (d->tp_ > 1) {
        // tensor parallel: one peer-visible allocation of two delta buffers of P x E {float, tag} words + P x 2 key words
        d->tp_bytes_ = ((size_t)2 * d->tp_ * E + (size_t)2 * d->tp_) * sizeof(uint2);
        if (dev_alloc(d->tp_buf_, d->tp_bytes_) != cudaSuccess || cudaMemset(d->tp_buf_.get(), 0, d->tp_bytes_) != cudaSuccess) {
            *err = "tensor-parallel buffer allocation failed";
            delete d;
            return nullptr;
        }
        cudaDeviceSynchronize();
        return d;  // the persistent kernel needs the peers' pointers: set up in tp_connect()
    }
    if (d->persistent_) {
        std::string why;
        cudaError_t me = d->build_persistent(&why);
        if (me == cudaErrorNotSupported) {
            d->persistent_ = false;  // shape outside the persistent kernel's envelope: one kernel per op
        } else if (me != cudaSuccess) {
            *err = std::string("persistent kernel setup failed: ") + why + " " + cudaGetErrorString(me);
            delete d;
            return nullptr;
        }
    }
    return d;
}

LlamaDecoder::~LlamaDecoder() {
    if (cap_stream_) cudaStreamDestroy(cap_stream_);
    for (int b = 0; b < 2; b++) {
        if (pf_expanded_[b]) cudaEventDestroy(pf_expanded_[b]);
        if (pf_consumed_[b]) cudaEventDestroy(pf_consumed_[b]);
    }
    if (pf_side_) cudaStreamDestroy(pf_side_);
    for (int p = 0; p < tp_; p++)
        if (p != cfg_.tp_rank && tp_peer_[p]) cudaIpcCloseMemHandle(tp_peer_[p]);
}

void *LlamaDecoder::kv_cache_slot(int slot, int layer, int which) const {
    if (slot < 0 || slot >= n_slots() || layer < 0 || layer >= cfg_.num_layers || which < 0 || which > 1) return nullptr;
    const size_t per = (size_t)cfg_.num_kv_heads * cfg_.max_ctx * cfg_.head_dim;
    return (slot == 0 ? d_kv_ : slot_kv_[slot - 1]).get() + ((size_t)layer * 2 + which) * per;
}

static W4Seg seg_of(const tce_w4_tensor &t) { return W4Seg{(const uint32_t *)t.w, (const uint32_t *)t.zeros, (const __half *)t.scales, t.oc}; }

cudaError_t LlamaDecoder::enqueue_gemvs(int *count) {
    DCK(batch_alloc(nullptr));
    for (const W4GemvParams &p : bs_->gemv_ops) DCK(launch_w4a16_gemv(ctx_, p));
    *count = (int)bs_->gemv_ops.size();
    return cudaSuccess;
}

cudaError_t LlamaDecoder::tp_handle(void *out64) {
    if (tp_ <= 1 || !tp_buf_) return cudaErrorInvalidValue;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
    return cudaIpcGetMemHandle(reinterpret_cast<cudaIpcMemHandle_t *>(out64), tp_buf_.get());
}

cudaError_t LlamaDecoder::tp_connect(const void *handles, std::string *err) {
    if (tp_ <= 1) return cudaErrorInvalidValue;
    const cudaIpcMemHandle_t *h = reinterpret_cast<const cudaIpcMemHandle_t *>(handles);
    for (int p = 0; p < tp_; p++) {
        if (p == cfg_.tp_rank) {
            tp_peer_[p] = tp_buf_.get();
        } else {
            DCK(cudaIpcOpenMemHandle((void **)&tp_peer_[p], h[p], cudaIpcMemLazyEnablePeerAccess));
        }
    }
    DCK(build_persistent(err));
    tp_connected_ = true;
    return cudaSuccess;
}

// Everything the persistent decode kernel (decode_persistent.cu) needs beyond the caller's weights: one 3-D tensor map per packed
// matrix (the [group][row][64 B] view, see pk::GemvOp), the per-stage scales|zeros records (a one-off repack of the QM_CUDA scales /
// zeros arrays into the order the TMA ring consumes them: SURVEY.md 8(f)2 "repack once into the TMA-friendly interleave"), the layer
// table and the tagged hand-off buffers.
cudaError_t LlamaDecoder::build_persistent(std::string *err) {
    const int E = cfg_.embed_dim, F = cfg_.hidden_dim, H = cfg_.num_heads, KVH = cfg_.num_kv_heads, hd = cfg_.head_dim, V = cfg_.vocab_size;
    const int Lyr = cfg_.num_layers, ncta = ctx_->num_sms;
    const int nrep = H / KVH;
    auto no = [&](const char *m) {
        if (err) *err = m;
        return cudaErrorNotSupported;
    };
    // 32-row tiles (pk::kTileRows; gate | up: 16 channels): with hd = 128 the q|k|v segment boundaries fall on tile boundaries
    if (hd != 128 || nrep > 4 || ncta < KVH || F % pk::kTileRows || V % pk::kTileRows) return no("shape outside the persistent kernel's envelope");
    // clusters of two CTAs split K (see pk::KRange): an even number of SMs, and two 128-groups or more in every op
    if (ncta % 2) return no("odd SM count: the persistent kernel runs on clusters of two CTAs");
    pk::Args a{};
    auto mk = [&](int IC, int rows, int nseg, int gate_up, int rows0, int rows1, int x_mode, int epi) {
        pk::GemvOp o{};
        o.IC = IC;
        o.NG = IC / kW4Group;
        o.num_tiles = rows / pk::kTileRows;
        o.nseg = nseg;
        o.gate_up = gate_up;
        o.rows0 = rows0;
        o.rows1 = rows1;
        o.x_mode = x_mode;
        o.epi = epi;
        return o;
    };
    const bool tp = tp_ > 1;
    a.op[pk::OPI_QKV] = mk(E, (H + 2 * KVH) * hd, 3, 0, H * hd, KVH * hd, pk::PX_RMS_F32, pk::PE_HALF_LL);
    a.op[pk::OPI_O] = mk(H * hd, E, 1, 0, E, 0, pk::PX_HALF, pk::PE_DELTA_LL);
    a.op[pk::OPI_GATEUP] = mk(E, 2 * F, 2, 1, F, F, pk::PX_RMS_F32, pk::PE_SILU_LL);
    a.op[pk::OPI_DOWN] = mk(F, E, 1, 0, E, 0, pk::PX_HALF, pk::PE_DELTA_LL);
    a.op[pk::OPI_LMHEAD] = mk(E, V, 1, 0, V, 0, pk::PX_RMS_F32, pk::PE_LOGITS);
    int max_ng = 0, min_ng = 1 << 30;
    for (int i = 0; i < pk::OPI_COUNT; i++) {
        if (a.op[i].NG > max_ng) max_ng = a.op[i].NG;
        if (a.op[i].NG < min_ng) min_ng = a.op[i].NG;
        if (a.op[i].IC % kW4Group || a.op[i].num_tiles < 1) return no("bad GEMV shape");
    }
    if (min_ng < 2) return no("a GEMV with a single 128-group: nothing to split across a cluster of two CTAs");
    a.max_ng = (max_ng + 3) & ~3;
    a.E = E;
    a.nrep = nrep;
    pk::plan_smem(a, ctx_->smem_optin);
    if (a.nst < 2) return no("shared memory too small for the persistent kernel");
    if (!pk::pair_supported(ctx_, a)) return no("the device cannot co-schedule num_sms / 2 clusters of two CTAs");

    auto dalloc = [&](size_t bytes) -> void * {
        DevPtr<uint8_t> p;
        if (dev_alloc(p, bytes ? bytes : 16) != cudaSuccess) return nullptr;
        pk_allocs_.push_back(std::move(p));
        return pk_allocs_.back().get();
    };
    cudaStream_t s = ctx_->stream;
    // ---- tensor maps: per cluster rank [Lyr][7] + lm_head, then the KV cache ----
    const size_t nmaps = (size_t)Lyr * 7 + 1;
    std::vector<CUtensorMap> maps(2 * nmaps + 1);
    memset(maps.data(), 0, maps.size() * sizeof(CUtensorMap));
    std::vector<pk::LayerDesc> descs(Lyr);
    const size_t per_kv = (size_t)KVH * cfg_.max_ctx;  // rows per (layer, K|V) slab
    for (int l = 0; l < Lyr; l++) {
        const tce_llama_layer &L = layers_[l];
        const tce_w4_tensor *t7[7] = {&L.q, &L.k, &L.v, &L.o, &L.gate, &L.up, &L.down};
        const int opi[7] = {pk::OPI_QKV, pk::OPI_QKV, pk::OPI_QKV, pk::OPI_O, pk::OPI_GATEUP, pk::OPI_GATEUP, pk::OPI_DOWN};
        for (int rank = 0; rank < 2; rank++) {
            for (int i = 0; i < 7; i++) {
                const pk::GemvOp &o = a.op[opi[i]];
                const pk::KRange kr = pk::k_range(o.NG, rank);
                const int box_rows = o.gate_up ? pk::kTileRows / 2 : pk::kTileRows;  // gate | up: a box of each matrix per stage
                DCK(encode_w4_tmap_units(&maps[rank * nmaps + (size_t)l * 7 + i], t7[i]->w, t7[i]->oc, t7[i]->ic, kr.bw, box_rows, kr.g0, kr.ng));
            }
        }
        pk::LayerDesc &D = descs[l];
        memset(&D, 0, sizeof(D));
        const W4Seg qkv[3] = {seg_of(L.q), seg_of(L.k), seg_of(L.v)}, o1[1] = {seg_of(L.o)}, gu[2] = {seg_of(L.gate), seg_of(L.up)}, d1[1] = {seg_of(L.down)};
        const W4Seg *segs[4] = {qkv, o1, gu, d1};
        const int nsegs[4] = {3, 1, 2, 1};
        const int ops4[4] = {pk::OPI_QKV, pk::OPI_O, pk::OPI_GATEUP, pk::OPI_DOWN};
        for (int rank = 0; rank < 2; rank++) {
            for (int i = 0; i < 4; i++) {
                const pk::GemvOp &o = a.op[ops4[i]];
                const pk::KRange kr = pk::k_range(o.NG, rank);
                uint8_t *m = (uint8_t *)dalloc((size_t)o.num_tiles * kr.nb * pk::kBoxMetaBytes);
                if (!m) return cudaErrorMemoryAllocation;
                DCK(pk::repack_meta(ctx_, segs[i], nsegs[i], o.gate_up, o.IC, kr, m, s));
                D.meta[rank][i] = m;
            }
        }
        D.input_norm = L.input_norm;
        D.post_norm = L.post_norm;
        D.k_cache = (__half *)kv_cache(l, 0);
        D.v_cache = (__half *)kv_cache(l, 1);
        D.k_row0 = (int)(((size_t)l * 2 + 0) * per_kv);
        D.v_row0 = (int)(((size_t)l * 2 + 1) * per_kv);
    }
    {
        const pk::GemvOp &o = a.op[pk::OPI_LMHEAD];
        const W4Seg lm[1] = {seg_of(w_.lm_head)};
        for (int rank = 0; rank < 2; rank++) {
            const pk::KRange kr = pk::k_range(o.NG, rank);
            DCK(encode_w4_tmap_units(&maps[rank * nmaps + (size_t)Lyr * 7], w_.lm_head.w, w_.lm_head.oc, w_.lm_head.ic, kr.bw, pk::kTileRows, kr.g0, kr.ng));
            uint8_t *m = (uint8_t *)dalloc((size_t)o.num_tiles * kr.nb * pk::kBoxMetaBytes);
            if (!m) return cudaErrorMemoryAllocation;
            DCK(pk::repack_meta(ctx_, lm, 1, 0, o.IC, kr, m, s));
            a.lm_meta[rank] = m;
        }
    }
    DCK(pk::encode_kv_tmap(&maps[2 * nmaps], d_kv_.get(), (long long)Lyr * 2 * per_kv));
    CUtensorMap *dmaps = (CUtensorMap *)dalloc(maps.size() * sizeof(CUtensorMap));
    pk::LayerDesc *ddesc = (pk::LayerDesc *)dalloc(descs.size() * sizeof(pk::LayerDesc));
    a.nsplit_max = pk::attn_nsplit_max(ncta, KVH, cfg_.max_ctx);
    // hand-off buffers ({payload, tag} words; tag 0 = never written)
    const size_t n_qkv = (size_t)(H + 2 * KVH) * 64, n_attn = (size_t)H * 64, n_act = (size_t)F / 2, n_part = (size_t)H * a.nsplit_max * 130;
    const size_t ll_words = n_qkv + n_attn + n_act + n_part + (tp ? 0 : (size_t)2 * E);
    uint2 *ll = (uint2 *)dalloc(ll_words * sizeof(uint2));
    // [arg-max cell u64][epoch u32][error i32][done u32]
    uint8_t *ctl = (uint8_t *)dalloc(32);
    if (!dmaps || !ddesc || !ll || !ctl) return cudaErrorMemoryAllocation;
    DCK(cudaMemcpyAsync(dmaps, maps.data(), maps.size() * sizeof(CUtensorMap), cudaMemcpyHostToDevice, s));
    DCK(cudaMemcpyAsync(ddesc, descs.data(), descs.size() * sizeof(pk::LayerDesc), cudaMemcpyHostToDevice, s));
    DCK(cudaMemsetAsync(ll, 0, ll_words * sizeof(uint2), s));
    DCK(cudaMemsetAsync(ctl, 0, 32, s));
    DCK(cudaStreamSynchronize(s));  // `maps` / `descs` are host temporaries
    a.layers = ddesc;
    a.num_layers = Lyr;
    a.maps = dmaps;
    a.final_norm = w_.final_norm;
    a.embed = (const __half *)w_.embed_f16;
    a.embed_rows = V * tp_;
    a.qkv_ll = ll;
    a.attn_ll = a.qkv_ll + n_qkv;
    a.act_ll = a.attn_ll + n_attn;
    a.part_ll = a.act_ll + n_act;
    a.logits = io1_.logits.get();
    a.tokpos = io1_.req.get();
    a.next_token = io1_.next.get();
    a.argmax_cell = reinterpret_cast<unsigned long long *>(ctl);
    a.epoch = reinterpret_cast<unsigned *>(ctl + 8);
    a.error = reinterpret_cast<int *>(ctl + 12);
    a.done = reinterpret_cast<unsigned *>(ctl + 16);
    a.cos = d_cos_;
    a.sin = d_sin_;
    a.alpha = cfg_.qk_alpha > 0 ? cfg_.qk_alpha : 1.0f / sqrtf((float)hd);
    a.eps = cfg_.rms_eps;
    a.H = H;
    a.KVH = KVH;
    a.max_ctx = cfg_.max_ctx;
    a.V = V;
    a.F = F;
    a.tp_size = tp_;
    a.tp_rank = tp ? cfg_.tp_rank : 0;
    a.vocab_base = tp ? cfg_.tp_rank * V : 0;
    if (tp) {
        // peer-visible allocation of every rank: [delta 0: P x E words][delta 1: P x E words][keys: P x 2 words]
        for (int q = 0; q < tp_; q++) {
            uint2 *base = reinterpret_cast<uint2 *>(tp_peer_[q]);
            a.tp_delta[0][q] = base;
            a.tp_delta[1][q] = base + (size_t)tp_ * E;
            a.tp_keys[q] = base + (size_t)2 * tp_ * E;
        }
        a.delta_ll[0] = a.tp_delta[0][a.tp_rank];
        a.delta_ll[1] = a.tp_delta[1][a.tp_rank];
    } else {
        a.delta_ll[0] = a.part_ll + n_part;
        a.delta_ll[1] = a.delta_ll[0] + E;
    }
    if (getenv("TCE_PK_DEBUG") && atoi(getenv("TCE_PK_DEBUG"))) {
        const size_t n = (size_t)ncta * ((size_t)5 * Lyr + 1) * 8 * sizeof(unsigned long long);
        a.dbg = (unsigned long long *)dalloc(n);
        if (!a.dbg) return cudaErrorMemoryAllocation;
        DCK(cudaMemset(a.dbg, 0, n));
    }
    if ((int)pk::smem_bytes(a) > ctx_->smem_optin) return no("shared memory");
    pargs_ = a;
    return cudaSuccess;
}

cudaError_t StepIO::alloc(int n, int v) {
    V = v;
    DCK(host_alloc(h_req, (size_t)n * 3));
    DCK(dev_alloc(req, (size_t)n * 3));
    DCK(dev_alloc(logits, (size_t)n * v));
    DCK(dev_alloc(next, (size_t)n));
    DCK(host_alloc(h_logits, (size_t)n * v));
    DCK(host_alloc(h_next, (size_t)n));
    DCK(cudaMemset(req.get(), 0, (size_t)n * 3 * sizeof(int)));
    return cudaMemset(logits.get(), 0, (size_t)n * v * sizeof(float));
}

void StepIO::stage(int slot, int pos0, int n, const int *tokens) {
    for (int i = 0; i < n; i++) {
        h_req.get()[3 * i] = tokens[i];
        h_req.get()[3 * i + 1] = pos0 + i;
        h_req.get()[3 * i + 2] = slot;
    }
}

cudaError_t StepIO::read_back(int n, ReadBack r, cudaStream_t s) {
    if (r == kNone) return cudaSuccess;
    if (r == kLogitsIds) DCK(cudaMemcpyAsync(h_logits.get(), logits.get(), (size_t)n * V * sizeof(float), cudaMemcpyDeviceToHost, s));
    return cudaMemcpyAsync(h_next.get(), next.get(), (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, s);
}

cudaError_t StepIO::copy_out(int n, float *logits_host, int *next_host, cudaStream_t s) const {
    DCK(cudaStreamSynchronize(s));
    if (logits_host) memcpy(logits_host, h_logits.get(), (size_t)n * V * sizeof(float));
    if (next_host) memcpy(next_host, h_next.get(), (size_t)n * sizeof(int));
    return cudaSuccess;
}

cudaError_t LlamaDecoder::step_ready(Step k, std::string *err) {
    if (k == Step::single && persistent_) return cudaSuccess;
    DCK(batch_alloc(err));
    return k == Step::span ? span_supported(err) : cudaSuccess;
}

cudaError_t LlamaDecoder::enqueue(Step k, int rows, const int *req, cudaStream_t s, bool pdl) {
    if (k == Step::single) return enqueue_step(req, s, pdl);
    return enqueue_batch(rows, req, bs_->io.logits.get(), bs_->io.next.get(), s, pdl, k == Step::span);
}

cudaError_t LlamaDecoder::enqueue_step(const int *tokpos, cudaStream_t s, bool pdl) {
    if (persistent_) {
        pk::Args m = pargs_;
        m.tokpos = tokpos;
        return pk::launch(ctx_, m, s);
    }
    // the batched embedding reads {token, position, slot}: the caller's pair goes in front of slot 0
    int *req = io1_.req.get();
    if (tokpos != req) DCK(cudaMemcpyAsync(req, tokpos, 2 * sizeof(int), cudaMemcpyDeviceToDevice, s));
    return enqueue_batch(1, req, io1_.logits.get(), io1_.next.get(), s, pdl);
}

cudaError_t LlamaDecoder::run_graphed(CachedGraph &g, const void *key, const std::function<cudaError_t(cudaStream_t, bool)> &body) {
    cudaStream_t s = ctx_->stream;
    if (!use_graphs_) return body(s, ctx_->use_pdl);
    if (g.exec && g.key == key && g.gen == ctx_->option_gen) return cudaGraphLaunch(g.exec, s);
    // a graph holds the context by value: after an option or the stream changed (option_gen) it is rebuilt.  This call runs eagerly, which
    // also loads the modules, sets kernel attributes and grows the GEMV fix-up records outside of capture; capture itself runs nothing.
    g.reset();
    DCK(body(s, ctx_->use_pdl));
    for (int attempt = ctx_->use_pdl ? 0 : 1; attempt < 2; attempt++) {
        const bool pdl = attempt == 0;
        cudaGraph_t graph = nullptr;
        cudaError_t e = cudaStreamBeginCapture(cap_stream_, cudaStreamCaptureModeThreadLocal);
        if (e == cudaSuccess) {
            e = body(cap_stream_, pdl);
            const cudaError_t e2 = cudaStreamEndCapture(cap_stream_, &graph);
            if (e == cudaSuccess) e = e2;
        }
        if (e == cudaSuccess) e = cudaGraphInstantiate(&g.exec, graph, 0);
        if (graph) cudaGraphDestroy(graph);
        if (e == cudaSuccess) {
            if (!pdl) ctx_->use_pdl = false;
            g.key = key;
            g.gen = ctx_->option_gen;  // read after the eager run: growing the fix-up records moves it
            return cudaSuccess;
        }
        cudaGetLastError();
        g.exec = nullptr;
    }
    use_graphs_ = false;  // the work above already ran: carry on without graphs
    return cudaSuccess;
}

cudaError_t LlamaDecoder::run_host(Step k, int rows, StepIO::ReadBack r) {
    StepIO &b = io(k);
    return run_graphed(graphs_[{kHost, k, rows, r}], nullptr, [&](cudaStream_t st, bool pdl) {
        DCK(cudaMemcpyAsync(b.req.get(), b.h_req.get(), (size_t)rows * 3 * sizeof(int), cudaMemcpyHostToDevice, st));
        DCK(enqueue(k, rows, b.req.get(), st, pdl));
        return b.read_back(rows, r, st);
    });
}

cudaError_t LlamaDecoder::decode_host(int token, int pos, float *logits_host, int *next_token, std::string *err) {
    const int tp = cfg_.tp_size > 1 ? cfg_.tp_size : 1;
    if (pos < 0 || pos >= cfg_.max_ctx || token < 0 || token >= cfg_.vocab_size * tp) return cudaErrorInvalidValue;
    if (tp > 1 && !tp_connected_) return cudaErrorNotReady;
    DCK(step_ready(Step::single, err));
    io1_.stage(0, pos, 1, &token);
    DCK(run_host(Step::single, 1, StepIO::wanted(logits_host)));
    return io1_.copy_out(1, logits_host, next_token, ctx_->stream);
}

// Generate loop of one sequence on slot 0: generate_rows on the single-sequence step.
cudaError_t LlamaDecoder::generate(int first_token, int pos0, int n_predict, const tce_sampling &sc, const int *history_host, int n_history, int eos_id,
                                   int *out_tokens_host, int *n_out, std::string *err) {
    if (cfg_.tp_size > 1) {
        if (err) *err = "generate: single GPU only (the vocabulary is sharded under tensor parallelism)";
        return cudaErrorNotSupported;
    }
    const tce_gen_request r{first_token, pos0, 0, n_predict, eos_id, history_host, n_history, sc};
    return generate_rows(Step::single, 1, &r, out_tokens_host, n_predict, n_out, err);
}

cudaError_t LlamaDecoder::decode_device(const int *tokpos_dev, std::string *err) {
    if (tp_ > 1 && !tp_connected_) return cudaErrorNotReady;
    DCK(step_ready(Step::single, err));
    return run_graphed(graphs_[{kDevice, Step::single, 1, StepIO::kNone}], tokpos_dev,
                       [&](cudaStream_t st, bool pdl) { return enqueue_step(tokpos_dev, st, pdl); });
}

}  // namespace tce

// ------------------------------------------------------------------------------------------------ prompt processing
// n tokens at once (sqlen > 1 in the reference's Int4LlamaForCausalLM::forward): every linear runs as one tensor-core GEMM over the
// [n][.] activation block (int4 weights expanded to fp16 once per GEMM), attention as one causal flash kernel over the KV cache.
namespace tce {

cudaError_t LlamaDecoder::prefill_reserve(int n) {
    if (n <= pf_.cap) return cudaSuccess;
    DCK(cudaStreamSynchronize(ctx_->stream));
    pf_ = PromptBufs{};  // the old buffers go first
    const size_t E = cfg_.embed_dim, F = cfg_.hidden_dim, Q = (size_t)(cfg_.num_heads + 2 * cfg_.num_kv_heads) * cfg_.head_dim,
                 A = (size_t)cfg_.num_heads * cfg_.head_dim;
    PromptBufs b;
    DCK(dev_alloc(b.x, n * E));
    DCK(dev_alloc(b.xn, n * E));
    DCK(dev_alloc(b.qkv, n * Q));
    DCK(dev_alloc(b.att, n * A));
    DCK(dev_alloc(b.act, n * F));
    DCK(dev_alloc(b.tok, (size_t)n));
    b.cap = n;
    pf_ = std::move(b);
    return cudaSuccess;
}

// C[n][rows] (row-major, leading dimension ldc) = X[n][ic] * W^T, W = the weights of job j stacked (q|k|v and gate|up share their input),
// expanded to fp16 on the side stream while the previous GEMM ran.  epi: EPI_STORE_HALF, EPI_ADD_F32 (residual add) or EPI_SILU_MUL_HALF
// (job = gate|up, C = SiLU(gate) * up)
cudaError_t LlamaDecoder::prefill_linear(int j, const __half *x, void *C, long long ldc, int n, EpiMode epi) {
    const PfJob &job = pf_jobs_[j];
    const int ic = job.ts[0]->ic;
    size_t rows = 0;
    for (int i = 0; i < job.count; i++) rows += (size_t)job.rows[i];
    const __half *w16 = nullptr;
    DCK(pf_job_begin(j, &w16));
    if (epi == EPI_SILU_MUL_HALF)
        DCK(launch_gemm_f16_pair_silu(ctx_, x, ic, w16, ic, (__half *)C, ldc, n, (int)(rows / 2), ic));
    else
        DCK(launch_gemm_f16_pair(ctx_, x, ic, w16, ic, C, ldc, n, (int)rows, ic, epi == EPI_ADD_F32 ? 1 : 0));
    return cudaEventRecord(pf_consumed_[j & 1], ctx_->stream);
}

cudaError_t LlamaDecoder::pf_job_begin(int j, const __half **w16) {
    if (j + 1 < pf_njobs_) DCK(pf_expand_job(j + 1));
    DCK(cudaStreamWaitEvent(ctx_->stream, pf_expanded_[j & 1], 0));
    *w16 = pf_w16_[j & 1].get();
    return cudaSuccess;
}

// expansion of job j into scratch half (j & 1) on the side stream, after the GEMM that last read that half
cudaError_t LlamaDecoder::pf_expand_job(int j) {
    const PfJob &job = pf_jobs_[j];
    const int b = j & 1;
    Ctx side = *ctx_;
    side.stream = pf_side_;
    if (j >= 2) DCK(cudaStreamWaitEvent(pf_side_, pf_consumed_[b], 0));
    size_t r0 = 0;
    const int ic = job.ts[0]->ic, zw = zeros_width(ic, kW4Group);
    for (int i = 0; i < job.count; i++) {
        const tce_w4_tensor &t = *job.ts[i];
        const size_t r = (size_t)job.r0[i];  // first row of the range: offset pointers into the packed words, zeros and scales
        DCK(launch_w4_expand(&side, (const uint32_t *)t.w + r * (ic / 8), (const uint32_t *)t.zeros + r * zw, (const __half *)t.scales + r * zw * 8,
                             pf_w16_[b].get() + r0 * ic, job.rows[i], ic));
        r0 += (size_t)job.rows[i];
    }
    return cudaEventRecord(pf_expanded_[b], pf_side_);
}

// the job list, the double-buffered scratch, its events and the side stream, on first use
cudaError_t LlamaDecoder::pf_setup() {
    if (!pf_jobs_.empty()) return cudaSuccess;
    std::vector<PfJob> jobs;
    auto job = [](const tce_w4_tensor *a, const tce_w4_tensor *b, const tce_w4_tensor *c) {
        PfJob j{{a, b, c}, c ? 3 : (b ? 2 : 1), {0, 0, 0}, {0, 0, 0}};
        for (int i = 0; i < j.count; i++) j.rows[i] = j.ts[i]->oc;
        return j;
    };
    for (int l = 0; l < cfg_.num_layers; l++) {
        const tce_llama_layer &L = layers_[l];
        jobs.push_back(job(&L.q, &L.k, &L.v));
        jobs.push_back(job(&L.o, nullptr, nullptr));
        jobs.push_back(job(&L.gate, &L.up, nullptr));
        jobs.push_back(job(&L.down, nullptr, nullptr));
    }
    size_t need = 0;
    for (const PfJob &jb : jobs) {
        size_t e = 0;
        for (int i = 0; i < jb.count; i++) e += (size_t)jb.ts[i]->oc * jb.ts[i]->ic;
        need = e > need ? e : need;
    }
    // the lm_head does not fit a half at real vocabularies (Llama-3-8B: 1.05 GB of fp16 against 235 MB): it is expanded in chunks of whole
    // 256-row blocks (the CTA-pair GEMM's weight tile) that do; q|k|v alone is >= 384 rows of E, so a chunk is at least one block
    const int E = cfg_.embed_dim, V = cfg_.vocab_size;
    pf_lm_chunk_ = (int)(need / (size_t)E / 256 * 256);
    for (int r0 = 0; r0 < V; r0 += pf_lm_chunk_) {
        PfJob j = job(&w_.lm_head, nullptr, nullptr);
        j.r0[0] = r0;
        j.rows[0] = V - r0 < pf_lm_chunk_ ? V - r0 : pf_lm_chunk_;
        jobs.push_back(j);
    }
    for (int b = 0; b < 2; b++) {
        DCK(dev_alloc(pf_w16_[b], need));
        if (!pf_expanded_[b]) DCK(cudaEventCreateWithFlags(&pf_expanded_[b], cudaEventDisableTiming));
        if (!pf_consumed_[b]) DCK(cudaEventCreateWithFlags(&pf_consumed_[b], cudaEventDisableTiming));
    }
    if (!pf_side_) DCK(cudaStreamCreateWithFlags(&pf_side_, cudaStreamNonBlocking));
    pf_jobs_ = std::move(jobs);  // last: a non-empty job list means the scratch, events and side stream exist
    return cudaSuccess;
}

cudaError_t LlamaDecoder::prefill_rows(int n_seqs, const int *tokens_host, const int *lengths, const int *pos0s, const int *slots, bool score) {
    int n = 0;
    for (int i = 0; i < n_seqs; i++) n += lengths[i];
    DCK(prefill_reserve(n));
    DCK(pf_setup());
    pf_njobs_ = score ? (int)pf_jobs_.size() : 4 * cfg_.num_layers;
    // the side stream starts after everything already queued on the main stream (a previous prompt's GEMMs read the scratch)
    DCK(cudaEventRecord(pf_consumed_[0], ctx_->stream));
    DCK(cudaStreamWaitEvent(pf_side_, pf_consumed_[0], 0));
    DCK(pf_expand_job(0));
    cudaStream_t s = ctx_->stream;
    const int E = cfg_.embed_dim, F = cfg_.hidden_dim, H = cfg_.num_heads, KVH = cfg_.num_kv_heads, hd = cfg_.head_dim;
    const long long Q = (long long)(H + 2 * KVH) * hd;
    DCK(cudaMemcpyAsync(pf_.tok.get(), tokens_host, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, s));
    DCK(launch_embedding_rows(ctx_, (const __half *)w_.embed_f16, pf_.tok.get(), pf_.x.get(), n, E));
    AttnPrefillArgs a{};
    a.qkv = pf_.qkv.get();
    a.cos = d_cos_;
    a.sin = d_sin_;
    a.out = pf_.att.get();
    a.alpha = cfg_.qk_alpha > 0 ? cfg_.qk_alpha : 1.0f / sqrtf((float)hd);
    a.num_heads = H;
    a.num_kv_heads = KVH;
    a.head_dim = hd;
    a.max_ctx = cfg_.max_ctx;
    a.n_seqs = n_seqs;
    for (int i = 0, row0 = 0; i < n_seqs; row0 += lengths[i++]) a.seq[i] = AttnPrefillSeq{row0, lengths[i], pos0s[i], nullptr, nullptr};
    for (int l = 0; l < cfg_.num_layers; l++) {
        const tce_llama_layer &L = layers_[l];
        DCK(launch_rmsnorm_rows_f32(ctx_, pf_.x.get(), L.input_norm, pf_.xn.get(), n, E, cfg_.rms_eps));
        DCK(prefill_linear(4 * l, pf_.xn.get(), pf_.qkv.get(), Q, n, EPI_STORE_HALF));
        for (int i = 0; i < n_seqs; i++) {
            a.seq[i].k_cache = (__half *)kv_cache_slot(slots[i], l, 0);
            a.seq[i].v_cache = (__half *)kv_cache_slot(slots[i], l, 1);
        }
        DCK(launch_attn_prefill(ctx_, a));
        DCK(prefill_linear(4 * l + 1, pf_.att.get(), pf_.x.get(), E, n, EPI_ADD_F32));  // residual add in the GEMM epilogue
        DCK(launch_rmsnorm_rows_f32(ctx_, pf_.x.get(), L.post_norm, pf_.xn.get(), n, E, cfg_.rms_eps));
        DCK(prefill_linear(4 * l + 2, pf_.xn.get(), pf_.act.get(), F, n, EPI_SILU_MUL_HALF));  // SiLU(gate) * up in the GEMM epilogue: gate|up never reach HBM
        DCK(prefill_linear(4 * l + 3, pf_.act.get(), pf_.x.get(), E, n, EPI_ADD_F32));
    }
    return cudaSuccess;
}

// only the last position of a prompt feeds the sampler.  Prompt b's last row is at row >= b, so moving it to row b of pf_.x overwrites no
// row that a later copy still reads.
cudaError_t LlamaDecoder::prompt_logits(int n_seqs, const int *lengths, float *logits, int *next) {
    const int E = cfg_.embed_dim;
    for (int b = 0, row = 0; b < n_seqs; b++) {
        row += lengths[b];
        if (row - 1 != b)
            DCK(cudaMemcpyAsync(pf_.x.get() + (size_t)b * E, pf_.x.get() + (size_t)(row - 1) * E, (size_t)E * sizeof(float), cudaMemcpyDeviceToDevice,
                                ctx_->stream));
    }
    W4GemvParams p = lm_head_gemv(pf_.x.get(), logits);
    p.M = n_seqs;
    DCK(launch_w4a16_gemv(ctx_, p));
    return launch_argmax_rows(ctx_, logits, n_seqs, cfg_.vocab_size, next, false);
}

cudaError_t LlamaDecoder::prefill(const int *tokens_host, int n, int pos0, float *logits_host, int *next_token, std::string *err, int slot) {
    if (tp_ > 1) {
        if (err) *err = "prefill is single-GPU in this build (tensor-parallel ranks process the prompt with decode steps)";
        return cudaErrorNotSupported;
    }
    int rows = 0;
    DCK(check_prompts(1, tokens_host, &n, &pos0, &slot, &rows));
    DCK(prefill_rows(1, tokens_host, &n, &pos0, &slot));
    DCK(prompt_logits(1, &n, io1_.logits.get(), io1_.next.get()));
    DCK(io1_.read_back(1, StepIO::wanted(logits_host), ctx_->stream));
    return io1_.copy_out(1, logits_host, next_token, ctx_->stream);
}

}  // namespace tce

// ------------------------------------------------------------------------------------------------ batched decode
// Up to TCE_LLAMA_MAX_BATCH sequences per step, each in its own KV-cache slot: a batched embedding kernel range-checks every request, then
// per layer the GEMVs run with M = batch rows (one pass over each weight matrix) and the attention kernel takes one grid layer per sequence.
// At batch 1 on slot 0 this is also the kernel-per-op single-sequence step.
namespace tce {

cudaError_t LlamaDecoder::batch_alloc(std::string *err) {
    auto no = [&](const char *m) {
        if (err) *err = m;
        return cudaErrorNotSupported;
    };
    if (tp_ > 1) return no("the batched step is single-GPU (tp_size > 1)");
    if (bs_) return cudaSuccess;
    const int nrep = cfg_.num_heads / cfg_.num_kv_heads;
    if (nrep != 1 && nrep != 2 && nrep != 4 && nrep != 8) return no("the batched attention kernel takes 1, 2, 4 or 8 query heads per KV head");
    const size_t B = TCE_LLAMA_MAX_BATCH, E = cfg_.embed_dim, F = cfg_.hidden_dim, V = cfg_.vocab_size,
                 Q = (size_t)(cfg_.num_heads + 2 * cfg_.num_kv_heads) * cfg_.head_dim, A = (size_t)cfg_.num_heads * cfg_.head_dim;
    // all or nothing: the set is built aside and published whole; a failed allocation frees what this call took
    std::unique_ptr<BatchState> st = std::make_unique<BatchState>();
    // the span step's attention runs the largest split that fits shared memory at 8 rows, and n <= 8 rows use the records of n sequences
    st->span_chunk = attn_span_chunk(cfg_.num_heads, cfg_.num_kv_heads, attn_chunk_, ctx_->smem_optin);
    st->attn_ws_floats = B * attn_decode_ws_floats(cfg_.num_heads, cfg_.max_ctx, attn_chunk_);
    if (st->span_chunk) {
        const size_t span_ws = (size_t)kMaxSpan * attn_decode_ws_floats(cfg_.num_heads, cfg_.max_ctx, st->span_chunk);
        st->attn_ws_floats = span_ws > st->attn_ws_floats ? span_ws : st->attn_ws_floats;
    }
    st->n_counters = B * cfg_.num_kv_heads;
    __half *kv0 = d_kv_.get();
    cudaError_t e = cudaSuccess;
    auto D = [&](auto &p, size_t count) {
        if (e == cudaSuccess) e = dev_alloc(p, count);
    };
    D(st->resid, B * E);
    D(st->qkv, B * Q);
    D(st->attn, B * A);
    D(st->act, B * F);
    D(st->safe, B * 4);
    D(st->attn_ws, st->attn_ws_floats);
    D(st->attn_counters, st->n_counters);
    D(st->slot_table, 1);
    if (e == cudaSuccess) e = st->io.alloc((int)B, (int)V);
    if (e == cudaSuccess) e = cudaMemset(st->attn_counters.get(), 0, st->n_counters * sizeof(unsigned));  // the split merge re-arms them after every use
    if (e == cudaSuccess) e = cudaMemcpy(st->slot_table.get(), &kv0, sizeof(__half *), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        if (err) *err = std::string("batched-step buffers: ") + cudaGetErrorString(e);
        return e;
    }
    auto gemv = [&](std::initializer_list<const tce_w4_tensor *> ts, const void *x, int ldx, const float *gamma, void *y, int ldy, int epi) {
        W4GemvParams p;
        p.nseg = 0;
        for (const tce_w4_tensor *t : ts) p.seg[p.nseg++] = seg_of(*t);
        p.pair_mode = epi == EPI_SILU_MUL_HALF ? 1 : 0;
        p.IC = ts.begin()[0]->ic;
        p.x = x;
        p.ldx = ldx;
        p.x_mode = gamma ? X_RMSNORM_F32 : X_HALF;
        p.gamma = gamma;
        p.eps = cfg_.rms_eps;
        p.y = y;
        p.ldy = ldy;
        p.epi = epi;
        p.atomic_residual = epi == EPI_ADD_F32 && atomic_residual_;
        st->gemv_ops.push_back(p);
    };
    for (int l = 0; l < cfg_.num_layers; l++) {
        const tce_llama_layer &L = layers_[l];
        // RMSNorm(input_layernorm) + q|k|v; o_proj accumulated into the residual; RMSNorm(post_attention_layernorm) + gate/up with the
        // SiLU(gate) * up epilogue; down_proj + residual
        gemv({&L.q, &L.k, &L.v}, st->resid.get(), (int)E, L.input_norm, st->qkv.get(), (int)Q, EPI_STORE_HALF);
        gemv({&L.o}, st->attn.get(), (int)A, nullptr, st->resid.get(), (int)E, EPI_ADD_F32);
        gemv({&L.gate, &L.up}, st->resid.get(), (int)E, L.post_norm, st->act.get(), (int)F, EPI_SILU_MUL_HALF);
        gemv({&L.down}, st->act.get(), (int)F, nullptr, st->resid.get(), (int)E, EPI_ADD_F32);
        // RoPE + in-place KV append + attention over the cache of each sequence's slot
        AttnDecodeArgs a{};
        a.qkv = st->qkv.get();
        a.cos = d_cos_;
        a.sin = d_sin_;
        a.out = st->attn.get();
        a.alpha = cfg_.qk_alpha > 0 ? cfg_.qk_alpha : 1.0f / sqrtf((float)cfg_.head_dim);
        a.num_heads = cfg_.num_heads;
        a.num_kv_heads = cfg_.num_kv_heads;
        a.head_dim = cfg_.head_dim;
        a.max_ctx = cfg_.max_ctx;
        a.chunk = attn_chunk_;
        a.ws = st->attn_ws.get();
        a.counters = st->attn_counters.get();
        a.ws_floats = st->attn_ws_floats;
        a.n_counters = st->n_counters;
        a.req = st->safe.get();
        a.k_off = (__half *)kv_cache(l, 0) - kv0;  // this layer's slabs within a slot
        a.v_off = (__half *)kv_cache(l, 1) - kv0;
        a.qkv_stride = (int)Q;
        a.out_stride = (int)A;
        st->attn_ops.push_back(a);
    }
    st->gemv_ops.push_back(lm_head_gemv(st->resid.get(), st->io.logits.get()));
    bs_ = std::move(st);
    return cudaSuccess;
}

// final RMSNorm + lm_head -> fp32 logits (reference: lm_head GEMV + half2float, cuda/Int4llamaForCausalLM.cu:33-38)
W4GemvParams LlamaDecoder::lm_head_gemv(const float *x, float *y) const {
    W4GemvParams p;
    p.seg[0] = seg_of(w_.lm_head);
    p.IC = cfg_.embed_dim;
    p.x = x;
    p.ldx = cfg_.embed_dim;
    p.x_mode = X_RMSNORM_F32;
    p.gamma = w_.final_norm;
    p.eps = cfg_.rms_eps;
    p.y = y;
    p.ldy = cfg_.vocab_size;
    p.epi = EPI_STORE_F32;
    return p;
}

const float *LlamaDecoder::batch_logits() { return batch_alloc(nullptr) == cudaSuccess ? bs_->io.logits.get() : nullptr; }

cudaError_t LlamaDecoder::reserve_slots(int n, std::string *err) {
    if (tp_ > 1) return batch_alloc(err);  // not supported, with its message
    if (n < 1 || n > 1024) return cudaErrorInvalidValue;
    DCK(batch_alloc(err));
    if (n <= n_slots()) return cudaSuccess;
    // queued work may still read the old table: drain it before the table (and the graphs holding it) go away
    DCK(cudaStreamSynchronize(ctx_->stream));
    DCK(cudaStreamSynchronize(cap_stream_));
    // all or nothing: the new slots and the table that lists them are built aside and only then published, so the slot count and the
    // device table always agree (a failed call leaves both as they were)
    const size_t kv_elems = (size_t)cfg_.num_layers * 2 * cfg_.num_kv_heads * cfg_.max_ctx * cfg_.head_dim;
    std::vector<DevPtr<__half>> added;
    DevPtr<__half *> table;
    std::vector<__half *> h;
    h.push_back(d_kv_.get());
    for (const DevPtr<__half> &p : slot_kv_) h.push_back(p.get());
    cudaError_t e = cudaSuccess;
    while (e == cudaSuccess && (int)h.size() < n) {
        added.emplace_back();
        e = dev_alloc(added.back(), kv_elems);
        if (e == cudaSuccess) e = cudaMemset(added.back().get(), 0, kv_elems * sizeof(__half));
        h.push_back(added.back().get());
    }
    if (e == cudaSuccess) e = dev_alloc(table, h.size());
    if (e == cudaSuccess) e = cudaMemcpy(table.get(), h.data(), h.size() * sizeof(__half *), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        cudaGetLastError();
        if (err) *err = std::string("slot allocation: ") + cudaGetErrorString(e);
        return e;
    }
    graphs_.clear();  // they hold the old table and slot count
    bs_->slot_table = std::move(table);
    for (DevPtr<__half> &p : added) slot_kv_.push_back(std::move(p));
    return cudaSuccess;
}

cudaError_t LlamaDecoder::enqueue_batch(int batch, const int *req, float *logits, int *next, cudaStream_t s, bool pdl, bool span) {
    const BatchState &st = *bs_;
    // the K-sliced GEMVs' fix-up records are grown on the context itself (the launches below see a copy of it); a no-op after the first step
    long long records = 0;
    for (W4GemvParams p : st.gemv_ops) {
        p.M = batch;
        const long long r = w4a16_gemv_fixup_records(ctx_, p);
        records = r > records ? r : records;
    }
    DCK(gemv_partials_reserve(ctx_, records));
    Ctx local = *ctx_;
    local.stream = s;
    Ctx *c = &local;
    auto gemv = [&](W4GemvParams p) {
        p.M = batch;
        p.pdl = pdl;
        return launch_w4a16_gemv(c, p);
    };
    DCK(launch_embedding_batch(c, (const __half *)w_.embed_f16, req, st.resid.get(), cfg_.embed_dim, batch, cfg_.vocab_size, cfg_.max_ctx, n_slots(),
                               st.safe.get(), false));
    for (int l = 0; l < cfg_.num_layers; l++) {
        DCK(gemv(st.gemv_ops[4 * l]));
        AttnDecodeArgs a = st.attn_ops[l];
        a.slots = st.slot_table.get();
        if (span) a.chunk = st.span_chunk;
        DCK(launch_attn_decode(c, a, span ? 1 : batch, span ? batch : 1, pdl));
        for (int i = 1; i < 4; i++) DCK(gemv(st.gemv_ops[4 * l + i]));
    }
    W4GemvParams lm = st.gemv_ops.back();
    lm.y = logits;
    DCK(gemv(lm));
    return launch_argmax_rows(c, logits, batch, cfg_.vocab_size, next, pdl);
}

cudaError_t LlamaDecoder::decode_batch_device(int batch, const int *req_dev, std::string *err) {
    if (tp_ > 1) return batch_alloc(err);  // not supported, with its message
    if (batch < 1 || batch > TCE_LLAMA_MAX_BATCH || !req_dev) return cudaErrorInvalidValue;
    DCK(step_ready(Step::batch, err));
    return run_graphed(graphs_[{kDevice, Step::batch, batch, StepIO::kNone}], req_dev,
                       [&](cudaStream_t st, bool pdl) { return enqueue(Step::batch, batch, req_dev, st, pdl); });
}

cudaError_t LlamaDecoder::decode_batch_host(int batch, const int *tokens, const int *positions, const int *slots, float *logits_host, int *next_tokens,
                                            std::string *err) {
    if (tp_ > 1) return batch_alloc(err);  // not supported, with its message
    if (batch < 1 || batch > TCE_LLAMA_MAX_BATCH || !tokens || !positions || !slots || !slots_ok(batch, slots)) return cudaErrorInvalidValue;
    for (int b = 0; b < batch; b++)
        if (tokens[b] < 0 || tokens[b] >= cfg_.vocab_size || positions[b] < 0 || positions[b] >= cfg_.max_ctx) return cudaErrorInvalidValue;
    DCK(step_ready(Step::batch, err));
    int *h_req = bs_->io.h_req.get();
    for (int b = 0; b < batch; b++) {
        h_req[3 * b] = tokens[b];
        h_req[3 * b + 1] = positions[b];
        h_req[3 * b + 2] = slots[b];
    }
    DCK(run_host(Step::batch, batch, StepIO::wanted(logits_host)));
    return bs_->io.copy_out(batch, logits_host, next_tokens, ctx_->stream);
}

// ------------------------------------------------------------------------------------------------ span step
// n consecutive tokens of one slot in one pass over the weights: the batched step's chain at M = n with every row in the same slot, and the
// span attention (append of the n new K / V rows, then causal multi-query attention) in place of the per-sequence attention.
bool LlamaDecoder::span_ok(int slot, int pos0, int n, const int *tokens) const {
    if (n < 1 || n > kMaxSpan || !tokens || slot < 0 || slot >= n_slots() || pos0 < 0 || pos0 > cfg_.max_ctx - n) return false;
    for (int i = 0; i < n; i++)
        if (tokens[i] < 0 || tokens[i] >= cfg_.vocab_size) return false;
    return true;
}

cudaError_t LlamaDecoder::span_supported(std::string *err) const {
    if (bs_->span_chunk > 0) return cudaSuccess;
    if (err) *err = "the span attention's CTA does not fit this device's shared memory at this head ratio";
    return cudaErrorNotSupported;
}

cudaError_t LlamaDecoder::decode_span_host(int slot, int pos0, int n, const int *tokens, float *logits_host, int *next_tokens, std::string *err) {
    if (tp_ > 1) return batch_alloc(err);  // not supported, with its message
    if (!span_ok(slot, pos0, n, tokens)) return cudaErrorInvalidValue;
    DCK(step_ready(Step::span, err));
    bs_->io.stage(slot, pos0, n, tokens);
    DCK(run_host(Step::span, n, StepIO::wanted(logits_host)));
    return bs_->io.copy_out(n, logits_host, next_tokens, ctx_->stream);
}

// ------------------------------------------------------------------------------------------------ speculative loop
// Prompt-lookup drafter (the rule stated at tce_llama_generate_lookup): the tokens that followed the most recent earlier occurrence of the
// longest suffix of S (ngram_max down to ngram_min) that has one.
static_assert(kMaxSpan == TCE_LLAMA_MAX_BATCH && kMaxDrafts + 1 == kMaxSpan, "a span is one batched step's rows: the last token plus the drafts");
static int lookup_draft(const std::vector<int> &S, const tce_lookup &lk, int d, int *out) {
    const int len = (int)S.size();
    if (d <= 0) return 0;
    for (int ng = lk.ngram_max; ng >= lk.ngram_min; ng--) {
        if (ng + 1 > len) continue;
        const int *suf = S.data() + len - ng;
        for (int p = len - ng - 1; p >= 0; p--) {
            if (memcmp(S.data() + p, suf, (size_t)ng * sizeof(int))) continue;
            const int avail = len - (p + ng), m = avail < d ? avail : d;
            for (int i = 0; i < m; i++) out[i] = S[p + ng + i];
            return m;
        }
    }
    return 0;
}

cudaError_t LlamaDecoder::generate_lookup(int first_token, int pos0, int n_predict, const tce_sampling &sc, const int *history, int n_history, const int *corpus,
                                          int n_corpus, const tce_lookup &lk, int eos_id, int *out_tokens, int *n_out, tce_lookup_stats *stats,
                                          std::string *err) {
    if (tp_ > 1) return batch_alloc(err);  // not supported, with its message
    const int cap = cfg_.max_ctx;
    if (first_token < 0 || first_token >= cfg_.vocab_size || pos0 < 0 || pos0 >= cap || n_predict < 0 || n_history < 0 || n_history > cap ||
        n_corpus < 0 || (n_history > 0 && !history) || (n_corpus > 0 && !corpus) || !n_out || (n_predict > 0 && !out_tokens) || lk.max_draft < 0 ||
        lk.max_draft > kMaxDrafts || lk.ngram_min < 1 || lk.ngram_min > lk.ngram_max)
        return cudaErrorInvalidValue;
    if (!sampling_supported(sc.temp, sc.top_k, cfg_.vocab_size)) {
        if (err) *err = "temp > 0 needs 1 <= top_k <= 1024";
        return cudaErrorNotSupported;
    }
    if (n_predict > cap - pos0) n_predict = cap - pos0;
    DCK(batch_alloc(err));
    if (lk.max_draft > 0) DCK(span_supported(err));
    cudaStream_t s = ctx_->stream;
    // [0] arrival counter, [1] history head, [4..15) step result, [16..24) replacement ids, [24..32) draft probabilities, then the history
    // ring [max_ctx]
    if (!d_spec_) DCK(dev_alloc(d_spec_, (size_t)(32 + cap)));
    if (!h_spec_) DCK(host_alloc(h_spec_, 16));
    int *ring = d_spec_.get() + 32;
    DCK(cudaMemsetAsync(d_spec_.get(), 0, 32 * sizeof(int), s));
    if (n_history > 0) DCK(cudaMemcpyAsync(ring, history, (size_t)n_history * sizeof(int), cudaMemcpyHostToDevice, s));
    const int head0 = n_history;
    DCK(cudaMemcpyAsync(d_spec_.get() + 1, &head0, sizeof(int), cudaMemcpyHostToDevice, s));
    DCK(cudaStreamSynchronize(s));  // head0 and the caller's arrays are read by now
    AcceptArgs acc{};
    acc.chain = sample_args(sc, nullptr, cfg_.vocab_size);
    acc.chain.hist = ring;
    acc.chain.hist_head = d_spec_.get() + 1;
    acc.chain.hist_cap = cap;
    acc.eos_id = eos_id;
    acc.ld = (size_t)cfg_.vocab_size;
    acc.repl = d_spec_.get() + 16;
    acc.q = reinterpret_cast<float *>(d_spec_.get() + 24);
    acc.arrive = reinterpret_cast<unsigned *>(d_spec_.get());
    acc.result = d_spec_.get() + 4;
    std::vector<int> S;
    S.reserve((size_t)n_corpus + n_history + 1 + n_predict);
    S.insert(S.end(), corpus, corpus + n_corpus);
    S.insert(S.end(), history, history + n_history);
    S.push_back(first_token);
    tce_lookup_stats st{0, 0, 0};
    int n = 0, pos = pos0, last = first_token;
    int *res = h_spec_.get();
    while (n < n_predict) {
        const int left = n_predict - n;
        int lim = lk.max_draft;
        if (lim > left - 1) lim = left - 1;
        if (lim > cap - pos - 1) lim = cap - pos - 1;
        const int d = lookup_draft(S, lk, lim, acc.drafts);
        acc.rows = d + 1;
        acc.budget = left;
        // without drafts the single-sequence step (the persistent kernel where it applies), as tce_llama_generate runs it
        const Step k = d == 0 ? Step::single : Step::span;
        int toks[kMaxSpan];
        toks[0] = last;
        for (int i = 0; i < d; i++) toks[i + 1] = acc.drafts[i];
        io(k).stage(0, pos, d + 1, toks);
        DCK(run_host(k, d + 1, StepIO::kNone));  // accept_kernel reads the logits on the device
        acc.chain.logits = io(k).logits.get();
        DCK(launch_accept(acc, s));
        // the host drafts the next step from these ids: one small read-back per step
        DCK(cudaMemcpyAsync(res, acc.result, 11 * sizeof(int), cudaMemcpyDeviceToHost, s));
        DCK(cudaStreamSynchronize(s));
        const int emitted = res[0];
        st.steps++;
        st.drafted += d;
        st.accepted += res[2];
        for (int i = 0; i < emitted; i++) {
            out_tokens[n + i] = res[3 + i];
            S.push_back(res[3 + i]);
        }
        n += emitted;
        pos += emitted;
        last = res[3 + emitted - 1];
        if (res[1]) break;
    }
    *n_out = n;
    if (stats) *stats = st;
    return cudaSuccess;
}

// ------------------------------------------------------------------------------------------------ batched prompt pass and generate loop
bool LlamaDecoder::slots_ok(int n, const int *slots) const {
    for (int b = 0; b < n; b++) {
        if (slots[b] < 0 || slots[b] >= n_slots()) return false;
        for (int o = 0; o < b; o++)
            if (slots[o] == slots[b]) return false;
    }
    return true;
}

cudaError_t LlamaDecoder::check_prompts(int n_seqs, const int *tokens_host, const int *lengths, const int *pos0s, const int *slots, int *n) const {
    if (n_seqs < 1 || n_seqs > TCE_LLAMA_MAX_BATCH || !tokens_host || !lengths || !pos0s || !slots || !slots_ok(n_seqs, slots))
        return cudaErrorInvalidValue;
    int rows = 0;
    for (int b = 0; b < n_seqs; b++) {
        if (lengths[b] < 1 || pos0s[b] < 0 || pos0s[b] > cfg_.max_ctx - lengths[b]) return cudaErrorInvalidValue;
        rows += lengths[b];
    }
    for (int i = 0; i < rows; i++)
        if (tokens_host[i] < 0 || tokens_host[i] >= cfg_.vocab_size) return cudaErrorInvalidValue;
    *n = rows;
    return cudaSuccess;
}

cudaError_t LlamaDecoder::prefill_batch(int n_seqs, const int *tokens_host, const int *lengths, const int *pos0s, const int *slots, float *logits_host,
                                        int *next_tokens, std::string *err) {
    if (tp_ > 1) return batch_alloc(err);  // not supported, with its message
    int n = 0;
    DCK(check_prompts(n_seqs, tokens_host, lengths, pos0s, slots, &n));
    DCK(batch_alloc(err));
    DCK(prefill_rows(n_seqs, tokens_host, lengths, pos0s, slots));
    StepIO &b = bs_->io;
    DCK(prompt_logits(n_seqs, lengths, b.logits.get(), b.next.get()));
    DCK(b.read_back(n_seqs, StepIO::wanted(logits_host), ctx_->stream));
    return b.copy_out(n_seqs, logits_host, next_tokens, ctx_->stream);
}

// ------------------------------------------------------------------------------------------------ teacher-forced scoring
cudaError_t LlamaDecoder::score_reserve(int n) {
    if (n <= sc_.cap) return cudaSuccess;
    DCK(cudaStreamSynchronize(ctx_->stream));
    sc_ = ScoreBufs{};  // the old buffers go first
    ScoreBufs b;
    DCK(dev_alloc(b.rec, (size_t)n * (pf_lm_chunk_ / 128)));
    DCK(dev_alloc(b.state, (size_t)n));
    DCK(dev_alloc(b.target, (size_t)n));
    DCK(dev_alloc(b.tgt, (size_t)n));
    DCK(dev_alloc(b.out, (size_t)3 * n));
    b.cap = n;
    sc_ = std::move(b);
    return cudaSuccess;
}

// The prompt pass of prefill_batch, then the final RMSNorm over all n rows and the lm_head as the W4A16 prompt-pass GEMM, chunk by chunk on the
// same double-buffered expansion (the first chunk expands while the last down_proj runs).  The GEMM epilogue reduces each row's 128-column
// slices to {max, sum of exp, arg-max} records; a merge kernel folds them in column order into a running state per row and, after the last
// chunk, writes the log-probabilities.  Every reduction has a fixed order: the results do not depend on the other rows of the call.
cudaError_t LlamaDecoder::score_batch(int n_seqs, const int *tokens_host, const int *lengths, const int *pos0s, const int *slots, const int *targets_host,
                                      float *logprobs_host, int *greedy_host, float *greedy_logprobs_host, float *logits_dev, std::string *err) {
    if (tp_ > 1) {
        if (err) *err = "scoring is single-GPU in this build (tp_size > 1)";
        return cudaErrorNotSupported;
    }
    int n = 0;
    DCK(check_prompts(n_seqs, tokens_host, lengths, pos0s, slots, &n));
    const int E = cfg_.embed_dim, V = cfg_.vocab_size;
    std::vector<int> target(n);
    if (targets_host) {
        for (int i = 0; i < n; i++) {
            if (targets_host[i] < -1 || targets_host[i] >= V) return cudaErrorInvalidValue;
            target[i] = targets_host[i];
        }
    } else {  // the next token of the same prompt; none after a prompt's last row
        for (int b = 0, row = 0; b < n_seqs; row += lengths[b++])
            for (int i = 0; i < lengths[b]; i++) target[row + i] = i + 1 < lengths[b] ? tokens_host[row + i + 1] : -1;
    }
    DCK(prefill_reserve(n));
    DCK(pf_setup());
    DCK(score_reserve(n));
    DCK(prefill_rows(n_seqs, tokens_host, lengths, pos0s, slots, true));
    cudaStream_t s = ctx_->stream;
    DCK(cudaMemcpyAsync(sc_.target.get(), target.data(), (size_t)n * sizeof(int), cudaMemcpyHostToDevice, s));
    DCK(launch_rmsnorm_rows_f32(ctx_, pf_.x.get(), w_.final_norm, pf_.xn.get(), n, E, cfg_.rms_eps));
    float *logprob = sc_.out.get(), *glp = sc_.out.get() + 2 * (size_t)n;
    int *greedy = reinterpret_cast<int *>(sc_.out.get() + n);
    const int rec_ld = pf_lm_chunk_ / 128, first = 4 * cfg_.num_layers;
    for (int j = first; j < pf_njobs_; j++) {
        const PfJob &job = pf_jobs_[j];
        const __half *w16 = nullptr;
        DCK(pf_job_begin(j, &w16));
        DCK(launch_gemm_f16_pair_stats(ctx_, pf_.xn.get(), E, w16, E, n, job.rows[0], E, job.r0[0], sc_.rec.get(), rec_ld, sc_.target.get(), sc_.tgt.get(),
                                       logits_dev, V));
        DCK(cudaEventRecord(pf_consumed_[j & 1], s));
        DCK(launch_lm_stats_merge(ctx_, sc_.rec.get(), rec_ld, (job.rows[0] + 127) / 128, n, j == first, j + 1 == pf_njobs_, sc_.state.get(),
                                  sc_.target.get(), sc_.tgt.get(), logprob, greedy, glp));
    }
    if (logprobs_host) DCK(cudaMemcpyAsync(logprobs_host, logprob, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, s));
    if (greedy_host) DCK(cudaMemcpyAsync(greedy_host, greedy, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, s));
    if (greedy_logprobs_host) DCK(cudaMemcpyAsync(greedy_logprobs_host, glp, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, s));
    return cudaStreamSynchronize(s);
}

cudaError_t LlamaDecoder::generate_batch(int batch, const tce_gen_request *reqs, int *out_tokens_host, int out_stride, int *n_out, std::string *err) {
    if (tp_ > 1) return batch_alloc(err);  // not supported, with its message
    return generate_rows(Step::batch, batch, reqs, out_tokens_host, out_stride, n_out, err);
}

// Generate loop (LLaMAGenerate.cu:67-252 without the tokenizer / console parts) of up to TCE_LLAMA_MAX_BATCH sequences: every token is one
// step of kind k on the request buffer io(k).req and one sampler launch with a block per row, which writes each row's next {token,
// position} into that buffer; both are one cached graph.  A row that stops gets the out-of-range position max_ctx there, so the step
// refuses it and it appends no KV row in any later step.  Stopped rows still ride along as rows of the GEMVs.  The host only looks at the
// stop flags every few tokens, and copies the generated ids out at the end.
cudaError_t LlamaDecoder::generate_rows(Step k, int batch, const tce_gen_request *reqs, int *out_tokens_host, int out_stride, int *n_out,
                                        std::string *err) {
    if (batch < 1 || batch > TCE_LLAMA_MAX_BATCH || !reqs || !n_out || out_stride < 0) return cudaErrorInvalidValue;
    const int cap = cfg_.max_ctx, V = cfg_.vocab_size, B = TCE_LLAMA_MAX_BATCH;
    int n_pred[TCE_LLAMA_MAX_BATCH], slots[TCE_LLAMA_MAX_BATCH], steps = 0;
    for (int b = 0; b < batch; b++) {
        const tce_gen_request &r = reqs[b];
        if (r.first_token < 0 || r.first_token >= V || r.pos0 < 0 || r.pos0 >= cap || r.n_predict < 0 || r.n_history < 0 || r.n_history > cap ||
            (r.n_history > 0 && !r.history))
            return cudaErrorInvalidValue;
        slots[b] = r.slot;
        n_pred[b] = r.n_predict < cap - r.pos0 ? r.n_predict : cap - r.pos0;
        if (out_stride < n_pred[b]) return cudaErrorInvalidValue;
        steps = n_pred[b] > steps ? n_pred[b] : steps;
    }
    if (!slots_ok(batch, slots) || (steps > 0 && !out_tokens_host)) return cudaErrorInvalidValue;
    for (int b = 0; b < batch; b++) {
        const tce_sampling &sc = reqs[b].sampling;
        if (!sampling_supported(sc.temp, sc.top_k, V)) {
            if (err) *err = "generate: temp > 0 needs 1 <= top_k <= 1024";
            return cudaErrorNotSupported;
        }
    }
    DCK(step_ready(k, err));
    if (!loop_) {
        std::unique_ptr<LoopState> l = std::make_unique<LoopState>();
        DCK(dev_alloc(l->words, (size_t)B * 4 + (size_t)2 * B * cap));
        DCK(dev_alloc(l->sample, (size_t)B));
        loop_ = std::move(l);
    }
    cudaStream_t s = ctx_->stream;
    StepIO &io_k = io(k);
    int *ctl = loop_->words.get(), *hist = ctl + 4 * B, *out_list = hist + (size_t)B * cap;  // per row: {history head, output count, stop flag, unused}
    int *h_req = io_k.h_req.get();
    int ctl_h[4 * TCE_LLAMA_MAX_BATCH] = {};
    SampleArgs args[TCE_LLAMA_MAX_BATCH];
    for (int b = 0; b < batch; b++) {
        const tce_gen_request &r = reqs[b];
        if (r.n_history > 0)
            DCK(cudaMemcpyAsync(hist + (size_t)b * cap, r.history, (size_t)r.n_history * sizeof(int), cudaMemcpyHostToDevice, s));
        ctl_h[4 * b] = r.n_history;
        ctl_h[4 * b + 2] = n_pred[b] == 0;  // nothing to generate: stopped from the start
        h_req[3 * b] = r.first_token;
        h_req[3 * b + 1] = n_pred[b] == 0 ? cap : r.pos0;
        h_req[3 * b + 2] = r.slot;
        SampleArgs &a = args[b];
        a = sample_args(r.sampling, io_k.logits.get() + (size_t)b * V, V);
        a.hist = hist + (size_t)b * cap;
        a.hist_head = ctl + 4 * b;
        a.hist_cap = cap;
        a.eos_id = r.eos_id;
        a.tokpos = io_k.req.get() + 3 * b;
        a.out_list = out_list + (size_t)b * cap;
        a.out_count = ctl + 4 * b + 1;
        a.out_cap = cap;
        a.stop = ctl + 4 * b + 2;
        a.out_limit = n_pred[b];
        a.pos_limit = cap;
    }
    DCK(cudaMemcpyAsync(ctl, ctl_h, (size_t)4 * batch * sizeof(int), cudaMemcpyHostToDevice, s));
    const bool one = k == Step::single;
    if (!one) DCK(cudaMemcpyAsync(loop_->sample.get(), args, (size_t)batch * sizeof(SampleArgs), cudaMemcpyHostToDevice, s));
    DCK(cudaMemcpyAsync(io_k.req.get(), h_req, (size_t)batch * 3 * sizeof(int), cudaMemcpyHostToDevice, s));
    auto body = [&](cudaStream_t st, bool pdl) {
        DCK(enqueue(k, batch, io_k.req.get(), st, pdl));
        return one ? launch_sample(args[0], st) : launch_sample_rows(loop_->sample.get(), batch, st);
    };
    constexpr int kCheckEvery = 16;
    CachedGraph &g = graphs_[{kLoop, k, batch, StepIO::kNone}];
    // one row's sampler takes its arguments as kernel parameters, which the graph holds by value: it is captured anew for every call
    if (one) g.reset();
    for (int i = 0; i < steps; i++) {
        DCK(run_graphed(g, nullptr, body));
        if ((i + 1) % kCheckEvery == 0 && i + 1 < steps) {
            DCK(cudaMemcpyAsync(ctl_h, ctl, (size_t)4 * batch * sizeof(int), cudaMemcpyDeviceToHost, s));
            DCK(cudaStreamSynchronize(s));
            bool all = true;
            for (int b = 0; b < batch; b++) all = all && ctl_h[4 * b + 2];
            if (all) break;
        }
    }
    DCK(cudaMemcpyAsync(ctl_h, ctl, (size_t)4 * batch * sizeof(int), cudaMemcpyDeviceToHost, s));
    DCK(cudaStreamSynchronize(s));
    for (int b = 0; b < batch; b++) {
        const int n = ctl_h[4 * b + 1] < n_pred[b] ? ctl_h[4 * b + 1] : n_pred[b];
        if (n > 0) DCK(cudaMemcpy(out_tokens_host + (size_t)b * out_stride, out_list + (size_t)b * cap, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost));
        n_out[b] = n;
    }
    return cudaSuccess;
}

// ------------------------------------------------------------------------------------------------ KV-cache row copies
// Forking a prompt's rows into other slots (d = 0) and shifting a slot's context down past n_keep (one destination, the source slot).  The
// slot table and slot count stay as they are, so no cached graph is dropped; the launch is stream-ordered with the steps and loops.
cudaError_t LlamaDecoder::kv_copy(int src_slot, int src_pos, int n, int n_dst, const int *dst_slots, const int *dst_pos, std::string *err) {
    static_assert(kMaxKvCopyDst == TCE_LLAMA_MAX_BATCH, "one launch covers the destinations of a batch");
    auto bad = [&](const char *m) {
        if (err) *err = m;
        return cudaErrorInvalidValue;
    };
    if (tp_ > 1) {
        if (err) *err = "KV-cache slots are single-GPU (tp_size > 1)";
        return cudaErrorNotSupported;
    }
    const int cap = cfg_.max_ctx;
    if (n_dst < 1 || n_dst > kMaxKvCopyDst || !dst_slots || !dst_pos) return bad("n_dst outside [1, TCE_LLAMA_MAX_BATCH]");
    if (n < 0) return bad("n < 0");
    auto in_range = [&](int pos) { return pos >= 0 && pos <= cap && n <= cap - pos; };  // rows pos..pos+n-1 within [0, max_ctx)
    if (src_slot < 0 || src_slot >= n_slots()) return bad("source slot not reserved");
    if (!in_range(src_pos)) return bad("source rows outside [0, max_ctx)");
    auto overlap = [&](int sa, int pa, int sb, int pb) { return sa == sb && (pa > pb ? pa - pb : pb - pa) < n; };
    for (int i = 0; i < n_dst; i++) {
        if (dst_slots[i] < 0 || dst_slots[i] >= n_slots()) return bad("destination slot not reserved");
        if (!in_range(dst_pos[i])) return bad("destination rows outside [0, max_ctx)");
        for (int j = 0; j < i; j++)
            if (overlap(dst_slots[i], dst_pos[i], dst_slots[j], dst_pos[j])) return bad("two destinations overlap in one slot");
        if (n_dst > 1 && overlap(dst_slots[i], dst_pos[i], src_slot, src_pos)) return bad("a destination overlaps the source (allowed for a single destination only)");
    }
    if (n == 0) return cudaSuccess;
    KvCopyArgs a{};
    auto base = [&](int slot) { return (__half *)kv_cache_slot(slot, 0, 0); };
    a.src = base(src_slot);
    for (int i = 0; i < n_dst; i++) {
        a.dst[i] = base(dst_slots[i]);
        a.dst_pos[i] = dst_pos[i];
    }
    a.n_dst = n_dst;
    a.src_pos = src_pos;
    a.n = n;
    a.num_kv_heads = cfg_.num_kv_heads;
    a.max_ctx = cap;
    a.cos = d_cos_;
    a.sin = d_sin_;
    a.in_place = n_dst == 1 && dst_pos[0] != src_pos && overlap(dst_slots[0], dst_pos[0], src_slot, src_pos);
    a.reverse = a.in_place && dst_pos[0] > src_pos;
    return launch_kv_copy(ctx_, a, cfg_.num_layers * 2 * cfg_.num_kv_heads);
}

}  // namespace tce
