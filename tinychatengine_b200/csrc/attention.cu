// attention.cu -- per-token KV-cache attention for decode (fp16 cache, GQA aware) on sm_90a.
//
// Replaces the attention part of Int4llamaAttention::forward between qkv_proj and o_proj
// (reference llm/src/nn_modules/cuda/Int4llamaAttention.cu:128-217: shape_qkv -> RotaryPosEmb_cuda_forward ->
// 4*heads cudaMemcpyAsync KV concat -> BMM_F16T QK^T -> batch_Add mask -> check_inf -> softmax_cuda ->
// transpose V -> BMM_F16T PV -> unshape) with ONE kernel, with the GQA head mapping of the CPU module
// (llm/src/nn_modules/non_cuda/Int4llamaAttention.cc:166-184: q head i reads kv head i / (H/KVH)).
//
//  * KV cache is [KVH][max_ctx][128] fp16 per layer, appended IN PLACE at `pos` (no ping-pong copy, no V
//    transpose);
//  * grid = (KVH, ceil(max_ctx/chunk)): a CTA owns `chunk` cached positions of one KV head and serves the
//    H/KVH query heads that share it, so each cached byte is read once per token;
//  * its K and V slabs (contiguous chunk*256 B each) are pulled into shared memory by two TMA bulk copies
//    issued up front -- the whole cache of the layer is in flight at once, the kernel is HBM-bound;
//  * fp32 RoPE / scores / softmax statistics / PV accumulation; split results are merged flash-decoding
//    style by the last CTA of each KV head to arrive (fixed order, deterministic).
#include "attention_impl.cuh"
#include "kernels.h"

namespace tce {
namespace {

using namespace attn;

template <int NREP>
__global__ void __launch_bounds__(kAttnThreads, 1) attn_decode_kernel(const __grid_constant__ AttnDecodeArgs a) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint64_t *bar = reinterpret_cast<uint64_t *>(smem + smem_bytes(NREP, a.chunk));
    int *flag = reinterpret_cast<int *>(bar + 2);
    const int tid = threadIdx.x;
    if (tid == 0) {
        mbar_init(&bar[0], 1);
        mbar_init(&bar[1], 1);
        mbar_fence_init();
    }
    __syncthreads();
    pdl_launch_dependents();
    pdl_wait();  // qkv of this token comes from the previous kernel; the cache was written by earlier steps
    uint32_t parity = 0;
    attn_item<NREP>(a, smem, bar, flag, parity, blockIdx.x, blockIdx.y, tid, *a.pos, [] { __syncthreads(); });
}

// grid (KVH, nsplit, batch): the work item of the single-sequence kernel on sequence blockIdx.z's rows, slot and position
template <int NREP>
__global__ void __launch_bounds__(kAttnThreads, 1) attn_decode_batch_kernel(const __grid_constant__ AttnBatchArgs b) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint64_t *bar = reinterpret_cast<uint64_t *>(smem + smem_bytes(NREP, b.base.chunk));
    int *flag = reinterpret_cast<int *>(bar + 2);
    const int tid = threadIdx.x, seq = blockIdx.z;
    if (tid == 0) {
        mbar_init(&bar[0], 1);
        mbar_init(&bar[1], 1);
        mbar_fence_init();
    }
    __syncthreads();
    pdl_launch_dependents();
    pdl_wait();  // the request records and q|k|v come from the previous kernels of the step
    const int *r = b.req + 4 * seq;
    if (r[3] == 0) return;  // refused entry (uniform over the CTA)
    AttnDecodeArgs a = b.base;
    a.qkv += (size_t)seq * b.qkv_stride;
    a.out += (size_t)seq * b.out_stride;
    __half *slot = b.slots[r[2]];
    a.k_cache = slot + b.k_off;
    a.v_cache = slot + b.v_off;
    a.ws += (size_t)seq * a.num_heads * a.nsplit_max * (HD + 2);
    a.counters += (size_t)seq * a.num_kv_heads;
    uint32_t parity = 0;
    attn_item<NREP>(a, smem, bar, flag, parity, blockIdx.x, blockIdx.y, tid, r[1], [] { __syncthreads(); });
}

size_t attn_smem_bytes(int nrep, int chunk) { return smem_bytes(nrep, chunk) + 2 * sizeof(uint64_t) + 16; }

template <int NREP>
cudaError_t launch(Ctx *ctx, const AttnDecodeArgs &a, bool pdl) {
    const size_t smem = attn_smem_bytes(NREP, a.chunk);
    static DeviceOnce attr_once;
    if (attr_once.pending(ctx->device)) {
        cudaError_t e = cudaFuncSetAttribute(attn_decode_kernel<NREP>, cudaFuncAttributeMaxDynamicSharedMemorySize, ctx->smem_optin);
        if (e != cudaSuccess) return e;
        attr_once.done(ctx->device);
    }
    if ((int)smem > ctx->smem_optin) return cudaErrorInvalidConfiguration;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(a.num_kv_heads, a.nsplit_max);
    cfg.blockDim = dim3(kAttnThreads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = ctx->stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, attn_decode_kernel<NREP>, a);
}

template <int NREP>
cudaError_t launch_batch(Ctx *ctx, const AttnBatchArgs &b, int batch, bool pdl) {
    const size_t smem = attn_smem_bytes(NREP, b.base.chunk);
    static DeviceOnce attr_once;
    if (attr_once.pending(ctx->device)) {
        cudaError_t e = cudaFuncSetAttribute(attn_decode_batch_kernel<NREP>, cudaFuncAttributeMaxDynamicSharedMemorySize, ctx->smem_optin);
        if (e != cudaSuccess) return e;
        attr_once.done(ctx->device);
    }
    if ((int)smem > ctx->smem_optin) return cudaErrorInvalidConfiguration;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(b.base.num_kv_heads, b.base.nsplit_max, batch);
    cfg.blockDim = dim3(kAttnThreads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = ctx->stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, attn_decode_batch_kernel<NREP>, b);
}

}  // namespace

size_t attn_batch_ws_floats(int num_heads, int max_ctx, int chunk) {
    if (chunk <= 0) chunk = 128;
    return (size_t)num_heads * ((max_ctx + chunk - 1) / chunk) * (HD + 2);
}

cudaError_t launch_attn_decode_batch(Ctx *ctx, AttnBatchArgs b, int batch, bool pdl) {
    AttnDecodeArgs &a = b.base;
    if (a.head_dim != HD) return cudaErrorNotSupported;
    if (a.num_heads % a.num_kv_heads || batch < 1) return cudaErrorInvalidValue;
    if (a.chunk <= 0) a.chunk = 128;
    a.nsplit_max = (a.max_ctx + a.chunk - 1) / a.chunk;
    // per sequence: its own partial records and split counters, in the caller's workspace
    if (!a.ws || !a.counters || (size_t)batch * attn_batch_ws_floats(a.num_heads, a.max_ctx, a.chunk) > b.ws_floats ||
        (size_t)batch * a.num_kv_heads > b.n_counters)
        return cudaErrorInvalidValue;
    switch (a.num_heads / a.num_kv_heads) {
        case 1: return launch_batch<1>(ctx, b, batch, pdl);
        case 2: return launch_batch<2>(ctx, b, batch, pdl);
        case 4: return launch_batch<4>(ctx, b, batch, pdl);
        case 8: return launch_batch<8>(ctx, b, batch, pdl);
        default: return cudaErrorNotSupported;
    }
}

cudaError_t launch_attn_decode(Ctx *ctx, AttnDecodeArgs a, bool pdl) {
    if (a.head_dim != HD) return cudaErrorNotSupported;
    if (a.num_heads % a.num_kv_heads) return cudaErrorInvalidValue;
    const int nrep = a.num_heads / a.num_kv_heads;
    if (a.chunk <= 0) a.chunk = 128;
    a.nsplit_max = (a.max_ctx + a.chunk - 1) / a.chunk;
    const size_t need = (size_t)a.num_heads * a.nsplit_max * (HD + 2) * sizeof(float);
    if (need > ctx->attn_ws_bytes || a.num_kv_heads > 1024) return cudaErrorInvalidValue;
    a.ws = ctx->attn_ws;
    a.counters = ctx->attn_counters;
    switch (nrep) {
        case 1: return launch<1>(ctx, a, pdl);
        case 2: return launch<2>(ctx, a, pdl);
        case 4: return launch<4>(ctx, a, pdl);
        case 8: return launch<8>(ctx, a, pdl);
        default: return cudaErrorNotSupported;
    }
}

}  // namespace tce
