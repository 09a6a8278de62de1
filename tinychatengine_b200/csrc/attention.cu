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

}  // namespace

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
