// elementwise.cu -- the small ops either side of the hot path (SURVEY.md 8(f).1): embedding gather, RMSNorm,
// argmax.  RMSNorm / residual add / SiLU*mul of the decode block are fused into the GEMV kernels
// (w4a16_gemv.cu); the standalone versions here serve the op-level API and the tests.
#include "common.cuh"
#include "kernels_attn.h"

namespace tce {
namespace {

// grid (blocks per row, batch): entry b of req = {token, position, slot}
__global__ void embedding_batch_kernel(const __half *__restrict__ table, const int *__restrict__ req, float *__restrict__ resid, int E, int rows,
                                       int max_ctx, int n_slots, int *__restrict__ safe) {
    pdl_launch_dependents();
    pdl_wait();
    const int b = blockIdx.y;
    const int tok = req[3 * b], pos = req[3 * b + 1], slot = req[3 * b + 2];
    const bool ok = tok >= 0 && tok < rows && pos >= 0 && pos < max_ctx && slot >= 0 && slot < n_slots;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        safe[4 * b] = ok ? tok : 0;
        safe[4 * b + 1] = ok ? pos : 0;
        safe[4 * b + 2] = ok ? slot : 0;
        safe[4 * b + 3] = ok ? 1 : 0;
    }
    const __half2 *row = reinterpret_cast<const __half2 *>(table + (size_t)(ok ? tok : 0) * E);
    float2 *dst = reinterpret_cast<float2 *>(resid + (size_t)b * E);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < E / 2; i += gridDim.x * blockDim.x) dst[i] = __half22float2(row[i]);
}

// one CTA per row; ties resolve to the lowest index
__global__ void __launch_bounds__(1024) argmax_rows_kernel(const float *__restrict__ logits, int n, int *__restrict__ out) {
    __shared__ float sval[32];
    __shared__ int sidx[32];
    pdl_launch_dependents();
    pdl_wait();
    const float *x = logits + (size_t)blockIdx.x * n;
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const float v = x[i];
        if (v > best) {  // indices rise within a thread: the first maximum stays
            best = v;
            bi = i;
        }
    }
    auto combine = [](float &bv, int &bidx, float ov, int oidx) {
        if (ov > bv || (ov == bv && oidx < bidx)) {
            bv = ov;
            bidx = oidx;
        }
    };
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) combine(best, bi, __shfl_xor_sync(0xffffffffu, best, o), __shfl_xor_sync(0xffffffffu, bi, o));
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) {
        sval[warp] = best;
        sidx[warp] = bi;
    }
    __syncthreads();
    if (warp == 0) {
        best = (lane < (int)(blockDim.x >> 5)) ? sval[lane] : -INFINITY;
        bi = (lane < (int)(blockDim.x >> 5)) ? sidx[lane] : 0x7fffffff;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) combine(best, bi, __shfl_xor_sync(0xffffffffu, best, o), __shfl_xor_sync(0xffffffffu, bi, o));
        if (lane == 0) out[blockIdx.x] = bi == 0x7fffffff ? 0 : bi;
    }
}

__global__ void rmsnorm_f16_kernel(const __half *__restrict__ x, const float *__restrict__ gamma, __half *__restrict__ y, int dim, float eps) {
    __shared__ float sred[32];
    const __half *xr = x + (size_t)blockIdx.x * dim;
    __half *yr = y + (size_t)blockIdx.x * dim;
    float ss = 0.f;
    for (int i = threadIdx.x; i < dim; i += blockDim.x) {
        const float v = __half2float(xr[i]);
        ss += v * v;
    }
    ss = warp_sum(ss);
    if ((threadIdx.x & 31) == 0) sred[threadIdx.x >> 5] = ss;
    __syncthreads();
    float tot = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); w++) tot += sred[w];
    const float inv = rsqrtf(tot / (float)dim + eps);
    for (int i = threadIdx.x; i < dim; i += blockDim.x) yr[i] = __float2half((__half2float(xr[i]) * inv) * gamma[i]);
}

// LayerNormQ::forward (llm/src/ops/LayerNormQ.cc:12-52): fp32 row -> int8 row, eps 1e-5.  The reference sums the row serially in fp32
// (mean, then squared deviations), and the int8 result depends on those sums to the last bit near rounding ties, so the two reductions
// are done by ONE thread in the reference's order (the loads are independent of the add chain and pipeline); the normalisation of the
// row is spread over the block, with the reference's operation order and no FMA contraction.  One block per row.
__global__ void layernorm_q_kernel(const float *__restrict__ x, const float *__restrict__ weight, const float *__restrict__ bias, int8_t *__restrict__ out,
                                   int dim) {
    extern __shared__ __align__(16) float srow[];  // [dim] + 2
    const float *xr = x + (size_t)blockIdx.x * dim;
    for (int i = threadIdx.x; i < dim; i += blockDim.x) srow[i] = xr[i];
    __syncthreads();
    if (threadIdx.x == 0) {
        // 16-byte loads in front of the dependent add chains: the chain (4 cycles per element) is what remains
        float mean = 0.f;
        int k = 0;
        for (; k + 4 <= dim; k += 4) {
            const float4 v = *reinterpret_cast<const float4 *>(srow + k);
            mean = __fadd_rn(mean, v.x);
            mean = __fadd_rn(mean, v.y);
            mean = __fadd_rn(mean, v.z);
            mean = __fadd_rn(mean, v.w);
        }
        for (; k < dim; k++) mean = __fadd_rn(mean, srow[k]);
        mean = __fdiv_rn(mean, (float)dim);
        float sq = 0.f;
        for (k = 0; k + 4 <= dim; k += 4) {
            const float4 v = *reinterpret_cast<const float4 *>(srow + k);
            const float d0 = __fsub_rn(v.x, mean), d1 = __fsub_rn(v.y, mean), d2 = __fsub_rn(v.z, mean), d3 = __fsub_rn(v.w, mean);
            sq = __fadd_rn(sq, __fmul_rn(d0, d0));
            sq = __fadd_rn(sq, __fmul_rn(d1, d1));
            sq = __fadd_rn(sq, __fmul_rn(d2, d2));
            sq = __fadd_rn(sq, __fmul_rn(d3, d3));
        }
        for (; k < dim; k++) {
            const float d = __fsub_rn(srow[k], mean);
            sq = __fadd_rn(sq, __fmul_rn(d, d));
        }
        const float var = __fdiv_rn(sq, (float)dim);
        srow[dim] = mean;
        srow[dim + 1] = __fsqrt_rn(__fadd_rn(var, 0.00001f));
    }
    __syncthreads();
    const float mean = srow[dim], sd = srow[dim + 1];
    int8_t *orow = out + (size_t)blockIdx.x * dim;
    for (int i = threadIdx.x; i < dim; i += blockDim.x) {
        const float fp = __fadd_rn(__fmul_rn(__fdiv_rn(__fsub_rn(srow[i], mean), sd), weight[i]), bias[i]);
        orow[i] = (int8_t)(int)roundf(fp);  // std::round: half away from zero, then the implementation's float -> int8 conversion
    }
}

// fp32 residual add of the OPT decoder layer (Int8OPTDecoderLayer::add, llm/src/nn_modules/Int8OPTDecoderLayer.cc:10-22)
__global__ void add_f32_kernel(const float *__restrict__ a, const float *__restrict__ b, float *__restrict__ out, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) out[i] = __fadd_rn(a[i], b[i]);
}

// ---- row-wise versions for prompt processing (n tokens at once)
__global__ void embedding_rows_kernel(const __half *__restrict__ table, const int *__restrict__ tokens, float *__restrict__ resid, int E) {
    const __half2 *row = reinterpret_cast<const __half2 *>(table + (size_t)tokens[blockIdx.x] * E);
    float2 *dst = reinterpret_cast<float2 *>(resid + (size_t)blockIdx.x * E);
    for (int i = threadIdx.x; i < E / 2; i += blockDim.x) dst[i] = __half22float2(row[i]);
}

// one 256-thread block per row; the row stays in registers between the two passes (dim <= 256 * 4 * kRmsVec), 16-byte loads, 8-byte stores
constexpr int kRmsVec = 8;  // float4 per thread: rows up to 8192 channels
__global__ void __launch_bounds__(256) rmsnorm_rows_f32_kernel(const float *__restrict__ x, const float *__restrict__ gamma, __half *__restrict__ y, int dim, float eps) {
    __shared__ float sred[8];
    const float4 *xr = reinterpret_cast<const float4 *>(x + (size_t)blockIdx.x * dim);
    const float4 *gr = reinterpret_cast<const float4 *>(gamma);
    uint2 *yr = reinterpret_cast<uint2 *>(y + (size_t)blockIdx.x * dim);
    const int nv = dim >> 2;
    float4 v[kRmsVec];
    float ss = 0.f;
#pragma unroll
    for (int k = 0; k < kRmsVec; k++) {
        const int i = threadIdx.x + k * 256;
        v[k] = i < nv ? xr[i] : make_float4(0.f, 0.f, 0.f, 0.f);
        ss += v[k].x * v[k].x + v[k].y * v[k].y + v[k].z * v[k].z + v[k].w * v[k].w;
    }
    ss = warp_sum(ss);
    if ((threadIdx.x & 31) == 0) sred[threadIdx.x >> 5] = ss;
    __syncthreads();
    float tot = 0.f;
#pragma unroll
    for (int w = 0; w < 8; w++) tot += sred[w];
    const float inv = rsqrtf(tot / (float)dim + eps);
#pragma unroll
    for (int k = 0; k < kRmsVec; k++) {
        const int i = threadIdx.x + k * 256;
        if (i < nv) {
            const float4 g = gr[i];
            yr[i] = make_uint2(pack_half2((v[k].x * inv) * g.x, (v[k].y * inv) * g.y), pack_half2((v[k].z * inv) * g.z, (v[k].w * inv) * g.w));
        }
    }
}
// general shapes (dim not a multiple of 4, or longer than the register tile)
__global__ void rmsnorm_rows_f32_generic_kernel(const float *__restrict__ x, const float *__restrict__ gamma, __half *__restrict__ y, int dim, float eps) {
    __shared__ float sred[32];
    const float *xr = x + (size_t)blockIdx.x * dim;
    __half *yr = y + (size_t)blockIdx.x * dim;
    float ss = 0.f;
    for (int i = threadIdx.x; i < dim; i += blockDim.x) ss += xr[i] * xr[i];
    ss = warp_sum(ss);
    if ((threadIdx.x & 31) == 0) sred[threadIdx.x >> 5] = ss;
    __syncthreads();
    float tot = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); w++) tot += sred[w];
    const float inv = rsqrtf(tot / (float)dim + eps);
    for (int i = threadIdx.x; i < dim; i += blockDim.x) yr[i] = __float2half((xr[i] * inv) * gamma[i]);
}

cudaError_t launch_cfg(cudaLaunchConfig_t &cfg, cudaLaunchAttribute *attr, dim3 grid, dim3 block, cudaStream_t s, bool pdl) {
    cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = 0;
    cfg.stream = s;
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl ? 1 : 0;
    return cudaSuccess;
}

}  // namespace

cudaError_t launch_embedding_batch(Ctx *ctx, const __half *table, const int *req, float *resid, int E, int batch, int rows, int max_ctx, int n_slots,
                                   int *safe, bool pdl) {
    cudaLaunchConfig_t cfg;
    cudaLaunchAttribute attr[1];
    launch_cfg(cfg, attr, dim3(4, batch), dim3(256), ctx->stream, pdl);
    return cudaLaunchKernelEx(&cfg, embedding_batch_kernel, table, req, resid, E, rows, max_ctx, n_slots, safe);
}

cudaError_t launch_argmax_rows(Ctx *ctx, const float *logits, int rows, int n, int *out, bool pdl) {
    cudaLaunchConfig_t cfg;
    cudaLaunchAttribute attr[1];
    launch_cfg(cfg, attr, dim3(rows), dim3(1024), ctx->stream, pdl);
    return cudaLaunchKernelEx(&cfg, argmax_rows_kernel, logits, n, out);
}

cudaError_t launch_embedding_rows(Ctx *ctx, const __half *table, const int *tokens, float *resid, int n, int E) {
    embedding_rows_kernel<<<n, 256, 0, ctx->stream>>>(table, tokens, resid, E);
    return cudaGetLastError();
}
cudaError_t launch_rmsnorm_rows_f32(Ctx *ctx, const float *x, const float *gamma, __half *y, int rows, int dim, float eps) {
    if ((dim & 3) == 0 && dim <= 256 * 4 * kRmsVec && !(((uintptr_t)x | (uintptr_t)gamma) & 15) && !((uintptr_t)y & 7))
        rmsnorm_rows_f32_kernel<<<rows, 256, 0, ctx->stream>>>(x, gamma, y, dim, eps);
    else
        rmsnorm_rows_f32_generic_kernel<<<rows, 256, 0, ctx->stream>>>(x, gamma, y, dim, eps);
    return cudaGetLastError();
}
cudaError_t launch_layernorm_q(Ctx *ctx, const float *x, const float *weight, const float *bias, int8_t *out, int rows, int dim) {
    const size_t smem = (size_t)(dim + 2) * sizeof(float);
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(layernorm_q_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
    }
    layernorm_q_kernel<<<rows, 128, smem, ctx->stream>>>(x, weight, bias, out, dim);
    return cudaGetLastError();
}
cudaError_t launch_add_f32(Ctx *ctx, const float *a, const float *b, float *out, long long n) {
    const long long nb = (n + 255) / 256;
    add_f32_kernel<<<(unsigned)(nb < 2368 ? nb : 2368), 256, 0, ctx->stream>>>(a, b, out, n);
    return cudaGetLastError();
}

cudaError_t launch_rmsnorm_f16(Ctx *ctx, const __half *x, const float *gamma, __half *y, int rows, int dim, float eps) {
    rmsnorm_f16_kernel<<<rows, 256, 0, ctx->stream>>>(x, gamma, y, dim, eps);
    return cudaGetLastError();
}

}  // namespace tce
