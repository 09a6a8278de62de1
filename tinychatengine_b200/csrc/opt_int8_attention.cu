// opt_int8_attention.cu -- the int8 attention core of Int8OPTAttention::forward (llm/src/nn_modules/Int8OPTAttention.cc:183-284)
// between the q/k/v projections and out_proj, as two kernels:
//   1. kv_concat: final_k/final_v[h][0..tgz) = past rows (skipped when the cache is updated in place) ++ this call's rows
//      (the reference's shape() + cat_past_keys_values memcpy, :207-243).
//   2. attn_rows: one CTA per (head, query row): scores (dp4a, exact int32) * qk_alpha + mask -> fp32 softmax -> P8 =
//      round(p*127) -> P8 x V (exact int32) -> clamp(round(acc * pv_alpha)) -> unshape.  Replaces BMM_S8T_S8N_F32T, batch_Add,
//      softmax, the int8 cast loop, transpose_1_2idx, BMM_S8T_S8N_S8T and unshape (:245-275) with no intermediate in HBM.
// Bit-exactness with the CPU reference is the contract: integer parts are exact in any order; the float parts keep the
// reference's evaluation order (serial float sum over the row; p = float(double(e) / (double(sum) + 1e-10))), and exp() is
// evaluated in double and rounded to float, which is what a correctly-rounded expf returns.  The running max of every row
// is seeded with element [0] of the score tensor (softmax.cc:13); the module runs softmax in place, so that element is the
// raw score for row (head 0, query 0) and the PROBABILITY p[0][0][0] for every later row.  Reproduced literally: the CTA of row (0,0)
// publishes p[0][0][0] behind an epoch flag; every other row folds it into its running maximum once its own scores are computed.
#include "common.cuh"
#include "kernels_w8a8.h"

namespace tce {
namespace {

constexpr int kThreads = 128;

__global__ void opt_kv_concat_kernel(const int8_t *__restrict__ k8, const int8_t *__restrict__ v8, const int8_t *__restrict__ past_k,
                                     const int8_t *__restrict__ past_v, long long past_hs, int8_t *__restrict__ final_k, int8_t *__restrict__ final_v,
                                     long long final_hs, int sqlen, int past, int H, int hd, int copy_past) {
    const int h = blockIdx.y;
    const int row0 = copy_past ? 0 : past, tgz = past + sqlen;
    const long long n = (long long)(tgz - row0) * hd;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
        const int t = row0 + (int)(e / hd), d = (int)(e % hd);
        int8_t kk, vv;
        if (t < past) {
            kk = past_k[h * past_hs + (long long)t * hd + d];
            vv = past_v[h * past_hs + (long long)t * hd + d];
        } else {
            kk = k8[(size_t)(t - past) * H * hd + h * hd + d];
            vv = v8[(size_t)(t - past) * H * hd + h * hd + d];
        }
        final_k[h * final_hs + (long long)t * hd + d] = kk;
        final_v[h * final_hs + (long long)t * hd + d] = vv;
    }
}

TCE_DEVINL int dot_s8(const int8_t *__restrict__ a, const int8_t *__restrict__ b, int n) {  // n % 4 == 0, both 4-byte aligned
    int acc = 0;
    for (int d = 0; d < n; d += 4) acc = __dp4a(*(const int *)(a + d), *(const int *)(b + d), acc);
    return acc;
}
// 16-byte flavour (n % 16 == 0, both 16-byte aligned): all loads of a key row are in flight before the first dp4a
TCE_DEVINL int dot_s8_v16(const int8_t *__restrict__ a, const int8_t *__restrict__ b, int n) {
    int acc = 0;
#pragma unroll 8
    for (int d = 0; d < n; d += 16) {
        const int4 x = *reinterpret_cast<const int4 *>(a + d), y = *reinterpret_cast<const int4 *>(b + d);
        acc = __dp4a(x.x, y.x, acc);
        acc = __dp4a(x.y, y.y, acc);
        acc = __dp4a(x.z, y.z, acc);
        acc = __dp4a(x.w, y.w, acc);
    }
    return acc;
}

// dynamic smem: float s[tgz] | int8 p8[tgz rounded to 16] | int8 q[hd rounded to 16] | int acc[hd]
// One launch for all rows: CTA (0, 0) is row (head 0, query 0); it publishes p[0][0][0] (value, fence, epoch flag) and every other CTA takes it into
// its running maximum after it has computed its own scores (max is order independent, so the late arrival of the seed changes nothing).
__global__ void __launch_bounds__(kThreads) opt_attn_rows_kernel(const int8_t *__restrict__ q8, const int8_t *__restrict__ final_k,
                                                                const int8_t *__restrict__ final_v, long long hs, const float *__restrict__ mask,
                                                                float qk_alpha, float pv_alpha, int sqlen, int past, int H, int hd,
                                                                int8_t *__restrict__ out, float *seed_ws, unsigned *seed_flag, unsigned epoch, int vec16) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int h = blockIdx.x, i = blockIdx.y, tgz = past + sqlen, tid = threadIdx.x;
    const bool first_row = (h == 0 && i == 0);
    float *s = (float *)smem_raw;
    int8_t *p8 = (int8_t *)(s + ((tgz + 3) & ~3));  // keeps p8 / q / acc 16-byte aligned
    int8_t *q = p8 + ((tgz + 15) & ~15);
    int *acc = (int *)(q + ((hd + 15) & ~15));
    __shared__ float red[kThreads / 32];
    __shared__ float s_sum, s_seed;

    for (int d = tid; d < hd; d += kThreads) {
        q[d] = q8[(size_t)i * H * hd + h * hd + d];
        acc[d] = 0;
    }
    __syncthreads();
    const int8_t *K = final_k + h * hs, *V = final_v + h * hs;
    const float neg = -3.402823466e38f;
    // softmax.cc:13: row (0,0) is seeded with its own first score (a member of the row: plain max), later rows with p[0][0][0]
    float mx = -INFINITY;
    // built-in causal mask (mask == nullptr): keys behind the query get -FLT_MAX added, their exp() is exactly 0, p8 is 0 and adding 0 to the serial
    // row sum changes no bit of it -- they are skipped altogether (half of the work of a prompt pass).  An explicit mask tensor is applied in full.
    const int jmax = mask ? tgz : min(tgz, past + i + 1);
    for (int j = tid; j < jmax; j += kThreads) {
        const int a = vec16 ? dot_s8_v16(q, K + (size_t)j * hd, hd) : dot_s8(q, K + (size_t)j * hd, hd);
        const float m = mask ? mask[(size_t)i * tgz + j] : (j > past + i ? neg : 0.f);
        const float v = __fadd_rn(__fmul_rn((float)a, qk_alpha), m);
        s[j] = v;
        mx = fmaxf(mx, v);
    }
    mx = warp_max(mx);
    if ((tid & 31) == 0) red[tid >> 5] = mx;
    if (!first_row && tid == 0) {  // the seed of this call: spin on the epoch flag, then read the value
        const long long t0 = clock64();
        while (*reinterpret_cast<volatile unsigned *>(seed_flag) != epoch) {
            if (clock64() - t0 > 20000000000LL) __trap();
        }
        __threadfence();
        s_seed = *reinterpret_cast<volatile float *>(seed_ws);
    }
    __syncthreads();
    mx = first_row ? red[0] : fmaxf(red[0], s_seed);
    for (int w = 1; w < kThreads / 32; w++) mx = fmaxf(mx, red[w]);
    for (int j = tid; j < jmax; j += kThreads) s[j] = (float)exp((double)__fsub_rn(s[j], mx));
    __syncthreads();
    if (tid == 0) {  // the reference's serial float sum (order matters for bit-exactness)
        float sum = 0.f;
        int j = 0;
        for (; j + 4 <= jmax; j += 4) {  // 16-byte loads in front of the dependent add chain (s is 16-byte aligned)
            const float4 v = *reinterpret_cast<const float4 *>(s + j);
            sum = __fadd_rn(sum, v.x);
            sum = __fadd_rn(sum, v.y);
            sum = __fadd_rn(sum, v.z);
            sum = __fadd_rn(sum, v.w);
        }
        for (; j < jmax; j++) sum = __fadd_rn(sum, s[j]);
        s_sum = sum;
    }
    __syncthreads();
    const double denom = (double)s_sum + 1e-10;
    for (int j = tid; j < jmax; j += kThreads) {
        const float p = (float)((double)s[j] / denom);
        p8[j] = (int8_t)(int)roundf(__fmul_rn(p, 127.f));
        if (first_row && j == 0) {
            *seed_ws = p;
            __threadfence();
            atomicExch(seed_flag, epoch);
        }
    }
    __syncthreads();
    if (vec16) {
        // P8 x V: thread (g, c) walks rows t = g, g + G, ... and owns 16 consecutive d's (one 16-byte load per row); four rows in flight
        const int lanes = hd / 16, G = kThreads / lanes;
        const int c = tid % lanes, g = tid / lanes;
        if (g < G) {
            int a16[16];
#pragma unroll
            for (int e = 0; e < 16; e++) a16[e] = 0;
            auto fma16 = [&](int pp, const int4 &v) {
                const int w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    a16[4 * k + 0] += pp * (int)(int8_t)(w[k] & 0xff);
                    a16[4 * k + 1] += pp * (int)(int8_t)((w[k] >> 8) & 0xff);
                    a16[4 * k + 2] += pp * (int)(int8_t)((w[k] >> 16) & 0xff);
                    a16[4 * k + 3] += pp * (int)(int8_t)((w[k] >> 24) & 0xff);
                }
            };
            int t = g;
            for (; t + 3 * G < jmax; t += 4 * G) {
                const int4 v0 = *reinterpret_cast<const int4 *>(V + (size_t)t * hd + c * 16), v1 = *reinterpret_cast<const int4 *>(V + (size_t)(t + G) * hd + c * 16);
                const int4 v2 = *reinterpret_cast<const int4 *>(V + (size_t)(t + 2 * G) * hd + c * 16), v3 = *reinterpret_cast<const int4 *>(V + (size_t)(t + 3 * G) * hd + c * 16);
                fma16(p8[t], v0);
                fma16(p8[t + G], v1);
                fma16(p8[t + 2 * G], v2);
                fma16(p8[t + 3 * G], v3);
            }
            for (; t < jmax; t += G) fma16(p8[t], *reinterpret_cast<const int4 *>(V + (size_t)t * hd + c * 16));
#pragma unroll
            for (int e = 0; e < 16; e++) atomicAdd(&acc[c * 16 + e], a16[e]);
        }
    } else {
        // P8 x V: thread (g, c) walks rows t = g, g+G, ... and owns 4 consecutive d's
        const int lanes = hd / 4, G = kThreads / lanes;  // hd % 4 == 0, lanes <= kThreads checked by the launcher
        const int c = tid % lanes, g = tid / lanes;
        if (g < G) {
            int a0 = 0, a1 = 0, a2 = 0, a3 = 0;
            for (int t = g; t < jmax; t += G) {
                const int p = p8[t];
                const int v4 = *(const int *)(V + (size_t)t * hd + c * 4);
                a0 += p * (int)(int8_t)(v4 & 0xff);
                a1 += p * (int)(int8_t)((v4 >> 8) & 0xff);
                a2 += p * (int)(int8_t)((v4 >> 16) & 0xff);
                a3 += p * (int)(int8_t)((v4 >> 24) & 0xff);
            }
            atomicAdd(&acc[c * 4 + 0], a0);
            atomicAdd(&acc[c * 4 + 1], a1);
            atomicAdd(&acc[c * 4 + 2], a2);
            atomicAdd(&acc[c * 4 + 3], a3);
        }
    }
    __syncthreads();
    for (int d = tid; d < hd; d += kThreads) {
        int r = (int)roundf(__fmul_rn((float)acc[d], pv_alpha));
        r = max(-128, min(127, r));
        out[(size_t)i * H * hd + h * hd + d] = (int8_t)r;
    }
}

}  // namespace

cudaError_t launch_opt_int8_attention(Ctx *ctx, const OptAttnParams &p) {
    const int tgz = p.past + p.sqlen;
    const bool in_place = (p.past_k == p.final_k && p.past_v == p.final_v && p.past_hs == p.final_hs);
    const int copy_past = (p.past > 0 && !in_place) ? 1 : 0;
    const long long n = (long long)(copy_past ? tgz : p.sqlen) * p.hd;
    const long long nb = (n + 255) / 256;
    dim3 g1((unsigned)(nb < 1024 ? nb : 1024), p.H);
    opt_kv_concat_kernel<<<g1, 256, 0, ctx->stream>>>(p.k8, p.v8, p.past_k, p.past_v, p.past_hs, p.final_k, p.final_v, p.final_hs, p.sqlen, p.past, p.H,
                                                       p.hd, copy_past);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    const size_t smem = (size_t)((tgz + 3) & ~3) * 4 + ((tgz + 15) & ~15) + ((p.hd + 15) & ~15) + (size_t)p.hd * 4;
    if (smem > 48 * 1024) {
        if (smem > (size_t)ctx->smem_optin) return cudaErrorInvalidValue;
        e = cudaFuncSetAttribute(opt_attn_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
    }
    // [0] the seed value p[0][0][0] of this call, [1] the epoch flag that says it is there (same-stream ordering makes the reuse safe)
    float *seed_ws = ctx->opt_seed;
    unsigned *seed_flag = reinterpret_cast<unsigned *>(ctx->opt_seed) + 1;
    const unsigned epoch = ++ctx->attn_seed_epoch;
    const int vec16 = (p.hd % 16 == 0) && (p.final_hs % 16 == 0) && !(((uintptr_t)p.final_k | (uintptr_t)p.final_v) & 15) ? 1 : 0;
    dim3 g2(p.H, p.sqlen);  // block (0, 0) = row (head 0, query 0) is in the first wave: the rows that wait for its seed cannot starve it
    opt_attn_rows_kernel<<<g2, kThreads, smem, ctx->stream>>>(p.q8, p.final_k, p.final_v, p.final_hs, p.mask, p.qk_alpha, p.pv_alpha, p.sqlen, p.past, p.H,
                                                             p.hd, p.out, seed_ws, seed_flag, epoch, vec16);
    return cudaGetLastError();
}

}  // namespace tce
