// w8a8.cu -- W8A8 (SmoothQuant) INT8 x INT8 -> INT32 linear / batched-matmul family on sm_90a.
//
// Replaces the eight MatmulOperator::mat_mul_accelerator_int8_fast_* methods
// (reference kernels/ref/matmul_ref_int8.cc:11-192, AVX: kernels/avx/matmul_avx_int8.cc).  Integer
// accumulation is order independent, and the float epilogue is evaluated with explicit round-to-nearest
// multiplies/adds in the reference's order (no FMA contraction), so int8 outputs are BIT-EXACT with the
// reference's `kernels/ref` semantics:
//     acc = sum_k A[i,k] * B[j,k]                                   (B stored [N][K] = torch [out,in])
//     int8 out : clamp(round_half_away((float)acc*alpha [+ (float)bias8[j]*beta]), q_min, q_max)
//     fp32 out : (float)acc*alpha [+ biasf[j]]
// `batch` flavours: row i of A uses its own B slab B[i][N][K] (per-head QK^T / PV at sqlen 1).
//
// This file holds the DP4A kernel: one warp per output column, 128-bit loads, up to 8 activation rows per
// pass -- HBM-bound for the M<=8 decode case.  Large-M prefill goes to the wgmma s8 x s8 GEMM (gemm_tc.cu).
#include "common.cuh"
#include "kernels.h"
#include "kernels_w8a8.h"

namespace tce {
namespace {

constexpr int kWarps = 8;
constexpr int MT = 8;

TCE_DEVINL int dp4a_s8(uint32_t a, uint32_t b, int c) {
    int r;
    asm("dp4a.s32.s32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
    return r;
}

TCE_DEVINL void epilogue(const W8A8Args &a, int i, int j, int acc) {
    const float v = __fmul_rn((float)acc, a.alpha);
    const size_t o = (size_t)i * a.N + j;
    switch (a.variant) {
        case W8_BIAS8_O8: {
            const float bb = __fmul_rn((float)a.bias8[j], a.beta);
            int q = (int)roundf(__fadd_rn(v, bb));
            q = max(q, a.q_min);
            q = min(q, a.q_max);
            a.C8[o] = (int8_t)q;
            break;
        }
        case W8_NOBIAS_O8: {
            int q = (int)roundf(v);
            q = max(q, a.q_min);
            q = min(q, a.q_max);
            a.C8[o] = (int8_t)q;
            break;
        }
        case W8_BIASF_OF32: a.Cf[o] = __fadd_rn(v, a.biasf[j]); break;
        default: a.Cf[o] = v; break;
    }
}

__global__ void __launch_bounds__(kWarps * 32) w8a8_dp4a_kernel(const W8A8Args a) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int j = blockIdx.x * kWarps + warp;
    if (j >= a.N) return;
    const int i0 = blockIdx.y * (a.batch ? 1 : MT);
    const int rows = a.batch ? 1 : min(MT, a.M - i0);
    const int8_t *Brow = a.B + (a.batch ? (size_t)i0 * a.N * a.K : 0) + (size_t)j * a.K;
    const int8_t *A0 = a.A + (size_t)i0 * a.K;
    int acc[MT];
#pragma unroll
    for (int r = 0; r < MT; r++) acc[r] = 0;
    if ((a.K & 15) == 0) {
        const uint4 *Bv = reinterpret_cast<const uint4 *>(Brow);
        for (int c = lane; c < a.K / 16; c += 32) {
            const uint4 b = ldg_nc_u4(Bv + c);
#pragma unroll
            for (int r = 0; r < MT; r++) {
                if (r < rows) {
                    const uint4 x = *reinterpret_cast<const uint4 *>(A0 + (size_t)r * a.K + c * 16);
                    acc[r] = dp4a_s8(x.x, b.x, acc[r]);
                    acc[r] = dp4a_s8(x.y, b.y, acc[r]);
                    acc[r] = dp4a_s8(x.z, b.z, acc[r]);
                    acc[r] = dp4a_s8(x.w, b.w, acc[r]);
                }
            }
        }
    } else {
        for (int k = lane; k < a.K; k += 32) {
            const int b = Brow[k];
#pragma unroll
            for (int r = 0; r < MT; r++)
                if (r < rows) acc[r] += (int)A0[(size_t)r * a.K + k] * b;
        }
    }
#pragma unroll
    for (int r = 0; r < MT; r++) {
        int v = acc[r];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0 && r < rows) epilogue(a, i0 + r, j, v);
    }
}

// Decode flavour (M <= 4 rows, one B for all rows, K % 16 == 0, K >= 512): HBM-bound weight streaming.  Persistent warps walk the output
// columns interleaved (neighbouring warps stream neighbouring weight rows), the activation rows sit in shared memory, and every
// lane keeps UNR 128-bit weight loads in flight (the simple kernel above has one load per warp in flight and short-lived warps).  Integer sums in any order are exact, the epilogue is the shared one.
template <int MR, int UNR>
__global__ void __launch_bounds__(kWarps * 32) w8a8_stream_kernel(const W8A8Args a) {
    extern __shared__ __align__(16) uint8_t sA[];  // [MR][K]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int chunks = a.K / 16;  // 16-byte chunks per row
    for (int i = threadIdx.x; i < MR * chunks; i += blockDim.x) {
        const int r = i / chunks, c = i % chunks;
        reinterpret_cast<uint4 *>(sA)[i] = r < a.M ? reinterpret_cast<const uint4 *>(a.A + (size_t)r * a.K)[c] : make_uint4(0, 0, 0, 0);
    }
    __syncthreads();
    const int total_warps = gridDim.x * kWarps;
    for (int j = blockIdx.x * kWarps + warp; j < a.N; j += total_warps) {
        const uint4 *Bv = reinterpret_cast<const uint4 *>(a.B + (size_t)j * a.K);
        int acc[MR];
#pragma unroll
        for (int r = 0; r < MR; r++) acc[r] = 0;
        for (int c0 = lane; c0 < chunks; c0 += 32 * UNR) {
            uint4 b[UNR];
#pragma unroll
            for (int u = 0; u < UNR; u++) b[u] = (c0 + 32 * u < chunks) ? ldg_nc_u4(Bv + c0 + 32 * u) : make_uint4(0, 0, 0, 0);  // ragged tail: zero weights
#pragma unroll
            for (int u = 0; u < UNR; u++) {
#pragma unroll
                for (int r = 0; r < MR; r++) {
                    const uint4 x = reinterpret_cast<const uint4 *>(sA + (size_t)r * a.K)[min(c0 + 32 * u, chunks - 1)];
                    acc[r] = dp4a_s8(x.x, b[u].x, acc[r]);
                    acc[r] = dp4a_s8(x.y, b[u].y, acc[r]);
                    acc[r] = dp4a_s8(x.z, b[u].z, acc[r]);
                    acc[r] = dp4a_s8(x.w, b[u].w, acc[r]);
                }
            }
        }
#pragma unroll
        for (int r = 0; r < MR; r++) {
            int v = acc[r];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            if (lane == 0 && r < a.M) epilogue(a, r, j, v);
        }
    }
}

template <int MR, int UNR>
cudaError_t launch_stream(Ctx *ctx, const W8A8Args &a) {
    const size_t smem = (size_t)MR * a.K;
    auto kern = w8a8_stream_kernel<MR, UNR>;
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
    }
    int grid = ctx->num_sms * 4;  // 32 warps per SM: 32 x 32 lanes x UNR x 16 B in flight
    const int need = (a.N + kWarps - 1) / kWarps;
    if (grid > need) grid = need;
    kern<<<grid, kWarps * 32, smem, ctx->stream>>>(a);
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_w8a8_dp4a(Ctx *ctx, const W8A8Args &a) {
    if (a.M <= 0 || a.N <= 0 || a.K <= 0) return cudaErrorInvalidValue;
    if (!a.batch && a.M <= 4 && (size_t)4 * a.K <= (size_t)ctx->smem_optin / 2 && !(((uintptr_t)a.A | (uintptr_t)a.B) & 15)) {
        if (a.K % 16 == 0 && a.K >= 2048) return a.M == 1 ? launch_stream<1, 4>(ctx, a) : launch_stream<4, 4>(ctx, a);
        if (a.K % 16 == 0 && a.K >= 512) return a.M == 1 ? launch_stream<1, 1>(ctx, a) : launch_stream<4, 1>(ctx, a);
    }
    dim3 grid((a.N + kWarps - 1) / kWarps, a.batch ? a.M : (a.M + MT - 1) / MT);
    w8a8_dp4a_kernel<<<grid, kWarps * 32, 0, ctx->stream>>>(a);
    return cudaGetLastError();
}

}  // namespace tce
