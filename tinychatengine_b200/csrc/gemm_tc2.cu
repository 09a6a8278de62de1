// gemm_tc2.cu -- the prefill GEMM on CTA pairs:  C[M][N] = X[M][K] (fp16) * W[N][K]^T, the CL = 2 instantiations of gemm_tc.cuh.
//
// Two CTAs of a cluster own two vertically adjacent 128-row tiles of the same N block; each fetches half of the weight rows of every 64-k
// block and multicasts them to both (see gemm_tc.cuh, CL = 2).  W is the fp16 expansion of the int4 weights (w4_expand_kernel, gemm_tc.cu).
// SiLU variant: W = [gate (F rows); up (F rows)]; tile columns 0..127 are 128 channels of gate (fetched by CTA 0), 128..255 the same
// channels of up (CTA 1), so a thread holds both accumulators of a channel and writes act = SiLU(gate) * up.
#include "gemm_tc.cuh"
#include "kernels.h"

namespace tce {
namespace {

using tc::GemmArgs;

struct EpiSiluMul {  // act[M][F] = SiLU(gate) * up (SiLuMul_half, llm/src/nn_modules/cuda/Int4llamaDecoderLayer.cu:12-30; fp32 math)
    static constexpr bool kSilu = true;
    TCE_DEVINL static void apply(const GemmArgs &a, int row, int col, float g0, float g1, float u0, float u1) {
        __half *dst = reinterpret_cast<__half *>(a.C) + (size_t)row * a.ldc + col;  // F % 128 == 0, ldc % 8 == 0: both columns exist, 4-byte aligned
        *reinterpret_cast<uint32_t *>(dst) = pack_half2((g0 / (1.f + __expf(-g0))) * u0, (g1 / (1.f + __expf(-g1))) * u1);
    }
};

cudaError_t fill_f16(GemmArgs &a, const __half *X, long long ldx, const __half *W, long long ldw, long long w_rows, int box_rows, int M, int K) {
    cudaError_t e = tc::encode_kmajor(&a.tmA, X, false, M, K, ldx, tc::kBlockM);
    if (e != cudaSuccess) return e;
    e = tc::encode_kmajor(&a.tmB, W, false, w_rows, K, ldw, box_rows);
    if (e != cudaSuccess) return e;
    a.M = M;
    a.k_blocks = K / 64;
    return cudaSuccess;
}

}  // namespace

// W fp16 [N][K] (ldw elements between rows)
cudaError_t launch_gemm_f16_pair(Ctx *ctx, const __half *X, long long ldx, const __half *W, long long ldw, void *C, long long ldc, int M, int N, int K, int add_f32) {
    if (M < 1 || N < 1 || K < 64 || (K % 64) || (ldx % 8) || (ldw % 8)) return cudaErrorInvalidValue;
    const int pn = tc::pick_block_n((M + 2 * tc::kBlockM - 1) / (2 * tc::kBlockM), N, ctx->num_sms / 2);  // 256-row blocks over the clusters
    GemmArgs a = {};
    cudaError_t e = fill_f16(a, X, ldx, W, ldw, N, pn / 2, M, K);
    if (e != cudaSuccess) return e;
    a.N = N;
    a.C = C;
    a.ldc = ldc;
    if (pn == 256) {
        if (add_f32) return tc::launch_wg<256, 4, false, 2, tc::EpiAddF32>(ctx, a);
        return tc::launch_wg<256, 4, false, 2, tc::EpiHalf>(ctx, a);
    }
    if (add_f32) return tc::launch_wg<128, 6, false, 2, tc::EpiAddF32>(ctx, a);
    return tc::launch_wg<128, 6, false, 2, tc::EpiHalf>(ctx, a);
}

// act[M][F] = SiLU(X Wg^T) * (X Wu^T), W = fp16 [2F][K] with the gate rows first; F % 128 == 0, ldc % 8 == 0
cudaError_t launch_gemm_f16_pair_silu(Ctx *ctx, const __half *X, long long ldx, const __half *W, long long ldw, __half *act, long long ldc, int M, int F, int K) {
    if (M < 1 || F < 128 || (F % 128) || K < 64 || (K % 64) || (ldx % 8) || (ldw % 8) || (ldc % 8)) return cudaErrorInvalidValue;
    GemmArgs a = {};
    cudaError_t e = fill_f16(a, X, ldx, W, ldw, 2LL * F, 128, M, K);
    if (e != cudaSuccess) return e;
    a.N = F;
    a.silu_F = F;
    a.C = act;
    a.ldc = ldc;
    return tc::launch_wg<256, 4, false, 2, EpiSiluMul>(ctx, a);
}

}  // namespace tce
