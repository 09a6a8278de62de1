// gemm_w4_tc.cu -- W4A16 prefill GEMM with the int4 unpack fused into the tensor-core tile pipeline (the slot
// MatmulOperator::gemm_forward_cuda, kernels/matmul.h:142-145, declared and never defined by the reference).
//
//   C[M][N] = X[M][K] (fp16) * dequant(W)[N][K]^T,   W = QM_CUDA int4 (uint32 [N][K/8], 8 sequential nibbles per word; fp16 scale and
//   4-bit zero per 128-k group), fp32 accumulation in the wgmma register fragment.
//
// Nothing but the packed nibbles ever leaves HBM for the weights (0.5 B per weight + scales, against 4.5 B per weight for an expansion
// pass to an fp16 scratch followed by a plain GEMM).  The kernel is the FUSED instantiation of gemm_tc.cuh:
//   warp 8 = TMA producer (128 x 64 fp16 activation tile + 128 rows x 32 bytes of nibbles per k-block, 5-deep ring); warps 9-12 = dequant
//   (one thread per weight row, the values w4_expand_kernel / the reference's gemv_cuda.cu:181-184 produce, 3-deep operand ring);
//   warps 0-7 = two consumer warpgroups (wgmma from both rings, then fp16 store or fp32 residual accumulate from the fragment).
// Persistent, one CTA per SM, tiles walked m-fastest so that the CTAs running concurrently share weight tiles in L2.
#include "gemm_tc.cuh"
#include "kernels.h"

namespace tce {

namespace {
constexpr int kBN = 128;       // weight rows per tile
constexpr int kLdStages = 5;   // ring of {activation tile, packed weight tile}
}  // namespace

// shared by the single-CTA and the CTA-pair launch (gemm_tc2.cu)
cudaError_t fill_w4_gemm_args(tc::GemmArgs &a, const __half *X, long long ldx, const uint32_t *w, const uint32_t *zeros, const __half *scales, void *C, long long ldc,
                              int M, int N, int K) {
    if (M < 1 || N < 1 || K < 128 || (K % 128) || (ldx % 8)) return cudaErrorInvalidValue;
    cudaError_t e = tc::encode_kmajor(&a.tmA, X, false, M, K, ldx, tc::kBlockM);
    if (e != cudaSuccess) return e;
    e = tc::encode_w4_packed(&a.tmB, w, N, K, kBN / 2);
    if (e != cudaSuccess) return e;
    a.scales = scales;
    a.zeros = zeros;
    a.zeros_w = zeros_width(K, kW4Group);
    a.sf_w = a.zeros_w * 8;
    a.M = M;
    a.N = N;
    a.k_blocks = K / 64;
    a.C = C;
    a.ldc = ldc;
    return cudaSuccess;
}

// C[M][N] (fp16, or fp32 accumulated into when add_f32) = X[M][K] fp16 * dequant(W)^T; W rows [N], K % 128 == 0, ldx % 8 == 0.
cudaError_t launch_gemm_w4_tc(Ctx *ctx, const __half *X, long long ldx, const uint32_t *w, const uint32_t *zeros, const __half *scales, void *C,
                              long long ldc, int M, int N, int K, int add_f32) {
    tc::GemmArgs a = {};
    cudaError_t e = fill_w4_gemm_args(a, X, ldx, w, zeros, scales, C, ldc, M, N, K);
    if (e != cudaSuccess) return e;
    if (add_f32) return tc::launch_wg<kBN, kLdStages, false, true, 1, tc::EpiAddF32>(ctx, a);
    return tc::launch_wg<kBN, kLdStages, false, true, 1, tc::EpiHalf>(ctx, a);
}

}  // namespace tce
