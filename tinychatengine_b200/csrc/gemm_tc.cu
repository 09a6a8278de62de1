// gemm_tc.cu -- instantiations of the wgmma GEMM for the two large-M slots of the path:
//   * W4A16 prefill (MatmulOperator::gemm_forward_cuda, declared-but-undefined in the reference, kernels/matmul.h:142-145): the
//     QM_CUDA int4 weights are expanded once per call to fp16 ((q - z) * s, one rounding) into an L2-resident scratch by a
//     bandwidth-bound kernel, then C = X * W16^T runs on the tensor cores with fp32 accumulation.  Expanding once per call
//     instead of once per M tile keeps the CUDA-core dequant work at OC*IC instead of OC*IC*ceil(M/128).
//   * W8A8 (mat_mul_accelerator_int8_fast_2x2_32unroll* at M >= 16, kernels/ref/matmul_ref_int8.cc:11-159): wgmma s8 x s8 with
//     int32 accumulation is exact, the float epilogue keeps the reference's evaluation order -> bit-identical int8 / fp32 outputs.
#include "gemm_tc.cuh"
#include "kernels.h"
#include "kernels_w8a8.h"

namespace tce {
namespace {

using tc::EpiAddF32;
using tc::EpiHalf;
using tc::GemmArgs;

// ------------------------------------------------------------------------------------------------ epilogues
template <int VARIANT>
struct EpiW8 {  // int32 accumulator -> the four W8A8 epilogues (same float op order as w8a8.cu / kernels/ref)
    static constexpr bool kSilu = false;
    TCE_DEVINL static void apply(const GemmArgs &a, int row, int col, int v0, int v1) {
        const size_t o = (size_t)row * a.ldc + col;
        const int v[2] = {v0, v1};
#pragma unroll
        for (int i = 0; i < 2; i++) {
            if (col + i >= a.N) break;
            float f = __fmul_rn((float)v[i], a.alpha);
            if constexpr (VARIANT == W8_BIAS8_O8 || VARIANT == W8_NOBIAS_O8) {
                if constexpr (VARIANT == W8_BIAS8_O8) f = __fadd_rn(f, __fmul_rn((float)a.bias8[col + i], a.beta));
                int qv = (int)roundf(f);
                qv = min(max(qv, a.q_min), a.q_max);
                reinterpret_cast<int8_t *>(a.C)[o + i] = (int8_t)qv;
            } else {
                if constexpr (VARIANT == W8_BIASF_OF32) f = __fadd_rn(f, a.biasf[col + i]);
                reinterpret_cast<float *>(a.C)[o + i] = f;
            }
        }
    }
};

// ------------------------------------------------------------------------------------------------ W4 -> fp16 expansion
// one thread per 32-bit word (8 sequential nibbles, weights 8c..8c+7 of row o) -> one 16-byte store
__global__ void w4_expand_kernel(const uint32_t *__restrict__ w, const uint32_t *__restrict__ zeros, const __half *__restrict__ scales, __half *__restrict__ out,
                                 int OC, int words_per_row, int zeros_w, int sf_w) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)OC * words_per_row) return;
    const int o = (int)(idx / words_per_row), c = (int)(idx % words_per_row);
    const int g = c >> 4;  // 16 words = 128 weights per group
    const uint32_t z = (zeros[(size_t)o * zeros_w + (g >> 3)] >> (4 * (g & 7))) & 0xFu;
    const __half s = scales[(size_t)o * sf_w + g];
    const __half2 s2 = __half2half2(s);
    const uint32_t zmagic = 0x64006400u | z | (z << 16);  // (1024 + z) in both halves
    const uint32_t word = w[idx];
    uint32_t r[4];
#pragma unroll
    for (int p = 0; p < 4; p++) {
        const uint32_t x = word >> (8 * p);
        const uint32_t qmagic = 0x64006400u | (x & 0xFu) | ((x & 0xF0u) << 12);  // (1024 + q) for weights 2p, 2p+1
        const __half2 d = __hsub2(*reinterpret_cast<const __half2 *>(&qmagic), *reinterpret_cast<const __half2 *>(&zmagic));  // exact
        const __half2 m = __hmul2(d, s2);                                                                                     // one rounding
        r[p] = *reinterpret_cast<const uint32_t *>(&m);
    }
    reinterpret_cast<uint4 *>(out)[idx] = make_uint4(r[0], r[1], r[2], r[3]);
}

// ------------------------------------------------------------------------------------------------ host side
template <int BLOCK_N, int STAGES, bool I8, class Epi>
cudaError_t launch(Ctx *ctx, GemmArgs &a, const void *A, long long lda, const void *B, long long ldb, long long K) {
    cudaError_t e = tc::encode_kmajor(&a.tmA, A, I8, a.M, K, lda, tc::kBlockM);
    if (e != cudaSuccess) return e;
    e = tc::encode_kmajor(&a.tmB, B, I8, a.N, K, ldb, BLOCK_N / 2);
    if (e != cudaSuccess) return e;
    a.k_blocks = (int)(K * (I8 ? 1 : 2) / tc::kAtomBytes);
    return tc::launch_wg<BLOCK_N, STAGES, I8, false, 1, Epi>(ctx, a);
}

// Tile width by wave quantisation: a persistent grid of `sms` CTAs needs ceil(tiles / sms) rounds, each costing ~BLOCK_N (the MMA
// time of one tile) times a penalty for the narrower tile (the 128-row A tile is re-read once per N block); the 1.12 is a guess, not measured on H100.
int pick_block_n(int M, int N, int sms) {
    const long long mb = (M + 127) / 128;
    const int bn[2] = {256, 128};
    const double pen[2] = {1.00, 1.12};
    int best = 256;
    double best_cost = 1e30;
    for (int i = 0; i < 2; i++) {
        const long long tiles = mb * ((N + bn[i] - 1) / bn[i]);
        const double cost = (double)((tiles + sms - 1) / sms) * bn[i] * pen[i];
        if (cost < best_cost) {
            best_cost = cost;
            best = bn[i];
        }
    }
    return best;
}

template <class Epi, bool I8>
cudaError_t dispatch(Ctx *ctx, GemmArgs &a, const void *A, long long lda, const void *B, long long ldb, long long K) {
    if (pick_block_n(a.M, a.N, ctx->num_sms) == 256) return launch<256, 4, I8, Epi>(ctx, a, A, lda, B, ldb, K);
    return launch<128, 6, I8, Epi>(ctx, a, A, lda, B, ldb, K);
}

}  // namespace

cudaError_t w4_scratch_reserve(Ctx *ctx, size_t elems) {
    if (ctx->w16_scratch_elems >= elems) return cudaSuccess;
    if (ctx->w16_scratch) {  // rare: grows to the largest weight matrix seen (cudaFree synchronises)
        cudaError_t e = cudaFree(ctx->w16_scratch);
        ctx->w16_scratch = nullptr;
        ctx->w16_scratch_elems = 0;
        if (e != cudaSuccess) return e;
    }
    cudaError_t e = cudaMalloc(&ctx->w16_scratch, elems * sizeof(__half));
    if (e == cudaSuccess) ctx->w16_scratch_elems = elems;
    return e;
}

cudaError_t launch_w4_expand(Ctx *ctx, const uint32_t *w, const uint32_t *zeros, const __half *scales, __half *out, int OC, int IC) {
    const int wpr = IC / 8, zw = zeros_width(IC, kW4Group);
    const long long n = (long long)OC * wpr;
    w4_expand_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(w, zeros, scales, out, OC, wpr, zw, zw * 8);
    return cudaGetLastError();
}

// C[M][N] = A[M][K] fp16 * B[N][K]^T fp16, fp32 accumulation; C is fp16 (stored) or, with add_f32, fp32 (accumulated into).  K % 64 == 0, pointers 16-byte aligned, lda/ldb % 8 == 0.
cudaError_t launch_gemm_f16_tc(Ctx *ctx, const __half *A, long long lda, const __half *B, long long ldb, void *C, long long ldc, int M, int N, int K,
                               int add_f32) {
    if (M < 1 || N < 1 || K < 64 || (K % 64) || (lda % 8) || (ldb % 8)) return cudaErrorInvalidValue;
    GemmArgs a = {};
    a.M = M;
    a.N = N;
    a.C = C;
    a.ldc = ldc;
    if (add_f32) return dispatch<EpiAddF32, false>(ctx, a, A, lda, B, ldb, K);
    return dispatch<EpiHalf, false>(ctx, a, A, lda, B, ldb, K);
}

// the four non-batched W8A8 variants on the int8 tensor cores.  K % 128 == 0 (one swizzle atom), pointers 16-byte aligned.
cudaError_t launch_w8a8_tc(Ctx *ctx, const W8A8Args &w) {
    if (w.batch || w.M < 1 || w.N < 1 || w.K < 128 || (w.K % 128)) return cudaErrorInvalidValue;
    GemmArgs a = {};
    a.M = w.M;
    a.N = w.N;
    a.ldc = w.N;
    a.bias8 = w.bias8;
    a.biasf = w.biasf;
    a.alpha = w.alpha;
    a.beta = w.beta;
    a.q_min = w.q_min;
    a.q_max = w.q_max;
    switch (w.variant) {
        case W8_BIAS8_O8: a.C = w.C8; return dispatch<EpiW8<W8_BIAS8_O8>, true>(ctx, a, w.A, w.K, w.B, w.K, w.K);
        case W8_NOBIAS_O8: a.C = w.C8; return dispatch<EpiW8<W8_NOBIAS_O8>, true>(ctx, a, w.A, w.K, w.B, w.K, w.K);
        case W8_BIASF_OF32: a.C = w.Cf; return dispatch<EpiW8<W8_BIASF_OF32>, true>(ctx, a, w.A, w.K, w.B, w.K, w.K);
        case W8_NOBIAS_OF32: a.C = w.Cf; return dispatch<EpiW8<W8_NOBIAS_OF32>, true>(ctx, a, w.A, w.K, w.B, w.K, w.K);
    }
    return cudaErrorInvalidValue;
}

}  // namespace tce
