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
    static constexpr bool kSilu = true, kRowStats = false;
    TCE_DEVINL static void apply(const GemmArgs &a, int row, int col, float g0, float g1, float u0, float u1) {
        __half *dst = reinterpret_cast<__half *>(a.C) + (size_t)row * a.ldc + col;  // F % 128 == 0, ldc % 8 == 0: both columns exist, 4-byte aligned
        *reinterpret_cast<uint32_t *>(dst) = pack_half2((g0 / (1.f + __expf(-g0))) * u0, (g1 / (1.f + __expf(-g1))) * u1);
    }
};

// folds record (om, os, oid) into (m, s, id): the larger maximum wins, ties go to the lowest id.  An empty record has m = -inf, s = 0.
TCE_DEVINL void lm_combine(float &m, float &s, int &id, float om, float os, int oid) {
    const float mn = fmaxf(m, om);
    s = (m == mn ? s : s * __expf(m - mn)) + (om == mn ? os : os * __expf(om - mn));
    if (om > m || (om == m && oid < id)) id = oid;
    m = mn;
}

// lm_head scoring: each 128-column half of a tile becomes one LmStat per row, so a row's records do not depend on the tile width (nor on how
// many rows share the call).  The 4 lanes of a quad hold the 128 columns of a row (32 each); each reduces its own columns in rising order
// (max and arg-max first, then the sum of exp(x - max)), then the quad combines with two xor shuffles in a fixed order.
struct EpiRowStats {
    static constexpr bool kSilu = false, kRowStats = true;
    TCE_DEVINL static void half(const GemmArgs &a, const float (&v)[64], int row0, int c0, int cq) {
        if (c0 >= a.N) return;  // the whole half lies past the chunk (uniform over the CTA)
#pragma unroll
        for (int r = 0; r < 2; r++) {
            const int row = row0 + 8 * r;
            float m = -INFINITY;
            int id = 0x7fffffff;
#pragma unroll
            for (int i = 0; i < 16; i++)
#pragma unroll
                for (int e = 0; e < 2; e++) {
                    const int col = c0 + 8 * i + cq + e;
                    const float x = v[4 * i + 2 * r + e];
                    if (col < a.N && x > m) {  // columns rise: the first maximum stays
                        m = x;
                        id = col;
                    }
                }
            const int t = row < a.M ? a.target[row] - a.col0 - c0 : -1;  // the target's column within this half, if it is here
            float s = 0.f, tv = 0.f;
            bool hit = false;
#pragma unroll
            for (int i = 0; i < 16; i++)
#pragma unroll
                for (int e = 0; e < 2; e++) {
                    const int col = c0 + 8 * i + cq + e;
                    const float x = v[4 * i + 2 * r + e];
                    if (col < a.N) s += __expf(x - m);
                    if (8 * i + cq + e == t) {
                        tv = x;
                        hit = true;
                    }
                }
#pragma unroll
            for (int o = 1; o <= 2; o <<= 1) {
                const float om = __shfl_xor_sync(0xffffffffu, m, o), os = __shfl_xor_sync(0xffffffffu, s, o);
                const int oid = __shfl_xor_sync(0xffffffffu, id, o);
                lm_combine(m, s, id, om, os, oid);
            }
            if (row < a.M) {
                if (cq == 0) a.stats[(size_t)row * a.stats_ld + c0 / 128] = LmStat{m, s, a.col0 + id, 0};
                if (hit) a.tgt[row] = tv;
                if (a.C) {
                    float *dst = reinterpret_cast<float *>(a.C) + (size_t)row * a.ldc;  // C = logits + col0; ldc and col0 even
#pragma unroll
                    for (int i = 0; i < 16; i++) {
                        const int col = c0 + 8 * i + cq;
                        if (col + 1 < a.N) *reinterpret_cast<float2 *>(dst + col) = make_float2(v[4 * i + 2 * r], v[4 * i + 2 * r + 1]);
                        else if (col < a.N) dst[col] = v[4 * i + 2 * r];
                    }
                }
            }
        }
    }
};

// one warp per row: lane l folds records l, l + 32, ... in column order, the warp combines in a fixed butterfly, and lane 0 folds the result
// into the row's running state (earlier chunks first)
__global__ void __launch_bounds__(256) lm_stats_merge_kernel(const LmStat *__restrict__ stats, int stats_ld, int n_rec, int rows, int first, int last,
                                                             LmStat *__restrict__ state, const int *__restrict__ target, const float *__restrict__ tgt,
                                                             float *__restrict__ logprob, int *__restrict__ greedy, float *__restrict__ greedy_logprob) {
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= rows) return;
    float m = -INFINITY, s = 0.f;
    int id = 0x7fffffff;
    for (int r = lane; r < n_rec; r += 32) {
        const LmStat q = stats[(size_t)row * stats_ld + r];
        lm_combine(m, s, id, q.m, q.s, q.id);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float om = __shfl_xor_sync(0xffffffffu, m, o), os = __shfl_xor_sync(0xffffffffu, s, o);
        const int oid = __shfl_xor_sync(0xffffffffu, id, o);
        lm_combine(m, s, id, om, os, oid);
    }
    if (lane != 0) return;
    if (!first) {
        LmStat p = state[row];
        lm_combine(p.m, p.s, p.id, m, s, id);
        m = p.m;
        s = p.s;
        id = p.id;
    }
    if (!last) {
        state[row] = LmStat{m, s, id, 0};
        return;
    }
    const float lse = m + logf(s);
    logprob[row] = target[row] >= 0 ? tgt[row] - lse : __int_as_float(0x7fc00000);
    greedy[row] = id;
    greedy_logprob[row] = m - lse;
}

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

// 128-column tiles only: the 256-wide tile holds 128 accumulators per thread and spills with the reduction at the 168-register cap of
// 384 threads per SM
cudaError_t launch_gemm_f16_pair_stats(Ctx *ctx, const __half *X, long long ldx, const __half *W, long long ldw, int M, int N, int K, int col0, LmStat *stats,
                                       int stats_ld, const int *target, float *tgt, float *logits, long long ld_logits) {
    if (M < 1 || N < 1 || K < 64 || (K % 64) || (ldx % 8) || (ldw % 8) || col0 < 0 || (col0 % 128) || !stats || stats_ld < (N + 127) / 128 || !target ||
        !tgt || (logits && (ld_logits % 2)))
        return cudaErrorInvalidValue;
    GemmArgs a = {};
    cudaError_t e = fill_f16(a, X, ldx, W, ldw, N, 64, M, K);
    if (e != cudaSuccess) return e;
    a.N = N;
    a.C = logits ? logits + col0 : nullptr;
    a.ldc = ld_logits;
    a.stats = stats;
    a.stats_ld = stats_ld;
    a.col0 = col0;
    a.target = target;
    a.tgt = tgt;
    return tc::launch_wg<128, 6, false, 2, EpiRowStats>(ctx, a);
}

cudaError_t launch_lm_stats_merge(Ctx *ctx, const LmStat *stats, int stats_ld, int n_rec, int rows, bool first, bool last, LmStat *state, const int *target,
                                  const float *tgt, float *logprob, int *greedy, float *greedy_logprob) {
    if (rows < 1 || n_rec < 1 || n_rec > stats_ld) return cudaErrorInvalidValue;
    lm_stats_merge_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, ctx->stream>>>(stats, stats_ld, n_rec, rows, first ? 1 : 0, last ? 1 : 0, state, target, tgt,
                                                                                logprob, greedy, greedy_logprob);
    return cudaGetLastError();
}

}  // namespace tce
