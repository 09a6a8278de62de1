// kernels_w8a8.h -- launch interface of the W8A8 family (internal).
#pragma once
#include "kernels.h"

namespace tce {

enum W8Variant : int {
    W8_BIAS8_O8 = 0,    // int8_ref_matmul              (matmul_ref_int8.cc:11-35)
    W8_NOBIAS_O8 = 1,   // int8_ref_matmul_nobias[_batch] (:37-87)
    W8_BIASF_OF32 = 2,  // int8_ref_matmul_bfp32_ofp32  (:89-111)
    W8_NOBIAS_OF32 = 3  // int8_ref_matmul_nobias_ofp32[_batch] (:113-159)
};

struct W8A8Args {
    const int8_t *A;      // [M][K]
    const int8_t *B;      // [N][K]  (batch: [M][N][K])
    const int8_t *bias8;  // [N] or null
    const float *biasf;   // [N] or null
    int8_t *C8;           // [M][N]
    float *Cf;            // [M][N]
    int M, N, K;
    float alpha, beta;
    int q_min, q_max;
    int variant;          // W8Variant
    int batch;            // 1: row i of A multiplies slab B[i]
};

cudaError_t launch_w8a8_dp4a(Ctx *ctx, const W8A8Args &a);
cudaError_t launch_w8a8_tc(Ctx *ctx, const W8A8Args &a);  // wgmma s8 x s8, non-batched, K % 128 == 0

// int8 attention core of Int8OPTAttention::forward (llm/src/nn_modules/Int8OPTAttention.cc:183-284)
struct OptAttnParams {
    const int8_t *q8, *k8, *v8;        // [sqlen][H*hd]
    const int8_t *past_k, *past_v;     // [H][past][hd], head stride past_hs (null when past == 0)
    long long past_hs;
    int8_t *final_k, *final_v;         // [H][tgz][hd], head stride final_hs; == past_* with equal stride -> in-place cache
    long long final_hs;
    const float *mask;                 // [sqlen][tgz] or null (causal)
    float qk_alpha, pv_alpha;
    int sqlen, past, H, hd;
    int8_t *out;                       // [sqlen][H*hd]
};
cudaError_t launch_opt_int8_attention(Ctx *ctx, const OptAttnParams &p);

}  // namespace tce
