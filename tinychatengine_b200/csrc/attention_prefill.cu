// attention_prefill.cu -- Int4llamaAttention::forward for sqlen > 1 (prompt processing; reference cuda/Int4llamaAttention.cu:116-229,
// GQA semantics non_cuda/Int4llamaAttention.cc:288-442) between the fused QKV projection and o_proj, as two kernels:
//   1. rope_kv_append: RoPE (rotate-half, llm/src/ops/RotaryPosEmb.cc:7-69; fp32 math, same expression as the decode kernel so the
//      cache bits do not depend on which path wrote them) on q in place and on k into the fp16 KV cache rows pos0..pos0+n-1; v copied.
//   2. flash prefill: one CTA per (64 query rows, head); K/V tiles of 64 cached rows staged in shared memory, S = alpha * Q K^T and
//      O += P V on mma.sync m16n8k16 (fp16 in, fp32 accumulate), causal mask by position, online softmax in fp32 -- no [n][T] score
//      tensor in HBM (the reference materialises it, plus a V transpose, per layer).
// head_dim is 128 (every Llama geometry of the reference, llm/include/model.h:71-83).
// One launch takes up to kMaxPrefillSeqs prompts with their rows concatenated (AttnPrefillArgs::seq, in row order): a token row and a
// query block find their sequence in that table and use its positions and its KV cache.  A single prompt is the one-entry table.
#include "common.cuh"
#include "kernels_attn.h"

namespace tce {
namespace {

constexpr int HD = 128;
constexpr int kQB = 64;        // query rows per CTA (16 per warp)
constexpr int kKT = 64;        // cached rows per tile
constexpr int kPitch = HD + 8; // halves; 272-byte rows: conflict-free fragment loads and 16-byte aligned ldmatrix rows

// query blocks of 64 rows of one sequence; block qb sees keys 0 .. block_keys(q, qb) - 1, a number that rises strictly with qb
__host__ __device__ inline int q_blocks(const AttnPrefillSeq &q) { return (q.n + kQB - 1) / kQB; }
TCE_DEVINL int block_keys(const AttnPrefillSeq &q, int qb) { return q.pos0 + min(q.n, (qb + 1) * kQB); }
TCE_DEVINL int blocks_upto(const AttnPrefillSeq &q, int keys) {  // blocks of q that see at most `keys` keys
    if (keys >= q.pos0 + q.n) return q_blocks(q);
    return keys < q.pos0 + kQB ? 0 : min((keys - q.pos0) / kQB, q_blocks(q) - 1);
}

// one 256-thread block per token; a warp per head slot (q heads, then kv heads), a lane per pair of adjacent dims and their rotate-half
// partners: 4-byte loads / stores, the position's cos / sin rows read as float2
__global__ void __launch_bounds__(256) rope_kv_append_kernel(const AttnPrefillArgs a) {
    const int i = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int QKV = (a.num_heads + 2 * a.num_kv_heads) * HD;
    int s = 0;
    for (int j = 1; j < a.n_seqs; j++)
        if (i >= a.seq[j].row0) s = j;
    const AttnPrefillSeq &sq = a.seq[s];
    const int pos = sq.pos0 + (i - sq.row0);
    const float2 c0 = *reinterpret_cast<const float2 *>(a.cos + (size_t)pos * HD + 2 * lane), c1 = *reinterpret_cast<const float2 *>(a.cos + (size_t)pos * HD + HD / 2 + 2 * lane);
    const float2 s0 = *reinterpret_cast<const float2 *>(a.sin + (size_t)pos * HD + 2 * lane), s1 = *reinterpret_cast<const float2 *>(a.sin + (size_t)pos * HD + HD / 2 + 2 * lane);
    for (int hh = warp; hh < a.num_heads + a.num_kv_heads; hh += 8) {
        __half *row = a.qkv + (size_t)i * QKV + (size_t)hh * HD;  // q head hh, or k head hh - H (k follows q in the fused projection)
        const float2 x0 = __half22float2(*reinterpret_cast<const __half2 *>(row + 2 * lane)), x1 = __half22float2(*reinterpret_cast<const __half2 *>(row + HD / 2 + 2 * lane));
        const __half2 r0 = __floats2half2_rn(x0.x * c0.x + (-x1.x) * s0.x, x0.y * c0.y + (-x1.y) * s0.y);
        const __half2 r1 = __floats2half2_rn(x1.x * c1.x + x0.x * s1.x, x1.y * c1.y + x0.y * s1.y);
        if (hh < a.num_heads) {
            *reinterpret_cast<__half2 *>(row + 2 * lane) = r0;
            *reinterpret_cast<__half2 *>(row + HD / 2 + 2 * lane) = r1;
        } else {
            const int kvh = hh - a.num_heads;
            __half *kc = sq.k_cache + ((size_t)kvh * a.max_ctx + pos) * HD, *vc = sq.v_cache + ((size_t)kvh * a.max_ctx + pos) * HD;
            const __half *v = a.qkv + (size_t)i * QKV + (size_t)(a.num_heads + a.num_kv_heads + kvh) * HD;
            *reinterpret_cast<__half2 *>(kc + 2 * lane) = r0;
            *reinterpret_cast<__half2 *>(kc + HD / 2 + 2 * lane) = r1;
            *reinterpret_cast<uint2 *>(vc + 4 * lane) = *reinterpret_cast<const uint2 *>(v + 4 * lane);  // 32 lanes x 4 halfs = the 128-dim row
        }
    }
}

__global__ void __launch_bounds__(128) attn_prefill_kernel(const AttnPrefillArgs a) {
    __shared__ __align__(16) __half sK[kKT * kPitch];
    __shared__ __align__(16) __half sV[kKT * kPitch];
    __shared__ int pick;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, grp = lane >> 2, qd = lane & 3;
    // longest blocks first over all sequences: CTA x takes the block of rank x in the order (keys seen descending, sequence ascending).
    // Candidate c (blocks numbered sequence by sequence) counts the blocks ahead of it; exactly one candidate has rank blockIdx.x.
    for (int c = tid; c < (int)gridDim.x; c += blockDim.x) {
        int t = 0, b = c;
        while (b >= q_blocks(a.seq[t])) b -= q_blocks(a.seq[t++]);
        const int keys = block_keys(a.seq[t], b);
        int rank = 0;
        for (int u = 0; u < a.n_seqs; u++) {
            const int upto = blocks_upto(a.seq[u], keys);
            rank += q_blocks(a.seq[u]) - upto;
            if (u < t) rank += upto - blocks_upto(a.seq[u], keys - 1);
        }
        if (rank == (int)blockIdx.x) pick = (t << 16) | b;
    }
    __syncthreads();
    const AttnPrefillSeq &sq = a.seq[pick >> 16];
    const int qb = pick & 0xffff;
    const int h = blockIdx.y, kvh = h / (a.num_heads / a.num_kv_heads);
    const int QKV = (a.num_heads + 2 * a.num_kv_heads) * HD;
    const int n = sq.n;
    const int r_lo = qb * kQB + warp * 16 + grp, r_hi = r_lo + 8;  // this thread's two query rows (index within the sequence)
    const __half *Kc = sq.k_cache + (size_t)kvh * a.max_ctx * HD, *Vc = sq.v_cache + (size_t)kvh * a.max_ctx * HD;
    __half *const qkv = a.qkv + (size_t)sq.row0 * QKV, *const out = a.out + (size_t)sq.row0 * a.num_heads * HD;

    // Q fragments (A operand, row-major 16 x 128): 8 k-steps x 4 registers, straight from the rotated projections
    uint32_t qf[8][4];
    {
        const __half *q_lo = qkv + (size_t)r_lo * QKV + (size_t)h * HD, *q_hi = qkv + (size_t)r_hi * QKV + (size_t)h * HD;
#pragma unroll
        for (int ks = 0; ks < 8; ks++) {
            const int c = ks * 16 + qd * 2;
            qf[ks][0] = r_lo < n ? *reinterpret_cast<const uint32_t *>(q_lo + c) : 0u;
            qf[ks][1] = r_hi < n ? *reinterpret_cast<const uint32_t *>(q_hi + c) : 0u;
            qf[ks][2] = r_lo < n ? *reinterpret_cast<const uint32_t *>(q_lo + c + 8) : 0u;
            qf[ks][3] = r_hi < n ? *reinterpret_cast<const uint32_t *>(q_hi + c + 8) : 0u;
        }
    }
    float o[16][4];
#pragma unroll
    for (int d = 0; d < 16; d++) o[d][0] = o[d][1] = o[d][2] = o[d][3] = 0.f;
    float m_lo = -INFINITY, m_hi = -INFINITY, l_lo = 0.f, l_hi = 0.f;
    const float sc = a.alpha * 1.4426950408889634f;  // scores kept in log2 units
    const int qpos_lo = sq.pos0 + r_lo, qpos_hi = sq.pos0 + r_hi;
    const int kv_len = block_keys(sq, qb);  // keys this block can see
    const int tiles = (kv_len + kKT - 1) / kKT;

    for (int kt = 0; kt < tiles; kt++) {
        __syncthreads();  // previous tile fully consumed
        for (int e = tid; e < kKT * (HD / 8); e += 128) {
            const int r = e / (HD / 8), c8 = e % (HD / 8);
            const int key = kt * kKT + r;
            uint4 kv4 = make_uint4(0, 0, 0, 0), vv4 = make_uint4(0, 0, 0, 0);
            if (key < kv_len) {
                kv4 = *reinterpret_cast<const uint4 *>(Kc + (size_t)key * HD + c8 * 8);
                vv4 = *reinterpret_cast<const uint4 *>(Vc + (size_t)key * HD + c8 * 8);
            }
            *reinterpret_cast<uint4 *>(sK + r * kPitch + c8 * 8) = kv4;
            *reinterpret_cast<uint4 *>(sV + r * kPitch + c8 * 8) = vv4;
        }
        __syncthreads();

        // ---- S = Q K^T for 16 rows x 64 keys
        float s[8][4];
#pragma unroll
        for (int nt = 0; nt < 8; nt++) {
            s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
            const __half *kr = sK + (nt * 8 + grp) * kPitch + qd * 2;
#pragma unroll
            for (int ks = 0; ks < 8; ks++) {
                const uint32_t b0 = *reinterpret_cast<const uint32_t *>(kr + ks * 16), b1 = *reinterpret_cast<const uint32_t *>(kr + ks * 16 + 8);
                mma_m16n8k16(s[nt], qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3], b0, b1);
            }
        }
        // ---- scale, causal mask, online softmax
        float tmax_lo = -INFINITY, tmax_hi = -INFINITY;
#pragma unroll
        for (int nt = 0; nt < 8; nt++) {
            const int key = kt * kKT + nt * 8 + qd * 2;
            s[nt][0] = (key <= qpos_lo) ? s[nt][0] * sc : -INFINITY;
            s[nt][1] = (key + 1 <= qpos_lo) ? s[nt][1] * sc : -INFINITY;
            s[nt][2] = (key <= qpos_hi) ? s[nt][2] * sc : -INFINITY;
            s[nt][3] = (key + 1 <= qpos_hi) ? s[nt][3] * sc : -INFINITY;
            tmax_lo = fmaxf(tmax_lo, fmaxf(s[nt][0], s[nt][1]));
            tmax_hi = fmaxf(tmax_hi, fmaxf(s[nt][2], s[nt][3]));
        }
        tmax_lo = fmaxf(tmax_lo, __shfl_xor_sync(0xffffffffu, tmax_lo, 1));
        tmax_lo = fmaxf(tmax_lo, __shfl_xor_sync(0xffffffffu, tmax_lo, 2));
        tmax_hi = fmaxf(tmax_hi, __shfl_xor_sync(0xffffffffu, tmax_hi, 1));
        tmax_hi = fmaxf(tmax_hi, __shfl_xor_sync(0xffffffffu, tmax_hi, 2));
        // key 0 is visible to every row, so after the first tile the running maxima are finite
        const float mn_lo = fmaxf(m_lo, tmax_lo), mn_hi = fmaxf(m_hi, tmax_hi);
        const float f_lo = exp2f(m_lo - mn_lo), f_hi = exp2f(m_hi - mn_hi);
        m_lo = mn_lo;
        m_hi = mn_hi;
        l_lo *= f_lo;
        l_hi *= f_hi;
#pragma unroll
        for (int d = 0; d < 16; d++) {
            o[d][0] *= f_lo;
            o[d][1] *= f_lo;
            o[d][2] *= f_hi;
            o[d][3] *= f_hi;
        }
        uint32_t pf[4][4];  // P as A fragments: 4 k-steps of 16 keys
#pragma unroll
        for (int nt = 0; nt < 8; nt++) {
            const float p0 = exp2f(s[nt][0] - m_lo), p1 = exp2f(s[nt][1] - m_lo), p2 = exp2f(s[nt][2] - m_hi), p3 = exp2f(s[nt][3] - m_hi);
            l_lo += p0 + p1;
            l_hi += p2 + p3;
            pf[nt >> 1][(nt & 1) * 2 + 0] = pack_half2(p0, p1);
            pf[nt >> 1][(nt & 1) * 2 + 1] = pack_half2(p2, p3);
        }
        // ---- O += P V : B fragments of V (row-major [key][dim]) through ldmatrix.trans, two 8-dim tiles per instruction
#pragma unroll
        for (int ks = 0; ks < 4; ks++) {
#pragma unroll
            for (int dp = 0; dp < 8; dp++) {
                uint32_t b0, b1, b2, b3;
                const __half *vrow = sV + (ks * 16 + (lane & 15)) * kPitch + dp * 16 + (lane >> 4) * 8;
                ldmatrix_x4_t(b0, b1, b2, b3, vrow);
                mma_m16n8k16(o[dp * 2], pf[ks][0], pf[ks][1], pf[ks][2], pf[ks][3], b0, b1);
                mma_m16n8k16(o[dp * 2 + 1], pf[ks][0], pf[ks][1], pf[ks][2], pf[ks][3], b2, b3);
            }
        }
    }
    l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 1);
    l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 2);
    l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 1);
    l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 2);
    const float inv_lo = 1.f / l_lo, inv_hi = 1.f / l_hi;
    const size_t ldo = (size_t)a.num_heads * HD;
#pragma unroll
    for (int d = 0; d < 16; d++) {
        const int c = d * 8 + qd * 2;
        if (r_lo < n) *reinterpret_cast<uint32_t *>(out + (size_t)r_lo * ldo + (size_t)h * HD + c) = pack_half2(o[d][0] * inv_lo, o[d][1] * inv_lo);
        if (r_hi < n) *reinterpret_cast<uint32_t *>(out + (size_t)r_hi * ldo + (size_t)h * HD + c) = pack_half2(o[d][2] * inv_hi, o[d][3] * inv_hi);
    }
}

}  // namespace

cudaError_t launch_attn_prefill(Ctx *ctx, const AttnPrefillArgs &a) {
    if (a.head_dim != HD || a.num_heads % a.num_kv_heads || a.n_seqs < 1 || a.n_seqs > kMaxPrefillSeqs) return cudaErrorInvalidValue;
    int rows = 0, blocks = 0;
    for (int s = 0; s < a.n_seqs; s++) {
        const AttnPrefillSeq &q = a.seq[s];
        if (q.row0 != rows || q.n < 1 || q.pos0 < 0 || q.pos0 + q.n > a.max_ctx || !q.k_cache || !q.v_cache) return cudaErrorInvalidValue;
        rows += q.n;
        blocks += q_blocks(q);
    }
    rope_kv_append_kernel<<<rows, 256, 0, ctx->stream>>>(a);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    attn_prefill_kernel<<<dim3(blocks, a.num_heads), 128, 0, ctx->stream>>>(a);
    return cudaGetLastError();
}

}  // namespace tce
