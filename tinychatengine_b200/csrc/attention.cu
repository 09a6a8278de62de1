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
//  * grid = (KVH, ceil(max_ctx/chunk), batch): a CTA owns `chunk` cached positions of one KV head of one sequence and
//    serves the H/KVH query heads that share it, so each cached byte is read once per token;
//  * its K and V rows are pulled into padded shared rows by 16-byte cp.async copies issued up front -- the whole cache of
//    the layer is in flight at once, the kernel is HBM-bound;
//  * the H/KVH query heads are the (up to 8) columns of one MMA tile: scores and P.V run on mma.sync m16n8k16 with fp16
//    operands (q * alpha, K, P, V) and fp32 accumulation; a scalar version of the two products cost ~6 of the kernel's ~18 us;
//  * fp32 RoPE / softmax statistics; split results are merged flash-decoding style through global partial records by the
//    last CTA of each KV head to arrive (fixed order, deterministic).
// A thread-block-cluster flavour -- one cluster of 8 / 16 CTAs per KV head, partials merged over distributed shared memory --
// was implemented and measured: 2.2 us per layer SLOWER (cluster co-scheduling + two cluster barriers), so it was removed.
#include "common.cuh"
#include "kernels_attn.h"

namespace tce {
namespace {

constexpr int HD = 128;  // head_dim (every Llama config in llm/include/model.h:71-83)
constexpr int kAttnThreads = 256;
constexpr int kPitch = HD + 8;  // halves per K/V/Q row in shared memory: 272-byte rows keep ldmatrix and fragment loads conflict free

int chunk_rows(int chunk) { return chunk > 0 ? chunk : 128; }  // cached positions per CTA; attn_chunk <= 0 selects the default

inline __host__ __device__ int rows16(int chunk) { return (chunk + 15) & ~15; }
inline __host__ __device__ int p_floats(int chunk) { return rows16(chunk) > HD + 8 ? rows16(chunk) : HD + 8; }
// shared memory of one CTA; the word after it elects the last split
inline __host__ __device__ size_t smem_bytes(int nrep, int chunk) {
    size_t b = (size_t)2 * rows16(chunk) * kPitch * 2;  // K, V slabs (padded rows)
    b += (size_t)8 * kPitch * 2;                         // q, fp16, 8 head rows (rows >= nrep are zero)
    b += (size_t)nrep * p_floats(chunk) * 4;             // scores fp32
    b += (size_t)nrep * rows16(chunk) * 2;               // probabilities fp16
    b += (size_t)nrep * HD * 4;                          // o
    b += (size_t)2 * nrep * 16 * 4;                      // stats [2][nrep][16]
    return (b + 15) & ~(size_t)15;
}

// one (kv head, split, sequence) work item per CTA
template <int NREP>
__global__ void __launch_bounds__(kAttnThreads, 1) attn_decode_kernel(const __grid_constant__ AttnDecodeArgs a) {
    static_assert(NREP <= 8, "the query heads of one KV head ride in the 8 MMA columns");
    extern __shared__ __align__(128) uint8_t smem[];
    const int chunk = a.chunk;
    const int R16 = rows16(chunk);
    __half *sK = reinterpret_cast<__half *>(smem);                       // [R16][kPitch]
    __half *sV = sK + (size_t)R16 * kPitch;                              // [R16][kPitch]
    __half *sQ = sV + (size_t)R16 * kPitch;                              // [8][kPitch] rotated * alpha, rows >= NREP zero
    float *sP = reinterpret_cast<float *>(sQ + 8 * kPitch);              // [NREP][p_floats] scores
    __half *sPh = reinterpret_cast<__half *>(sP + NREP * p_floats(chunk));  // [NREP][R16] probabilities
    float *sO = reinterpret_cast<float *>(sPh + NREP * R16);             // [NREP][HD] unnormalised output of this split
    float *sStat = sO + NREP * HD;                                       // [NREP][16] max | [NREP][16] sum
    int *flag = reinterpret_cast<int *>(smem + smem_bytes(NREP, chunk));
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, qd = lane & 3;
    const int kvh = blockIdx.x, split = blockIdx.y, seq = blockIdx.z;
    pdl_launch_dependents();
    pdl_wait();  // q|k|v (and the request records) come from the previous kernels; the cache was written by earlier steps

    // ---- this sequence's position and K / V slabs: its request's slot, or the caller's cache ----
    int pos;
    __half *Kc, *Vc;
    if (a.req) {
        const int4 r = reinterpret_cast<const int4 *>(a.req)[seq];  // one load: the position is not left behind the slot-table lookup
        if (r.w == 0) return;  // refused entry (uniform over the CTA)
        __half *slot = a.slots[r.z];
        Kc = slot + a.k_off;
        Vc = slot + a.v_off;
        pos = r.y;
    } else {
        Kc = a.k_cache;
        Vc = a.v_cache;
        pos = *a.pos;
    }
    Kc += (size_t)kvh * a.max_ctx * HD;
    Vc += (size_t)kvh * a.max_ctx * HD;
    const __half *qkv = a.qkv + (size_t)seq * a.qkv_stride;
    __half *out = a.out + (size_t)seq * a.out_stride;
    float *ws = a.ws + (size_t)seq * a.num_heads * a.nsplit_max * (HD + 2);  // [H][nsplit_max][HD + 2]
    unsigned *counters = a.counters + (size_t)seq * a.num_kv_heads;

    const int T = pos + 1;  // visible positions
    const int t0 = min(T, split * chunk);
    if (t0 >= T) return;  // empty split
    const int t1 = min(T, t0 + chunk);
    const int nrows = t1 - t0;
    const bool owns_new = (pos >= t0 && pos < t1);
    const int ncached = owns_new ? nrows - 1 : nrows;  // rows that already live in the cache
    const int mtiles = (nrows + 15) >> 4;

    // ---- cached K/V rows -> padded shared rows (16-byte cp.async, whole slab in flight at once) ----
    for (int e = tid; e < ncached * (HD / 8); e += kAttnThreads) {
        const int r = e >> 4, c8 = e & 15;
        cp_async16(sK + (size_t)r * kPitch + c8 * 8, Kc + (size_t)(t0 + r) * HD + c8 * 8);
        cp_async16(sV + (size_t)r * kPitch + c8 * 8, Vc + (size_t)(t0 + r) * HD + c8 * 8);
    }
    // rows of the last 16-row tile beyond nrows: finite zeros (their probabilities are zero, 0 * garbage must not be NaN)
    for (int e = tid; e < (mtiles * 16 - nrows) * (HD / 8); e += kAttnThreads) {
        const int r = nrows + (e >> 4), c8 = e & 15;
        *reinterpret_cast<uint4 *>(sK + (size_t)r * kPitch + c8 * 8) = make_uint4(0, 0, 0, 0);
        *reinterpret_cast<uint4 *>(sV + (size_t)r * kPitch + c8 * 8) = make_uint4(0, 0, 0, 0);
    }

    // ---- RoPE (llm/src/ops/RotaryPosEmb.cc:7-69 rotate-half) on the NREP query heads and, if this CTA owns the new position, on
    //      the new key; fp32 math, tables [max_ctx][HD] fp32; q * alpha is rounded to fp16 for the tensor-core product ----
    const float *cosr = a.cos + (size_t)pos * HD, *sinr = a.sin + (size_t)pos * HD;
    const int H = a.num_heads, KVH = a.num_kv_heads;
    for (int i = tid; i < 8 * HD; i += kAttnThreads) {
        const int r = i / HD, j = i % HD;
        float v = 0.f;
        if (r < NREP) {
            const __half *q = qkv + (size_t)(kvh * NREP + r) * HD;
            const float x = __half2float(q[j]);
            const float xr = (j < HD / 2) ? -__half2float(q[j + HD / 2]) : __half2float(q[j - HD / 2]);
            v = (x * cosr[j] + xr * sinr[j]) * a.alpha;
        }
        sQ[r * kPitch + j] = __float2half(v);
    }
    if (owns_new && tid < HD) {
        const int j = tid;
        const __half *k = qkv + (size_t)H * HD + (size_t)kvh * HD;
        const __half *v = qkv + (size_t)(H + KVH) * HD + (size_t)kvh * HD;
        const float x = __half2float(k[j]);
        const float xr = (j < HD / 2) ? -__half2float(k[j + HD / 2]) : __half2float(k[j - HD / 2]);
        const __half kh = __float2half(x * cosr[j] + xr * sinr[j]);
        sK[(size_t)(nrows - 1) * kPitch + j] = kh;  // row `pos` of the slab; the copies above never touch it
        sV[(size_t)(nrows - 1) * kPitch + j] = v[j];
        Kc[(size_t)pos * HD + j] = kh;              // in-place append
        Vc[(size_t)pos * HD + j] = v[j];
    }
    cp_async_wait_all();
    __syncthreads();

    // ---- scores on the tensor cores: S^T[key][head] = K[key][:] . q[head][:]  (m16n8k16: 16 keys x 8 head columns x 16 dims) ----
    {
        uint32_t qb[8][2];  // B operand: q[head = g][dims], all 8 k-steps
#pragma unroll
        for (int ks = 0; ks < 8; ks++) {
            qb[ks][0] = *reinterpret_cast<const uint32_t *>(sQ + g * kPitch + ks * 16 + qd * 2);
            qb[ks][1] = *reinterpret_cast<const uint32_t *>(sQ + g * kPitch + ks * 16 + 8 + qd * 2);
        }
        for (int mt = warp; mt < mtiles; mt += kAttnThreads / 32) {
            float c[4] = {0.f, 0.f, 0.f, 0.f};
            const __half *arow = sK + (size_t)(mt * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * kPitch + (lane >> 4) * 8;
#pragma unroll
            for (int ks = 0; ks < 8; ks++) {
                uint32_t a0, a1, a2, a3;
                ldmatrix_x4(a0, a1, a2, a3, arow + ks * 16);
                mma_m16n8k16(c, a0, a1, a2, a3, qb[ks][0], qb[ks][1]);
            }
            const int key = mt * 16 + g, h0 = qd * 2;  // c0,c1: (key, heads h0, h0+1); c2,c3: (key + 8, ...)
            if (h0 < NREP) {
                if (key < nrows) sP[h0 * p_floats(chunk) + key] = c[0];
                if (key + 8 < nrows) sP[h0 * p_floats(chunk) + key + 8] = c[2];
            }
            if (h0 + 1 < NREP) {
                if (key < nrows) sP[(h0 + 1) * p_floats(chunk) + key] = c[1];
                if (key + 8 < nrows) sP[(h0 + 1) * p_floats(chunk) + key + 8] = c[3];
            }
        }
    }
    __syncthreads();

    // ---- softmax statistics of this split (fp32): m = max, p = exp(s - m) (kept as fp16 for the P.V product), l = sum p ----
    float m_loc[NREP], l_loc[NREP];
#pragma unroll
    for (int r = 0; r < NREP; r++) {
        float m = -INFINITY;
        for (int i = tid; i < nrows; i += kAttnThreads) m = fmaxf(m, sP[r * p_floats(chunk) + i]);
        m = warp_max(m);
        if (lane == 0) sStat[r * 16 + warp] = m;
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < NREP; r++) {
        float m = sStat[r * 16];
#pragma unroll
        for (int w = 1; w < kAttnThreads / 32; w++) m = fmaxf(m, sStat[r * 16 + w]);
        m_loc[r] = m;
        float l = 0.f;
        for (int i = tid; i < mtiles * 16; i += kAttnThreads) {
            float p = 0.f;
            if (i < nrows) {
                p = __expf(sP[r * p_floats(chunk) + i] - m);
                l += p;
            }
            sPh[r * R16 + i] = __float2half(p);
        }
        l = warp_sum(l);
        if (lane == 0) sStat[NREP * 16 + r * 16 + warp] = l;
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < NREP; r++) {
        float l = 0.f;
#pragma unroll
        for (int w = 0; w < kAttnThreads / 32; w++) l += sStat[NREP * 16 + r * 16 + w];
        l_loc[r] = l;
    }

    // ---- O[head][dim] = sum_key P[head][key] V[key][dim] on the tensor cores: warp w owns dims 16w..16w+15 over all keys ----
    {
        float o0[4] = {0.f, 0.f, 0.f, 0.f}, o1[4] = {0.f, 0.f, 0.f, 0.f};
        const int dbase = warp * 16;
        for (int kt = 0; kt < mtiles; kt++) {
            uint32_t a0 = 0u, a2 = 0u;  // A = P: rows = heads (g < NREP valid, rows 8..15 zero), k = 16 keys
            if (g < NREP) {
                a0 = *reinterpret_cast<const uint32_t *>(sPh + g * R16 + kt * 16 + qd * 2);
                a2 = *reinterpret_cast<const uint32_t *>(sPh + g * R16 + kt * 16 + 8 + qd * 2);
            }
            uint32_t b0, b1, b2, b3;
            ldmatrix_x4_t(b0, b1, b2, b3, sV + (size_t)(kt * 16 + (lane & 15)) * kPitch + dbase + (lane >> 4) * 8);
            mma_m16n8k16(o0, a0, 0u, a2, 0u, b0, b1);
            mma_m16n8k16(o1, a0, 0u, a2, 0u, b2, b3);
        }
        if (g < NREP) {  // c0,c1: (head g, dims 2qd, 2qd+1)
            sO[g * HD + dbase + qd * 2] = o0[0];
            sO[g * HD + dbase + qd * 2 + 1] = o0[1];
            sO[g * HD + dbase + 8 + qd * 2] = o1[0];
            sO[g * HD + dbase + 8 + qd * 2 + 1] = o1[1];
        }
    }
    __syncthreads();

    // ---- per-split result (unnormalised o, m, l) ----
    const int nsplit_active = (T + chunk - 1) / chunk;
    const int wstride = HD + 2;
    for (int i = tid; i < NREP * HD; i += kAttnThreads) {
        const int r = i / HD, d = i % HD;
        const float o = sO[i];
        const int head = kvh * NREP + r;
        if (nsplit_active == 1) {
            out[(size_t)head * HD + d] = __float2half(o / l_loc[r]);
        } else {
            float *rec = ws + ((size_t)head * a.nsplit_max + split) * wstride;
            rec[d] = o;
            if (d == 0) {
                rec[HD] = m_loc[r];
                rec[HD + 1] = l_loc[r];
            }
        }
    }
    if (nsplit_active == 1) return;

    // ---- merge: the last split of this KV head to arrive combines all of them in split order ----
    __threadfence();
    __syncthreads();
    if (tid == 0) {
        const unsigned prev = atomicAdd(&counters[kvh], 1u);
        const int last = (prev == (unsigned)(nsplit_active - 1)) ? 1 : 0;
        if (last) counters[kvh] = 0;
        *flag = last;
    }
    __syncthreads();
    if (*flag == 0) return;
    __threadfence();
    for (int i = tid; i < NREP * HD; i += kAttnThreads) {
        const int r = i / HD, d = i % HD;
        const int head = kvh * NREP + r;
        const float *base = ws + (size_t)head * a.nsplit_max * wstride;
        float m = -INFINITY;
        for (int s = 0; s < nsplit_active; s++) m = fmaxf(m, ldg_cg_f32(base + (size_t)s * wstride + HD));
        float l = 0.f, o = 0.f;
        for (int s = 0; s < nsplit_active; s++) {
            const float w = __expf(ldg_cg_f32(base + (size_t)s * wstride + HD) - m);
            l += w * ldg_cg_f32(base + (size_t)s * wstride + HD + 1);
            o += w * ldg_cg_f32(base + (size_t)s * wstride + d);
        }
        out[(size_t)head * HD + d] = __float2half(o / l);
    }
}

template <int NREP>
cudaError_t launch(Ctx *ctx, const AttnDecodeArgs &a, int batch, bool pdl) {
    const size_t smem = smem_bytes(NREP, a.chunk) + 16;  // + the last-split flag
    static DeviceOnce attr_once;
    if (attr_once.pending(ctx->device)) {
        cudaError_t e = cudaFuncSetAttribute(attn_decode_kernel<NREP>, cudaFuncAttributeMaxDynamicSharedMemorySize, ctx->smem_optin);
        if (e != cudaSuccess) return e;
        attr_once.done(ctx->device);
    }
    if ((int)smem > ctx->smem_optin) return cudaErrorInvalidConfiguration;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(a.num_kv_heads, a.nsplit_max, batch);
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

// ---- span attention: n consecutive tokens of ONE sequence (the span step, tce_llama_decode_span_host) ----
// Query row i (position pos0 + i) of head r of the CTA's KV head is column c = i * NREP + r of the MMA tiles, so a CTA reads each cached
// K / V row of its chunk once for all n * NREP columns (up to 64).  The n new K / V rows are rotated and appended by the CTA whose chunk
// holds them, before any CTA of the launch could need them from the cache: a chunk reads from the cache only rows below pos0.  Column c
// sees keys 0 .. pos0 + i.  fp32 softmax statistics, fixed-order split merge, as attn_decode_kernel.
inline __host__ __device__ size_t span_smem_bytes(int nrep, int chunk, int n) {
    const int nc = n * nrep, nc16 = (nc + 15) & ~15;
    size_t b = (size_t)2 * rows16(chunk) * kPitch * 2;   // K, V slabs
    b += (size_t)nc16 * kPitch * 2;                      // q columns, fp16 (rows >= nc zero)
    b += (size_t)nc * p_floats(chunk) * 4;               // scores fp32; reused for the unnormalised output [nc][HD]
    b += (size_t)nc16 * rows16(chunk) * 2;               // probabilities fp16 (rows >= nc zero)
    b += (size_t)2 * nc * 4;                             // m, l per column
    return (b + 15) & ~(size_t)15;
}

template <int NREP>
__global__ void __launch_bounds__(kAttnThreads, 1) attn_span_kernel(const __grid_constant__ AttnDecodeArgs a, int n) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int chunk = a.chunk;
    const int R16 = rows16(chunk), PF = p_floats(chunk);
    const int NC = n * NREP, NC16 = (NC + 15) & ~15;
    __half *sK = reinterpret_cast<__half *>(smem);                        // [R16][kPitch]
    __half *sV = sK + (size_t)R16 * kPitch;                               // [R16][kPitch]
    __half *sQ = sV + (size_t)R16 * kPitch;                               // [NC16][kPitch]
    float *sP = reinterpret_cast<float *>(sQ + (size_t)NC16 * kPitch);    // [NC][PF] scores, then [NC][HD] output
    __half *sPh = reinterpret_cast<__half *>(sP + (size_t)NC * PF);       // [NC16][R16]
    float *sM = reinterpret_cast<float *>(sPh + (size_t)NC16 * R16);      // [NC]
    float *sL = sM + NC;                                                  // [NC]
    int *flag = reinterpret_cast<int *>(smem + span_smem_bytes(NREP, chunk, n));
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, qd = lane & 3;
    const int kvh = blockIdx.x, split = blockIdx.y;
    pdl_launch_dependents();
    pdl_wait();

    // with a request table every row names the same slot at consecutive positions (host-checked): row 0 gives both; without one, the
    // caller's cache and first position
    int pos0;
    __half *Kc, *Vc;
    if (a.req) {
        const int4 r0 = reinterpret_cast<const int4 *>(a.req)[0];
        if (r0.w == 0) return;
        pos0 = r0.y;
        Kc = a.slots[r0.z] + a.k_off;
        Vc = a.slots[r0.z] + a.v_off;
    } else {
        pos0 = a.span_pos0;
        Kc = a.k_cache;
        Vc = a.v_cache;
    }
    Kc += (size_t)kvh * a.max_ctx * HD;
    Vc += (size_t)kvh * a.max_ctx * HD;
    const int H = a.num_heads, KVH = a.num_kv_heads;

    const int T = pos0 + n;  // keys visible to the last row
    const int t0 = split * chunk;
    if (t0 >= T) return;
    const int t1 = min(T, t0 + chunk);
    const int nrows = t1 - t0;
    const int ncached = max(0, min(nrows, pos0 - t0));
    const int mtiles = (nrows + 15) >> 4;

    for (int e = tid; e < ncached * (HD / 8); e += kAttnThreads) {
        const int r = e >> 4, c8 = e & 15;
        cp_async16(sK + (size_t)r * kPitch + c8 * 8, Kc + (size_t)(t0 + r) * HD + c8 * 8);
        cp_async16(sV + (size_t)r * kPitch + c8 * 8, Vc + (size_t)(t0 + r) * HD + c8 * 8);
    }
    for (int e = tid; e < (mtiles * 16 - nrows) * (HD / 8); e += kAttnThreads) {
        const int r = nrows + (e >> 4), c8 = e & 15;
        *reinterpret_cast<uint4 *>(sK + (size_t)r * kPitch + c8 * 8) = make_uint4(0, 0, 0, 0);
        *reinterpret_cast<uint4 *>(sV + (size_t)r * kPitch + c8 * 8) = make_uint4(0, 0, 0, 0);
    }
    // new rows of this chunk: RoPE on k (fp32, rounded to fp16), in-place append of k and v
    for (int e = tid; e < (nrows - ncached) * HD; e += kAttnThreads) {
        const int r = ncached + e / HD, j = e % HD, t = t0 + r, i = t - pos0;
        const __half *qkv = a.qkv + (size_t)i * a.qkv_stride;
        const __half *k = qkv + (size_t)H * HD + (size_t)kvh * HD;
        const __half *v = qkv + (size_t)(H + KVH) * HD + (size_t)kvh * HD;
        const float x = __half2float(k[j]);
        const float xr = (j < HD / 2) ? -__half2float(k[j + HD / 2]) : __half2float(k[j - HD / 2]);
        const __half kh = __float2half(x * a.cos[(size_t)t * HD + j] + xr * a.sin[(size_t)t * HD + j]);
        sK[(size_t)r * kPitch + j] = kh;
        sV[(size_t)r * kPitch + j] = v[j];
        Kc[(size_t)t * HD + j] = kh;
        Vc[(size_t)t * HD + j] = v[j];
    }
    // query columns: RoPE at the row's position, * alpha, fp16
    for (int e = tid; e < NC16 * HD; e += kAttnThreads) {
        const int c = e / HD, j = e % HD;
        float v = 0.f;
        if (c < NC) {
            const int i = c / NREP, r = c % NREP, t = pos0 + i;
            const __half *q = a.qkv + (size_t)i * a.qkv_stride + (size_t)(kvh * NREP + r) * HD;
            const float x = __half2float(q[j]);
            const float xr = (j < HD / 2) ? -__half2float(q[j + HD / 2]) : __half2float(q[j - HD / 2]);
            v = (x * a.cos[(size_t)t * HD + j] + xr * a.sin[(size_t)t * HD + j]) * a.alpha;
        }
        sQ[(size_t)c * kPitch + j] = __float2half(v);
    }
    cp_async_wait_all();
    __syncthreads();

    // ---- scores S^T[key][column]: one (16-key, 8-column) tile per warp iteration ----
    const int ntiles = NC16 / 8;
    for (int tile = warp; tile < mtiles * ntiles; tile += kAttnThreads / 32) {
        const int mt = tile / ntiles, nt = tile % ntiles;
        float c[4] = {0.f, 0.f, 0.f, 0.f};
        const __half *arow = sK + (size_t)(mt * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * kPitch + (lane >> 4) * 8;
        const __half *brow = sQ + (size_t)(nt * 8 + g) * kPitch + qd * 2;
#pragma unroll
        for (int ks = 0; ks < 8; ks++) {
            uint32_t a0, a1, a2, a3;
            ldmatrix_x4(a0, a1, a2, a3, arow + ks * 16);
            const uint32_t b0 = *reinterpret_cast<const uint32_t *>(brow + ks * 16);
            const uint32_t b1 = *reinterpret_cast<const uint32_t *>(brow + ks * 16 + 8);
            mma_m16n8k16(c, a0, a1, a2, a3, b0, b1);
        }
        const int key = mt * 16 + g, col = nt * 8 + qd * 2;
        if (col < NC) {
            if (key < nrows) sP[(size_t)col * PF + key] = c[0];
            if (key + 8 < nrows) sP[(size_t)col * PF + key + 8] = c[2];
        }
        if (col + 1 < NC) {
            if (key < nrows) sP[(size_t)(col + 1) * PF + key] = c[1];
            if (key + 8 < nrows) sP[(size_t)(col + 1) * PF + key + 8] = c[3];
        }
    }
    __syncthreads();

    // ---- causal softmax statistics per column (one warp per column): column c of row i sees keys t <= pos0 + i ----
    for (int c = warp; c < NC16; c += kAttnThreads / 32) {
        const int lim = c < NC ? min(nrows, pos0 + c / NREP - t0 + 1) : 0;  // visible keys of this chunk (may be <= 0)
        float m = -INFINITY;
        for (int k = lane; k < lim; k += 32) m = fmaxf(m, sP[(size_t)c * PF + k]);
        m = warp_max(m);
        float l = 0.f;
        for (int k = lane; k < mtiles * 16; k += 32) {
            float p = 0.f;
            if (k < lim) {
                p = __expf(sP[(size_t)c * PF + k] - m);
                l += p;
            }
            sPh[(size_t)c * R16 + k] = __float2half(p);
        }
        l = warp_sum(l);
        if (lane == 0 && c < NC) {
            sM[c] = m;
            sL[c] = l;
        }
    }
    __syncthreads();

    // ---- O[column][dim] = sum_key P[column][key] V[key][dim]: warp w owns dims 16w..16w+15, 16 columns per MMA row tile ----
    float *sO = sP;  // [NC][HD]: the scores are no longer read
    {
        const int dbase = warp * 16;
        for (int ct = 0; ct < NC16 / 16; ct++) {
            float o0[4] = {0.f, 0.f, 0.f, 0.f}, o1[4] = {0.f, 0.f, 0.f, 0.f};
            const __half *pa = sPh + (size_t)(ct * 16 + g) * R16 + qd * 2, *pb = pa + (size_t)8 * R16;
            for (int kt = 0; kt < mtiles; kt++) {
                const uint32_t a0 = *reinterpret_cast<const uint32_t *>(pa + kt * 16), a2 = *reinterpret_cast<const uint32_t *>(pa + kt * 16 + 8);
                const uint32_t a1 = *reinterpret_cast<const uint32_t *>(pb + kt * 16), a3 = *reinterpret_cast<const uint32_t *>(pb + kt * 16 + 8);
                uint32_t b0, b1, b2, b3;
                ldmatrix_x4_t(b0, b1, b2, b3, sV + (size_t)(kt * 16 + (lane & 15)) * kPitch + dbase + (lane >> 4) * 8);
                mma_m16n8k16(o0, a0, a1, a2, a3, b0, b1);
                mma_m16n8k16(o1, a0, a1, a2, a3, b2, b3);
            }
            const int c = ct * 16 + g;  // c0,c1: (column c, dims 2qd, 2qd+1); c2,c3: column c + 8
            if (c < NC) {
                sO[(size_t)c * HD + dbase + qd * 2] = o0[0];
                sO[(size_t)c * HD + dbase + qd * 2 + 1] = o0[1];
                sO[(size_t)c * HD + dbase + 8 + qd * 2] = o1[0];
                sO[(size_t)c * HD + dbase + 8 + qd * 2 + 1] = o1[1];
            }
            if (c + 8 < NC) {
                sO[(size_t)(c + 8) * HD + dbase + qd * 2] = o0[2];
                sO[(size_t)(c + 8) * HD + dbase + qd * 2 + 1] = o0[3];
                sO[(size_t)(c + 8) * HD + dbase + 8 + qd * 2] = o1[2];
                sO[(size_t)(c + 8) * HD + dbase + 8 + qd * 2 + 1] = o1[3];
            }
        }
    }
    __syncthreads();

    // ---- per-split result; split records [row][head][split][HD + 2] ----
    const int nsplit_active = (T + chunk - 1) / chunk;
    const int wstride = HD + 2;
    auto rec_of = [&](int c) {
        const int i = c / NREP, head = kvh * NREP + c % NREP;
        return a.ws + ((size_t)i * H + head) * a.nsplit_max * wstride;
    };
    auto out_of = [&](int c) { return a.out + (size_t)(c / NREP) * a.out_stride + (size_t)(kvh * NREP + c % NREP) * HD; };
    for (int e = tid; e < NC * HD; e += kAttnThreads) {
        const int c = e / HD, d = e % HD;
        const float o = sO[e];
        if (nsplit_active == 1) {
            out_of(c)[d] = __float2half(o / sL[c]);  // split 0 holds key 0, visible to every row: l > 0
        } else {
            float *rec = rec_of(c) + (size_t)split * wstride;
            rec[d] = o;
            if (d == 0) {
                rec[HD] = sM[c];
                rec[HD + 1] = sL[c];
            }
        }
    }
    if (nsplit_active == 1) return;

    __threadfence();
    __syncthreads();
    if (tid == 0) {
        const unsigned prev = atomicAdd(&a.counters[kvh], 1u);
        const int last = (prev == (unsigned)(nsplit_active - 1)) ? 1 : 0;
        if (last) a.counters[kvh] = 0;
        *flag = last;
    }
    __syncthreads();
    if (*flag == 0) return;
    __threadfence();
    for (int e = tid; e < NC * HD; e += kAttnThreads) {
        const int c = e / HD, d = e % HD;
        const float *base = rec_of(c);
        float m = -INFINITY;
        for (int s = 0; s < nsplit_active; s++) m = fmaxf(m, ldg_cg_f32(base + (size_t)s * wstride + HD));
        float l = 0.f, o = 0.f;
        for (int s = 0; s < nsplit_active; s++) {
            const float w = __expf(ldg_cg_f32(base + (size_t)s * wstride + HD) - m);  // a split with no visible key: m_s = -inf, w = 0
            l += w * ldg_cg_f32(base + (size_t)s * wstride + HD + 1);
            o += w * ldg_cg_f32(base + (size_t)s * wstride + d);
        }
        out_of(c)[d] = __float2half(o / l);
    }
}

template <int NREP>
cudaError_t launch_span(Ctx *ctx, const AttnDecodeArgs &a, int n, bool pdl) {
    const size_t smem = span_smem_bytes(NREP, a.chunk, n) + 16;
    static DeviceOnce attr_once;
    if (attr_once.pending(ctx->device)) {
        cudaError_t e = cudaFuncSetAttribute(attn_span_kernel<NREP>, cudaFuncAttributeMaxDynamicSharedMemorySize, ctx->smem_optin);
        if (e != cudaSuccess) return e;
        attr_once.done(ctx->device);
    }
    if ((int)smem > ctx->smem_optin) return cudaErrorInvalidConfiguration;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(a.num_kv_heads, a.nsplit_max, 1);
    cfg.blockDim = dim3(kAttnThreads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = ctx->stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, attn_span_kernel<NREP>, a, n);
}

}  // namespace

int attn_span_chunk(int num_heads, int num_kv_heads, int chunk, int smem_optin) {
    if (num_kv_heads < 1 || num_heads % num_kv_heads) return 0;
    const int nrep = num_heads / num_kv_heads;
    for (int c = chunk_rows(chunk) & ~15; c >= 16; c -= 16)
        if (span_smem_bytes(nrep, c, kMaxSpan) + 16 <= (size_t)smem_optin) return c;
    return 0;
}

cudaError_t launch_attn_span(Ctx *ctx, const AttnDecodeArgs &args, int n, bool pdl) {
    AttnDecodeArgs a = args;
    if (a.head_dim != HD) return cudaErrorNotSupported;
    if (a.num_heads % a.num_kv_heads || n < 1 || n > kMaxSpan || (a.req ? !a.slots : (!a.k_cache || !a.v_cache))) return cudaErrorInvalidValue;
    a.chunk = chunk_rows(a.chunk);
    a.nsplit_max = (a.max_ctx + a.chunk - 1) / a.chunk;
    // n rows of one sequence use the split records and counters of n sequences of the batched step
    if (!a.ws || !a.counters || (size_t)n * attn_decode_ws_floats(a.num_heads, a.max_ctx, a.chunk) > a.ws_floats || (size_t)a.num_kv_heads > a.n_counters)
        return cudaErrorInvalidValue;
    switch (a.num_heads / a.num_kv_heads) {
        case 1: return launch_span<1>(ctx, a, n, pdl);
        case 2: return launch_span<2>(ctx, a, n, pdl);
        case 4: return launch_span<4>(ctx, a, n, pdl);
        case 8: return launch_span<8>(ctx, a, n, pdl);
        default: return cudaErrorNotSupported;
    }
}

size_t attn_decode_ws_floats(int num_heads, int max_ctx, int chunk) {
    chunk = chunk_rows(chunk);
    return (size_t)num_heads * ((max_ctx + chunk - 1) / chunk) * (HD + 2);
}

cudaError_t launch_attn_decode(Ctx *ctx, const AttnDecodeArgs &args, int batch, bool pdl) {
    AttnDecodeArgs a = args;
    if (a.head_dim != HD) return cudaErrorNotSupported;
    if (a.num_heads % a.num_kv_heads || batch < 1) return cudaErrorInvalidValue;
    a.chunk = chunk_rows(a.chunk);
    a.nsplit_max = (a.max_ctx + a.chunk - 1) / a.chunk;
    // per sequence: its own partial records and split counters, in the caller's workspace
    if (!a.ws || !a.counters || (size_t)batch * attn_decode_ws_floats(a.num_heads, a.max_ctx, a.chunk) > a.ws_floats ||
        (size_t)batch * a.num_kv_heads > a.n_counters)
        return cudaErrorInvalidValue;
    switch (a.num_heads / a.num_kv_heads) {
        case 1: return launch<1>(ctx, a, batch, pdl);
        case 2: return launch<2>(ctx, a, batch, pdl);
        case 4: return launch<4>(ctx, a, batch, pdl);
        case 8: return launch<8>(ctx, a, batch, pdl);
        default: return cudaErrorNotSupported;
    }
}

}  // namespace tce
