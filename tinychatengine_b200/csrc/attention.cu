// attention.cu -- per-token KV-cache attention for decode (fp16 cache, GQA aware) on sm_90a.
//
// Replaces the attention part of Int4llamaAttention::forward between qkv_proj and o_proj
// (reference llm/src/nn_modules/cuda/Int4llamaAttention.cu:128-217: shape_qkv -> RotaryPosEmb_cuda_forward ->
// 4*heads cudaMemcpyAsync KV concat -> BMM_F16T QK^T -> batch_Add mask -> check_inf -> softmax_cuda ->
// transpose V -> BMM_F16T PV -> unshape) with ONE kernel, with the GQA head mapping of the CPU module
// (llm/src/nn_modules/non_cuda/Int4llamaAttention.cc:166-184: q head i reads kv head i / (H/KVH)).
//
//  * KV cache is [KVH][max_ctx][128] fp16 per layer, appended IN PLACE at the new positions (no ping-pong copy, no V
//    transpose);
//  * grid = (KVH, ceil(max_ctx/chunk), seqs): a CTA owns `chunk` cached positions of one KV head of one sequence and
//    serves the H/KVH query heads that share it, for each of the sequence's n consecutive rows (n = 1: the per-token step;
//    n > 1: the span step), so each cached byte is read once per step;
//  * its K and V rows are pulled into padded shared rows by 16-byte cp.async copies issued up front -- the whole cache of
//    the layer is in flight at once, the kernel is HBM-bound;
//  * the n * H/KVH query rows are the columns of 8-column MMA tiles: scores and P.V run on mma.sync m16n8k16 with fp16
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
// shared memory of one CTA serving nc query columns; the word after it elects the last split
inline __host__ __device__ size_t smem_bytes(int nc, int chunk) {
    size_t b = (size_t)2 * rows16(chunk) * kPitch * 2;  // K, V slabs (padded rows)
    b += (size_t)nc * kPitch * 2;                        // q columns, fp16
    b += (size_t)nc * p_floats(chunk) * 4;               // scores fp32; reused for the unnormalised output [nc][HD]
    b += (size_t)nc * rows16(chunk) * 2;                 // probabilities fp16
    b += (size_t)2 * nc * 4;                             // m, l per column
    return (b + 15) & ~(size_t)15;
}

// One (KV head, split, sequence) work item per CTA.  Sequence s = blockIdx.z owns rows s * n .. s * n + n - 1 of qkv / out and of the split
// records: row s * n + i is its position pos0 + i.  Query row i of head r of the CTA's KV head is column c = i * NREP + r of the MMA tiles,
// so a CTA reads each cached K / V row of its chunk once for all n * NREP columns (up to 64).  The n new K / V rows are rotated and appended
// by the CTA whose chunk holds them, before any CTA of the launch could need them from the cache: a chunk reads from the cache only rows
// below pos0.  Column c sees keys 0 .. pos0 + c / NREP.  The per-column buffers hold n * NREP rows; MMA rows and columns beyond them are
// fed as zero registers, so the single-row step (n = 1) reads and computes what it needs and no padding.
template <int NREP>
__global__ void __launch_bounds__(kAttnThreads, 1) attn_decode_kernel(const __grid_constant__ AttnDecodeArgs a, int n) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int chunk = a.chunk;
    const int R16 = rows16(chunk), PF = p_floats(chunk);
    const int NC = n * NREP;
    __half *sK = reinterpret_cast<__half *>(smem);                        // [R16][kPitch]
    __half *sV = sK + (size_t)R16 * kPitch;                               // [R16][kPitch]
    __half *sQ = sV + (size_t)R16 * kPitch;                               // [NC][kPitch] rotated * alpha
    float *sP = reinterpret_cast<float *>(sQ + (size_t)NC * kPitch);      // [NC][PF] scores, then [NC][HD] output
    __half *sPh = reinterpret_cast<__half *>(sP + (size_t)NC * PF);       // [NC][R16]
    float *sM = reinterpret_cast<float *>(sPh + (size_t)NC * R16);        // [NC]
    float *sL = sM + NC;                                                  // [NC]
    int *flag = reinterpret_cast<int *>(smem + smem_bytes(NC, chunk));
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, qd = lane & 3;
    const int kvh = blockIdx.x, split = blockIdx.y, seq = blockIdx.z;
    pdl_launch_dependents();
    pdl_wait();  // q|k|v (and the request records) come from the previous kernels; the cache was written by earlier steps

    // ---- this sequence's first position and K / V slabs.  With a request table, row seq * n gives both (the other rows of a span name the
    //      same slot at consecutive positions, host-checked); without one, the caller's cache and position ----
    int pos0;
    __half *Kc, *Vc;
    if (a.req) {
        const int4 r = reinterpret_cast<const int4 *>(a.req)[seq * n];  // one load: the position is not left behind the slot-table lookup
        if (r.w == 0) return;  // refused entry (uniform over the CTA)
        __half *slot = a.slots[r.z];
        Kc = slot + a.k_off;
        Vc = slot + a.v_off;
        pos0 = r.y;
    } else {
        Kc = a.k_cache;
        Vc = a.v_cache;
        pos0 = a.pos ? *a.pos : a.pos0;
    }
    Kc += (size_t)kvh * a.max_ctx * HD;
    Vc += (size_t)kvh * a.max_ctx * HD;
    const int H = a.num_heads, KVH = a.num_kv_heads;
    const __half *qkv = a.qkv + (size_t)seq * n * a.qkv_stride;
    __half *out = a.out + (size_t)seq * n * a.out_stride;
    float *ws = a.ws + (size_t)seq * n * H * a.nsplit_max * (HD + 2);  // [n][H][nsplit_max][HD + 2]
    unsigned *counters = a.counters + (size_t)seq * KVH;

    const int T = pos0 + n;  // keys visible to the last row
    const int t0 = split * chunk;
    if (t0 >= T) return;  // empty split
    const int t1 = min(T, t0 + chunk);
    const int nrows = t1 - t0;
    const int ncached = max(0, min(nrows, pos0 - t0));  // rows that already live in the cache
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
    // ---- RoPE (llm/src/ops/RotaryPosEmb.cc:7-69 rotate-half), fp32 math, tables [max_ctx][HD] fp32.  New rows of this chunk: k rounded to
    //      fp16, in-place append of k and v (the copies above never touch these rows) ----
    for (int e = tid; e < (nrows - ncached) * HD; e += kAttnThreads) {
        const int r = ncached + e / HD, j = e % HD, t = t0 + r, i = t - pos0;
        const __half *k = qkv + (size_t)i * a.qkv_stride + (size_t)H * HD + (size_t)kvh * HD;
        const __half *v = qkv + (size_t)i * a.qkv_stride + (size_t)(H + KVH) * HD + (size_t)kvh * HD;
        const float x = __half2float(k[j]);
        const float xr = (j < HD / 2) ? -__half2float(k[j + HD / 2]) : __half2float(k[j - HD / 2]);
        const __half kh = __float2half(x * a.cos[(size_t)t * HD + j] + xr * a.sin[(size_t)t * HD + j]);
        sK[(size_t)r * kPitch + j] = kh;
        sV[(size_t)r * kPitch + j] = v[j];
        Kc[(size_t)t * HD + j] = kh;
        Vc[(size_t)t * HD + j] = v[j];
    }
    // query columns: RoPE at the row's position, * alpha, rounded to fp16 for the tensor-core product
    for (int e = tid; e < NC * HD; e += kAttnThreads) {
        const int c = e / HD, j = e % HD, i = c / NREP, r = c % NREP, t = pos0 + i;
        const __half *q = qkv + (size_t)i * a.qkv_stride + (size_t)(kvh * NREP + r) * HD;
        const float x = __half2float(q[j]);
        const float xr = (j < HD / 2) ? -__half2float(q[j + HD / 2]) : __half2float(q[j - HD / 2]);
        sQ[(size_t)c * kPitch + j] = __float2half((x * a.cos[(size_t)t * HD + j] + xr * a.sin[(size_t)t * HD + j]) * a.alpha);
    }
    cp_async_wait_all();
    __syncthreads();

    // ---- scores on the tensor cores: S^T[key][column] = K[key][:] . q[column][:], one (16-key, 8-column) m16n8k16 tile per warp iteration ----
    const int ntiles = (NC + 7) >> 3;
    for (int tile = warp; tile < mtiles * ntiles; tile += kAttnThreads / 32) {
        const int mt = tile / ntiles, nt = tile % ntiles;
        float c[4] = {0.f, 0.f, 0.f, 0.f};
        const __half *arow = sK + (size_t)(mt * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * kPitch + (lane >> 4) * 8;
        const int bc = nt * 8 + g;  // this lane's B column
        const __half *brow = sQ + (size_t)bc * kPitch + qd * 2;
#pragma unroll
        for (int ks = 0; ks < 8; ks++) {
            uint32_t a0, a1, a2, a3, b0 = 0u, b1 = 0u;
            ldmatrix_x4(a0, a1, a2, a3, arow + ks * 16);
            if (bc < NC) {
                b0 = *reinterpret_cast<const uint32_t *>(brow + ks * 16);
                b1 = *reinterpret_cast<const uint32_t *>(brow + ks * 16 + 8);
            }
            mma_m16n8k16(c, a0, a1, a2, a3, b0, b1);
        }
        const int key = mt * 16 + g, col = nt * 8 + qd * 2;  // c0,c1: (key, columns col, col+1); c2,c3: (key + 8, ...)
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

    // ---- causal softmax statistics per column (fp32, one warp per column): m = max, p = exp(s - m) (kept as fp16 for the P.V product),
    //      l = sum p.  Column c sees keys t <= pos0 + c / NREP ----
    for (int c = warp; c < NC; c += kAttnThreads / 32) {
        const int lim = min(nrows, pos0 + c / NREP - t0 + 1);  // visible keys of this chunk (may be <= 0)
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
        if (lane == 0) {
            sM[c] = m;
            sL[c] = l;
        }
    }
    __syncthreads();

    // ---- O[column][dim] = sum_key P[column][key] V[key][dim] on the tensor cores: warp w owns dims 16w..16w+15, 16 columns per MMA row tile ----
    float *sO = sP;  // [NC][HD]: the scores are no longer read
    {
        const int dbase = warp * 16;
        for (int ct = 0; ct < (NC + 15) >> 4; ct++) {
            const int c = ct * 16 + g;  // A rows c and c + 8
            const __half *pa = sPh + (size_t)c * R16 + qd * 2, *pb = pa + (size_t)8 * R16;
            float o0[4] = {0.f, 0.f, 0.f, 0.f}, o1[4] = {0.f, 0.f, 0.f, 0.f};
            for (int kt = 0; kt < mtiles; kt++) {
                uint32_t a0 = 0u, a1 = 0u, a2 = 0u, a3 = 0u;
                if (c < NC) {
                    a0 = *reinterpret_cast<const uint32_t *>(pa + kt * 16);
                    a2 = *reinterpret_cast<const uint32_t *>(pa + kt * 16 + 8);
                }
                if (c + 8 < NC) {
                    a1 = *reinterpret_cast<const uint32_t *>(pb + kt * 16);
                    a3 = *reinterpret_cast<const uint32_t *>(pb + kt * 16 + 8);
                }
                uint32_t b0, b1, b2, b3;
                ldmatrix_x4_t(b0, b1, b2, b3, sV + (size_t)(kt * 16 + (lane & 15)) * kPitch + dbase + (lane >> 4) * 8);
                mma_m16n8k16(o0, a0, a1, a2, a3, b0, b1);
                mma_m16n8k16(o1, a0, a1, a2, a3, b2, b3);
            }
            // c0,c1: (column c, dims 2qd, 2qd+1); c2,c3: column c + 8
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

    // ---- per-split result (unnormalised o, m, l); split records [row][head][split][HD + 2] ----
    const int nsplit_active = (T + chunk - 1) / chunk;
    const int wstride = HD + 2;
    auto rec_of = [&](int c) { return ws + ((size_t)(c / NREP) * H + kvh * NREP + c % NREP) * a.nsplit_max * wstride; };
    auto out_of = [&](int c) { return out + (size_t)(c / NREP) * a.out_stride + (size_t)(kvh * NREP + c % NREP) * HD; };
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
cudaError_t launch(Ctx *ctx, const AttnDecodeArgs &a, int seqs, int n, bool pdl) {
    const size_t smem = smem_bytes(n * NREP, a.chunk) + 16;  // + the last-split flag
    static DeviceOnce attr_once;
    if (attr_once.pending(ctx->device)) {
        cudaError_t e = cudaFuncSetAttribute(attn_decode_kernel<NREP>, cudaFuncAttributeMaxDynamicSharedMemorySize, ctx->smem_optin);
        if (e != cudaSuccess) return e;
        attr_once.done(ctx->device);
    }
    if ((int)smem > ctx->smem_optin) return cudaErrorInvalidConfiguration;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(a.num_kv_heads, a.nsplit_max, seqs);
    cfg.blockDim = dim3(kAttnThreads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = ctx->stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, attn_decode_kernel<NREP>, a, n);
}

}  // namespace

int attn_span_chunk(int num_heads, int num_kv_heads, int chunk, int smem_optin) {
    if (num_kv_heads < 1 || num_heads % num_kv_heads) return 0;
    const int nrep = num_heads / num_kv_heads;
    for (int c = chunk_rows(chunk) & ~15; c >= 16; c -= 16)
        if (smem_bytes(kMaxSpan * nrep, c) + 16 <= (size_t)smem_optin) return c;
    return 0;
}

size_t attn_decode_ws_floats(int num_heads, int max_ctx, int chunk) {
    chunk = chunk_rows(chunk);
    return (size_t)num_heads * ((max_ctx + chunk - 1) / chunk) * (HD + 2);
}

cudaError_t launch_attn_decode(Ctx *ctx, const AttnDecodeArgs &args, int seqs, int n, bool pdl) {
    AttnDecodeArgs a = args;
    if (a.head_dim != HD) return cudaErrorNotSupported;
    if (a.num_heads % a.num_kv_heads || seqs < 1 || n < 1 || n > kMaxSpan || (a.req ? !a.slots : (!a.k_cache || !a.v_cache))) return cudaErrorInvalidValue;
    a.chunk = chunk_rows(a.chunk);
    a.nsplit_max = (a.max_ctx + a.chunk - 1) / a.chunk;
    // every row has its own split records and every sequence its own split counters, in the caller's workspace
    if (!a.ws || !a.counters || (size_t)seqs * n * attn_decode_ws_floats(a.num_heads, a.max_ctx, a.chunk) > a.ws_floats ||
        (size_t)seqs * a.num_kv_heads > a.n_counters)
        return cudaErrorInvalidValue;
    switch (a.num_heads / a.num_kv_heads) {
        case 1: return launch<1>(ctx, a, seqs, n, pdl);
        case 2: return launch<2>(ctx, a, seqs, n, pdl);
        case 4: return launch<4>(ctx, a, seqs, n, pdl);
        case 8: return launch<8>(ctx, a, seqs, n, pdl);
        default: return cudaErrorNotSupported;
    }
}

}  // namespace tce
