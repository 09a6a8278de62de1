// w4a16_gemv.cu -- stand-alone W4A16 GEMV launch (batch 1..8 decode) on sm_90a.
//
// Replaces MatmulOperator::gemv_forward_cuda + gemv_kernel_g128 (reference kernels/cuda/gemv_cuda.cu:140-260).
// The device-side roles live in w4a16_gemv_impl.cuh; this file is the kernel wrapper, the independent cross-check
// kernel (also the group-64 path) and the host-side launch logic.
#include <stdio.h>

#include "w4a16_gemv_impl.cuh"

namespace tce {

namespace {

using namespace gemv;

template <int NCOLS, int CW>
__global__ void __launch_bounds__(32 * (kProducerWarps + 1 + CW), (NCOLS == 1 && CW == 8) ? 2 : 1) w4a16_gemv_kernel(const __grid_constant__ KArgs a) {
    extern __shared__ __align__(128) uint8_t smem[];
    using L = Layout<NCOLS, CW>;
    const int xw = a.sl * 128;  // activation elements staged per column: one K-slice (the whole row when nsl == 1)
    const Smem sm = carve<NCOLS, CW>(smem, a.IC, a.nst, xw);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int cta = blockIdx.x, ncta = gridDim.x;

    if (a.pdl_early) pdl_launch_dependents();
    if (warp == 0) {
        if (lane == 0) dbg_stamp(a, cta, 0);
        init_barriers_warp<CW>(sm, lane);
    } else if (tid == 32) {
        // the TMA unit's first use of a tensor map costs a descriptor fetch: start it while warp 0 initialises the barriers
        for (int i = 0; i < a.nseg; i++) asm volatile("prefetch.tensormap [%0];" ::"l"(&a.tmap[i]) : "memory");
    }
    // Warp 0 (which initialised the barriers) only signals; the others wait where they first need the barriers: the epilogue warp
    // right away, the consumers after they have staged the activations (staging touches no mbarrier), so that barrier set-up, the
    // first weight copies and the activation staging all overlap.
    if (warp == 0) {
        __syncwarp();
        asm volatile("bar.arrive 3, %0;" ::"r"(32 * (kProducerWarps + 1 + CW)) : "memory");
    } else if (warp == kProducerWarps) {
        asm volatile("bar.sync 3, %0;" ::"r"(32 * (kProducerWarps + 1 + CW)) : "memory");
    }

    if (warp < kProducerWarps) {
        produce<NCOLS>(a, sm, cta, ncta, lane, l2_policy_evict_first());
        // this CTA has requested its last byte of weights: a programmatically dependent kernel may become resident
        pdl_launch_dependents();
        return;
    }
    if (warp == kProducerWarps) {
        pdl_wait();  // outputs (and the residual we add into) belong to earlier kernels
        epilogue<NCOLS, CW>(a, sm, cta, ncta, lane);
        if (lane == 0) dbg_stamp(a, cta, 5);
        return;
    }
    const int ctid = tid - 32 * (kProducerWarps + 1);
    const int cw = warp - (kProducerWarps + 1);
    pdl_wait();  // activations belong to the previous kernel until here
    if (a.x_mode == X_RMSNORM_F32) rms_partials<NCOLS, CW>(a, sm, ctid, cw, lane);
    const int s0 = first_slice<NCOLS>(a, cta, ncta);
    stage_slice<NCOLS, CW>(a, sm, L::x_pitch(xw), s0, ctid, cw, lane);
    if (ctid == 0) dbg_stamp(a, cta, 2);
    asm volatile("bar.sync 3, %0;" ::"r"(32 * (kProducerWarps + 1 + CW)) : "memory");
    if constexpr (NCOLS == 1) {
        if (a.full)
            consume1<CW, true>(a, sm, L::x_pitch(xw), s0, cta, ncta, ctid, cw, lane);
        else
            consume1<CW, false>(a, sm, L::x_pitch(xw), s0, cta, ncta, ctid, cw, lane);
    } else {
        consume_cols<NCOLS, CW>(a, sm, L::x_pitch(xw), s0, cta, ncta, ctid, cw, lane);
    }
    if (ctid == 0) dbg_stamp(a, cta, 4);
}

// ------------------------------------------------------------------------------------------------------
// Simple cross-check kernel: one warp per output row, 128-bit loads, scalar fp32 math like the reference.  Not the product
// path for performance; kept as an independently-written second implementation ("gemv_impl" = 0), for the < 16 trailing
// rows of an OC that is not a multiple of 16, and as the group-64 GEMV (GS = 64, reference gemv_kernel_g64,
// kernels/cuda/gemv_cuda.cu:68-123: the same QM_CUDA layout with zeros_w = zeros_width(IC, 64) and one scale / zero point per
// 64 input channels; QM_CUDA models are quantised with group 128, that slot exists for interface completeness).
// ------------------------------------------------------------------------------------------------------
template <int GS>
__global__ void w4a16_gemv_simple_kernel(const KArgs a, int total_rows) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= total_rows) return;
    int si = 0, r = row;
    if (a.nseg > 1 && r >= a.seg[0].rows) {
        r -= a.seg[0].rows;
        si = 1;
        if (a.nseg > 2 && r >= a.seg[1].rows) {
            r -= a.seg[1].rows;
            si = 2;
        }
    }
    const W4Seg &s = a.seg[si];
    const uint4 *wrow = reinterpret_cast<const uint4 *>(s.w + (size_t)r * (a.IC / 8));
    const uint32_t *zrow = s.zeros + (size_t)r * a.zeros_w;
    const __half *srow = s.scales + (size_t)r * a.sf_w;
    for (int m = 0; m < a.M; m++) {
        const __half *x = reinterpret_cast<const __half *>(a.x) + (size_t)m * a.ldx;
        float acc = 0.f;
        for (int c = lane; c < a.IC / 32; c += 32) {  // 32 nibbles per uint4
            const uint4 wv = wrow[c];
            const int G = c >> (GS == 128 ? 2 : 1);
            const float sc = __half2float(srow[G]);
            const float z = (float)((zrow[G >> 3] >> ((G & 7) * 4)) & 0xF);
            const uint32_t words[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
            for (int j = 0; j < 4; j++) {
#pragma unroll
                for (int i = 0; i < 8; i++) {
                    const float q = (float)((words[j] >> (4 * i)) & 0xF);
                    acc += (sc * (q - z)) * __half2float(x[c * 32 + j * 8 + i]);
                }
            }
        }
        acc = warp_sum(acc);
        if (lane == 0) {
            const size_t o = (size_t)m * a.ldy + row;
            if (a.epi == EPI_STORE_HALF)
                reinterpret_cast<__half *>(a.y)[o] = __float2half(acc);
            else if (a.epi == EPI_STORE_F32)
                reinterpret_cast<float *>(a.y)[o] = acc;
            else
                reinterpret_cast<float *>(a.y)[o] += acc;
        }
    }
}

}  // namespace

cudaError_t launch_w4a16_gemv_g64(Ctx *ctx, const __half *x, const uint32_t *w, const uint32_t *zeros, const __half *scales, __half *y, int M, int IC, int OC) {
    KArgs a = {};
    a.seg[0].w = w;
    a.seg[0].zeros = zeros;
    a.seg[0].scales = scales;
    a.seg[0].rows = OC;
    a.nseg = 1;
    a.IC = IC;
    a.zeros_w = zeros_width(IC, 64);
    a.sf_w = a.zeros_w * 8;
    a.M = M;
    a.ldx = IC;
    a.x = x;
    a.y = y;
    a.epi = EPI_STORE_HALF;
    a.ldy = OC;
    const int warps = 8;
    w4a16_gemv_simple_kernel<64><<<(OC + warps - 1) / warps, warps * 32, 0, ctx->stream>>>(a, OC);
    return cudaGetLastError();
}

// 2-D tensor map of one packed weight segment: uint32 [rows][IC/8], box = [box_rows][sg*16 words], no swizzle.
cudaError_t encode_w4_tmap(CUtensorMap *out, const void *w, int rows, int IC, int sg, int box_rows) {
    const TmapEncodeFn fn = tmap_encoder();
    if (!fn) return cudaErrorNotSupported;
    const cuuint64_t gdim[2] = {(cuuint64_t)(IC / 8), (cuuint64_t)rows};
    const cuuint64_t gstride[1] = {(cuuint64_t)(IC / 2)};
    const cuuint32_t box[2] = {(cuuint32_t)(sg * 16), (cuuint32_t)box_rows};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_UINT32, 2, const_cast<void *>(w), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                          CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? cudaSuccess : cudaErrorInvalidValue;
}

// 3-D view [group][row][64 B] of the same matrix: a box {64 B, box_rows, sg groups} lands in shared memory group-major with the rows of a group 64 B apart,
// so the 16 rows x 64 B of one (tile, group) unit are 1 KiB contiguous and a quarter-warp's LDS.128 covers 128 consecutive bytes (no bank conflicts)
cudaError_t encode_w4_tmap_units(CUtensorMap *out, const void *w, int rows, int IC, int sg, int box_rows) {
    const TmapEncodeFn fn = tmap_encoder();
    if (!fn) return cudaErrorNotSupported;
    const cuuint64_t gdim[3] = {16, (cuuint64_t)rows, (cuuint64_t)(IC / 128)};
    const cuuint64_t gstride[2] = {(cuuint64_t)(IC / 2), 64};
    const cuuint32_t box[3] = {16, (cuuint32_t)box_rows, (cuuint32_t)sg};
    const cuuint32_t estr[3] = {1, 1, 1};
    const CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_UINT32, 3, const_cast<void *>(w), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                          CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? cudaSuccess : cudaErrorInvalidValue;
}

namespace {

KArgs make_kargs(Ctx *ctx, const W4GemvParams &p, int *total_rows) {
    KArgs a;
    for (int i = 0; i < 3; i++) a.seg[i] = p.seg[i < p.nseg ? i : 0];
    a.nseg = p.nseg;
    a.pair_mode = p.pair_mode;
    a.IC = p.IC;
    a.NG = p.IC / kW4Group;
    a.zeros_w = zeros_width(p.IC, kW4Group);
    a.sf_w = a.zeros_w * 8;
    int rows = 0;
    for (int i = 0; i < p.nseg; i++) rows += p.seg[i].rows;
    *total_rows = rows;
    a.num_tiles = rows / 16;
    a.M = p.M;
    a.ldx = p.ldx ? p.ldx : p.IC;
    a.x_mode = p.x_mode;
    a.x = p.x;
    a.gamma = p.gamma;
    a.eps = p.eps;
    a.y = p.y;
    a.epi = p.epi;
    a.ldy = p.ldy ? p.ldy : (p.pair_mode ? rows / 2 : rows);
    a.partials = ctx->gemv_partials;
    a.counters = ctx->gemv_counters;
    a.dbg = ctx->gemv_dbg;
    a.pdl_early = 0;
    a.nst = kStages;
    a.atomic_add = (p.atomic_residual && p.epi == EPI_ADD_F32 && !p.pair_mode) ? 1 : 0;
    a.aligned = 0;
    a.sg = a.NG < kStageGroups ? a.NG : kStageGroups;
    a.full = (a.NG % kStageGroups == 0) ? 1 : 0;
    a.sl = a.NG;
    a.nsl = 1;
    return a;
}

// The one rule for what fits in shared memory: the deepest TMA ring of 2..max_nst stages next to `xw` staged activation elements per column,
// within `budget` bytes; 0 when not even two stages fit.
template <int NCOLS, int CW>
int ring_fit(int IC, int xw, int budget, int max_nst) {
    for (int nst = max_nst; nst >= 2; nst--)
        if ((int)Layout<NCOLS, CW>::bytes(IC, nst, xw) <= budget) return nst;
    return 0;
}

// K-slice of the multi-column kernel: the whole row when it fits next to a kStages ring, else the widest whole number of 16-group stages
// that does (at least one stage's worth of groups, with the shallowest ring)
template <int CW>
int pick_slice(int IC, int budget) {
    const int NG = IC / kW4Group;
    if (ring_fit<8, CW>(IC, IC, budget, kStages) == kStages) return NG;
    for (int sl = (NG - 1) / kStageGroups * kStageGroups; sl >= kStageGroups; sl -= kStageGroups)
        if (ring_fit<8, CW>(IC, sl * kW4Group, budget, kStages) >= kStages) return sl;
    return ring_fit<8, CW>(IC, kStageGroups * kW4Group, budget, kStages) ? kStageGroups : 0;
}

template <int NCOLS, int CW>
cudaError_t launch_mma(Ctx *ctx, const KArgs &a_in, bool pdl) {
    KArgs a = a_in;
    const int xw = a.sl * kW4Group;
    if (!ring_fit<NCOLS, CW>(a.IC, xw, ctx->smem_optin, kStages)) return cudaErrorInvalidConfiguration;
    static DeviceOnce attr_once;  // per template instantiation
    if (attr_once.pending(ctx->device)) {
        cudaError_t e = cudaFuncSetAttribute(w4a16_gemv_kernel<NCOLS, CW>, cudaFuncAttributeMaxDynamicSharedMemorySize, ctx->smem_optin);
        if (e != cudaSuccess) return e;
        attr_once.done(ctx->device);
    }
    const long long U = (long long)a.num_tiles * a.NG;
    // Two co-resident CTAs per SM (two independent TMA rings, 16 consumer warps) stream faster than one on large
    // matrices but double the per-launch activation
    // staging, which dominates small launches and long rows: only used when every CTA still gets >= 128 units and the
    // activation vector is short.  "gemv_ctas_per_sm" > 1 forces it.
    int per_sm = ctx->gemv_ctas_per_sm;
    a.pdl_early = (pdl && ctx->pdl_early) ? 1 : 0;
    const bool allow2 = !(pdl && ctx->pdl_early == 2);  // an early-resident dependent needs the second CTA slot of every SM
    if (allow2 && per_sm == 1 && NCOLS == 1 && CW == 8 && a.IC <= 8192 && U >= (long long)ctx->num_sms * 2 * 128) per_sm = 2;
    int nc = ctx->num_sms * per_sm;
    if (nc > ctx->gemv_max_ctas) nc = ctx->gemv_max_ctas;
    const long long cuts = a.full ? U / kStageGroups : U;  // stream-K cuts fall on whole stages when every stage is full
    if ((long long)nc > cuts) nc = (int)cuts;
    if (a.nsl > 1) {
        // CTA ranges are cut at (slice, tile) segment boundaries: one fix-up record per segment
        if ((long long)nc > (long long)a.num_tiles * a.nsl) nc = a.num_tiles * a.nsl;
        if ((long long)a.num_tiles * a.nsl > ctx->gemv_partial_records) return cudaErrorInvalidValue;  // launch_w4a16_gemv reserves them
    }
    // Epilogues that need a single ordered writer per output (stores, SiLU*mul, deterministic residual) avoid split
    // tiles altogether when there is at least one whole tile per CTA: the fix-up protocol adds a tail to every
    // launch, more than the <= 1/tiles_per_cta imbalance it removes.  Slice-major units have no whole tiles.
    a.aligned = (!a.atomic_add && a.num_tiles >= nc && a.nsl == 1) ? 1 : 0;
    // Ring depth = bytes in flight per SM.  HBM latency under load (~1.2 us) x 3.35 TB/s / 132 SMs = ~30 KB must be in flight per SM
    // all the time, and a slot is only re-requested after it was consumed: the deepest ring that fits the per-CTA share of shared
    // memory (1 KiB per CTA is reserved by the driver), at most kMaxStages and no more stages than the CTA has work for.
    {
        const int budget = ctx->smem_optin / per_sm - (per_sm > 1 ? 1024 : 0);
        int nst = ctx->gemv_stages > 0 ? ctx->gemv_stages : kMaxStages;
        if (nst > kMaxStages) nst = kMaxStages;
        const int fit = ring_fit<NCOLS, CW>(a.IC, xw, budget, nst);
        nst = fit ? fit : 2;
        const long long stages_per_cta = (U / nc + a.sg - 1) / a.sg + 1;
        if (nst > stages_per_cta && stages_per_cta >= 2) nst = (int)stages_per_cta;
        a.nst = nst;
    }
    const size_t smem = Layout<NCOLS, CW>::bytes(a.IC, a.nst, xw);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(nc);
    cfg.blockDim = dim3(32 * (kProducerWarps + 1 + CW));
    cfg.dynamicSmemBytes = smem;
    cfg.stream = ctx->stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, w4a16_gemv_kernel<NCOLS, CW>, a);
}

}  // namespace

cudaError_t launch_w4a16_gemv_simple(Ctx *ctx, const W4GemvParams &p) {
    if (p.pair_mode || p.x_mode != X_HALF) return cudaErrorNotSupported;
    int rows;
    KArgs a = make_kargs(ctx, p, &rows);
    const int warps = 8;
    w4a16_gemv_simple_kernel<kW4Group><<<(rows + warps - 1) / warps, warps * 32, 0, ctx->stream>>>(a, rows);
    return cudaGetLastError();
}

namespace {
// 16 consumer warps pay off on long rows (down_proj, IC = 14336), where one CTA per SM stages a long activation
// vector and the 2-CTA mode is off; 8 warps (x 2 CTAs on large launches) everywhere else
int consumer_warps(const Ctx *ctx, const W4GemvParams &p) {
    return ctx->gemv_consumer_warps == 16 ? 16 : (ctx->gemv_consumer_warps == 8 ? 8 : (p.IC > 8192 && p.M == 1 ? 16 : 8));
}
// K-slice of a multi-column launch (groups; 0 = nothing fits)
int slice_of(const Ctx *ctx, const W4GemvParams &p) {
    return consumer_warps(ctx, p) == 16 ? pick_slice<16>(p.IC, ctx->smem_optin) : pick_slice<8>(p.IC, ctx->smem_optin);
}
}  // namespace

long long w4a16_gemv_fixup_records(const Ctx *ctx, const W4GemvParams &p) {
    if (p.M <= 1 || p.IC < kW4Group) return 0;
    const int NG = p.IC / kW4Group, sl = slice_of(ctx, p);
    if (sl <= 0 || sl >= NG) return 0;
    int rows = 0;
    for (int i = 0; i < p.nseg && i < 3; i++) rows += p.seg[i].rows;
    return (long long)(rows / 16) * ((NG + sl - 1) / sl);
}

cudaError_t gemv_partials_reserve(Ctx *ctx, long long records) {
    if (records <= ctx->gemv_partial_records) return cudaSuccess;
    if (records > (1ll << 24)) return cudaErrorInvalidValue;
    cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
    cudaError_t e = cudaStreamIsCapturing(ctx->stream, &st);
    if (e != cudaSuccess) return e;
    if (st != cudaStreamCaptureStatusNone) return cudaErrorStreamCaptureUnsupported;  // grow it with one launch outside of capture first
    float *p = nullptr;
    e = cudaMalloc(&p, (size_t)records * 16 * 8 * sizeof(float));
    if (e != cudaSuccess) return e;
    e = cudaFree(ctx->gemv_partials);  // synchronises: no launch still uses the old records
    if (e != cudaSuccess) {
        cudaFree(p);
        return e;
    }
    ctx->gemv_partials = p;
    ctx->gemv_partial_records = (int)records;
    ctx->option_gen++;  // graphs captured on this context hold the old pointer
    return cudaSuccess;
}

cudaError_t launch_w4a16_gemv(Ctx *ctx, const W4GemvParams &p) {
    if (p.M < 1 || p.M > 8 || p.IC % kW4Group || p.nseg < 1 || p.nseg > 3) return cudaErrorInvalidValue;
    int rows;
    KArgs a = make_kargs(ctx, p, &rows);
    for (int i = 0; i < p.nseg; i++)
        if (p.seg[i].rows % (p.pair_mode ? 8 : 16)) return cudaErrorInvalidValue;
    if (p.pair_mode && (p.nseg != 2 || p.seg[0].rows != p.seg[1].rows)) return cudaErrorInvalidValue;
    if (a.num_tiles > ctx->gemv_max_tiles) return cudaErrorInvalidValue;
    for (int i = 0; i < p.nseg; i++) {
        cudaError_t e = encode_w4_tmap(&a.tmap[i], p.seg[i].w, p.seg[i].rows, p.IC, a.sg, p.pair_mode ? 8 : 16);
        if (e != cudaSuccess) return e;
    }
    const int cw = consumer_warps(ctx, p);
    if (p.M == 1) return (cw == 16) ? launch_mma<1, 16>(ctx, a, p.pdl) : launch_mma<1, 8>(ctx, a, p.pdl);
    // M = 2..8: one pass over the weights, the activation rows staged one K-slice at a time where the whole rows do not fit
    a.sl = slice_of(ctx, p);
    if (a.sl == 0) return cudaErrorInvalidConfiguration;
    a.nsl = (a.NG + a.sl - 1) / a.sl;
    if (a.nsl > kMaxSlices) return cudaErrorInvalidConfiguration;
    if (a.nsl > 1) {  // one fix-up record per (slice, row tile)
        cudaError_t e = gemv_partials_reserve(ctx, (long long)a.num_tiles * a.nsl);
        if (e != cudaSuccess) return e;
        a.partials = ctx->gemv_partials;
    }
    return (cw == 16) ? launch_mma<8, 16>(ctx, a, p.pdl) : launch_mma<8, 8>(ctx, a, p.pdl);
}

}  // namespace tce
