// w4a16_gemv_impl.cuh -- device-side roles of the W4A16 group-128 GEMV (producer / consumer / epilogue), shared by
// the stand-alone kernel (w4a16_gemv.cu) and the persistent decode kernel (decode_persistent.cu).
//
// Data contract = the reference's QM_CUDA layout (kernels/cuda/gemv_cuda.cu:140-260, quantize_methods.py:370-442):
//     w uint32[OC][IC/8] sequential nibbles, zeros uint32[OC][zeros_w] (nibble g = zero of group g),
//     scales half[OC][zeros_w*8];   y[m][oc] = sum_ic s[oc,g] * (q[oc,ic] - z[oc,g]) * x[m][ic]
//
//  * work unit = (16-row tile, one 128-k group) = 1 KiB of packed weights; the units of a launch are cut into equal
//    contiguous per-CTA ranges (stream-K) or, for epilogues that need one ordered writer, at row-tile boundaries.
//  * producer (1 warp, 1 elected lane): ONE 2-D TMA tensor copy (UTMALDG) per stage moves the [16 rows x <=16 groups]
//    weight box into a ring of KArgs::nst stages (8 by default) guarded by full/empty mbarriers, L2 evict-first; the tile's
//    scales/zeros slabs (1-D bulk copies, UBLKCP) ride on the first stage's barrier.  Producers depend on nothing but the weights,
//    so they run ahead of everything else (in particular of the consumers' activation staging).
//  * consumers (CW warps): 128-bit LDS of the packed nibbles; activations held as four int8 planes (32-bit block fixed point per
//    128-group, exact integer accumulation); mma.sync.m16n8k32 u8 x s8 -> s32; per-group epilogue
//    tot += (s * step) * (acc - z * sum_X).  One activation row (decode, consume1): the four planes ride in MMA columns 0..3 and
//    nibbles become bytes with one mask each (even slots w & 0x0f0f0f0f, odd slots w & 0xf0f0f0f0 = 16 x nibble, shifted back
//    after accumulation): 4 IMMAs per (16 rows x 128 k).  Up to 8 rows (consume<8>): the 8 MMA columns carry the rows, planes in
//    separate MMAs, (w >> 4) & 0x0f0f0f0f for the odd slots.
//  * tile partials go to the epilogue warp through a triple-buffered smem slot + mbarrier (consumers never wait for
//    each other); the epilogue warp runs the fused epilogue (fp16/fp32 store, residual +=, SiLU(gate)*up), the
//    RED.ADD residual path or the ordered stream-K fix-up.
//  * fused prologue: RMSNorm of an fp32 residual stream (LlamaRMSNorm semantics) + activation quantisation.
#pragma once
#include "common.cuh"
#include "kernels.h"

namespace tce {
namespace gemv {

constexpr int kStageGroups = 16;               // 128-k groups per pipeline stage (per row: up to 1024 B)
constexpr int kStageBytes = 16 * kStageGroups * 64;  // 16 KiB: dense [16 rows][sg*64 B] box written by ONE 2-D TMA instruction
constexpr int kStages = 4;         // default ring depth (persistent kernel); the per-op kernel picks the deepest ring that fits (KArgs::nst)
constexpr int kMaxStages = 12;
constexpr int kRedBufs = 3;
constexpr float kActQ = 2130706432.f;  // 127 * 2^24: activation fixed-point full scale (four balanced base-256 digits = int8 planes)
constexpr int kMaxSlices = 16;  // K-slices of the multi-column kernel (the fix-up sums them from registers)
constexpr int kProducerWarps = 1;        // a stage is one UTMALDG (two in gate/up pair mode): a single elected lane keeps up
// per-tile scales/zeros slabs in flight: ring depth + 1 (a tile spans >= 1 stage)

struct KArgs {
    W4Seg seg[3];
    int nseg, pair_mode;
    int IC, NG, zeros_w, sf_w;
    int num_tiles;
    int M, ldx, x_mode;
    const void *x;
    const float *gamma;
    float eps;
    void *y;
    int epi, ldy;
    float *partials;
    unsigned *counters;
    int sg;          // groups per stage = min(16, NG); the stage row pitch is sg*64 bytes (dense TMA box)
    int aligned;     // 1: CTA ranges are cut at row-tile boundaries (no split tiles, no fix-up)
    int atomic_add;  // 1: EPI_ADD_F32 partial tiles use RED.ADD.F32 instead of the ordered fix-up
    unsigned long long *dbg;  // optional per-CTA phase timestamps (globaltimer ns), 8 slots per CTA
    int full;        // 1: every stage carries 16 whole groups (IC % 2048 == 0): the single-column consumer drops its bounds checks
    int nst;         // TMA ring depth of this launch (4..kMaxStages stages of 16 KiB)
    int pdl_early;   // 1: griddepcontrol.launch_dependents at kernel entry instead of after the last weight request
    // multi-column kernel: the activation columns are staged one K-slice at a time.  A slice is `sl` groups (a multiple of kStageGroups, or NG)
    // and the units are ordered slice-major, u = T*sl*s + rt*len(s) + (g - s*sl): a CTA stages only the slices its range touches
    int sl, nsl;
    // one 2-D tensor map per weight segment: uint32 [rows][IC/8], box = [16 (8 in pair mode) rows][sg*16 words]
    alignas(64) CUtensorMap tmap[3];
};

struct RowRef {
    const uint8_t *w;
    const uint32_t *z;
    const __half *s;
};

// source row `l` (0..15) of row tile `rt`
TCE_DEVINL RowRef tile_row(const KArgs &a, int rt, int l) {
    int si = 0, r;
    if (a.pair_mode) {
        si = l >> 3;
        r = rt * 8 + (l & 7);
    } else {
        r = rt * 16 + l;
        if (a.nseg > 1 && r >= a.seg[0].rows) {
            r -= a.seg[0].rows;
            si = 1;
            if (a.nseg > 2 && r >= a.seg[1].rows) {
                r -= a.seg[1].rows;
                si = 2;
            }
        }
    }
    const W4Seg &s = a.seg[si];
    RowRef ref;
    ref.w = reinterpret_cast<const uint8_t *>(s.w) + (size_t)r * (a.IC / 2);
    ref.z = s.zeros + (size_t)r * a.zeros_w;
    ref.s = s.scales + (size_t)r * a.sf_w;
    return ref;
}

TCE_DEVINL void dbg_stamp(const KArgs &a, int cta, int k) {
    if (a.dbg) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        a.dbg[(size_t)cta * 8 + k] = t;
    }
}

// shared-memory layout (offsets from a 128-B aligned base)
template <int NCOLS, int CW>
struct Layout {
    static constexpr int kXPad = (NCOLS > 1) ? 64 : 0;  // column pitch = 64 (mod 128) B for the per-column B loads
    static constexpr int kVals = 16 * NCOLS;
    // four int8 planes per activation (32-bit block fixed point): planes (p3, p2) interleaved in region A (2 B per element),
    // planes (p1, p0) in region B that follows region A of the same column
    static __host__ __device__ int x_pitch(int IC) { return IC * 4 + kXPad; }
    // one meta slot = scales half[16][zeros_w*8] followed by zeros uint32[16][zeros_w] = 320 * zeros_w bytes
    static __host__ __device__ int meta_slot_bytes(int IC) { return 320 * (((IC / 128) + 7) / 8); }
    static __host__ __device__ size_t off_meta(int nst) { return (size_t)nst * kStageBytes; }
    static __host__ __device__ size_t off_xs(int IC, int nst) { return off_meta(nst) + (size_t)(nst + 1) * meta_slot_bytes(IC); }
    // `xw`: activation elements staged per column (IC, or one K-slice of the multi-column kernel)
    static __host__ __device__ size_t off_gx(int IC, int nst, int xw) { return off_xs(IC, nst) + (size_t)NCOLS * x_pitch(xw); }
    // gx: float step[NCOLS][NG] followed by int gsum[NCOLS][NG][2] = {256 * sum(p3) + sum(p2), 256 * sum(p1) + sum(p0)}
    static __host__ __device__ size_t off_red(int IC, int nst, int xw) { return off_gx(IC, nst, xw) + (size_t)3 * NCOLS * (IC / 128) * sizeof(float); }
    static __host__ __device__ size_t off_rms(int IC, int nst, int xw) { return off_red(IC, nst, xw) + (size_t)kRedBufs * CW * kVals * sizeof(float); }
    static __host__ __device__ size_t off_bar(int IC, int nst, int xw) { return (off_rms(IC, nst, xw) + (size_t)NCOLS * CW * sizeof(float) + 15) & ~(size_t)15; }
    static __host__ __device__ size_t bytes(int IC, int nst, int xw) { return off_bar(IC, nst, xw) + (2 * nst + 2 * kRedBufs) * sizeof(uint64_t) + 16; }
    static __host__ __device__ size_t off_gx(int IC, int nst) { return off_gx(IC, nst, IC); }
    static __host__ __device__ size_t off_red(int IC, int nst) { return off_red(IC, nst, IC); }
    static __host__ __device__ size_t off_rms(int IC, int nst) { return off_rms(IC, nst, IC); }
    static __host__ __device__ size_t off_bar(int IC, int nst) { return off_bar(IC, nst, IC); }
    static __host__ __device__ size_t bytes(int IC, int nst = kStages) { return bytes(IC, nst, IC); }
};

struct Smem {
    uint8_t *stages, *meta, *xs;
    float *gx;
    int *gsum;
    float *red, *rms;
    uint64_t *full_bar, *empty_bar, *red_full, *red_empty;
    int meta_bytes;
    int nst;  // ring depth
};

// `IC` here is the LARGEST IC the kernel will see (the persistent kernel carves once for all phases)
template <int NCOLS, int CW>
TCE_DEVINL Smem carve(uint8_t *base, int IC, int nst, int xw) {
    using L = Layout<NCOLS, CW>;
    Smem s;
    s.nst = nst;
    s.stages = base;
    s.meta = base + L::off_meta(nst);
    s.xs = base + L::off_xs(IC, nst);
    s.gx = reinterpret_cast<float *>(base + L::off_gx(IC, nst, xw));
    s.gsum = reinterpret_cast<int *>(s.gx + (size_t)NCOLS * (IC / 128));
    s.red = reinterpret_cast<float *>(base + L::off_red(IC, nst, xw));
    s.rms = reinterpret_cast<float *>(base + L::off_rms(IC, nst, xw));
    s.full_bar = reinterpret_cast<uint64_t *>(base + L::off_bar(IC, nst, xw));
    s.empty_bar = s.full_bar + nst;
    s.red_full = s.empty_bar + nst;
    s.red_empty = s.red_full + kRedBufs;
    s.meta_bytes = L::meta_slot_bytes(IC);
    return s;
}
template <int NCOLS, int CW>
TCE_DEVINL Smem carve(uint8_t *base, int IC, int nst = kStages) { return carve<NCOLS, CW>(base, IC, nst, IC); }

template <int CW>
TCE_DEVINL void init_barriers(const Smem &sm) {  // one thread
    for (int s = 0; s < sm.nst; s++) {
        mbar_init(&sm.full_bar[s], 1);
        mbar_init(&sm.empty_bar[s], CW);
    }
#pragma unroll
    for (int s = 0; s < kRedBufs; s++) {
        mbar_init(&sm.red_full[s], CW);
        mbar_init(&sm.red_empty[s], 1);
    }
    mbar_fence_init();
}

// same, spread over the lanes of one warp (one barrier pair per lane instead of ~14 dependent inits on one thread)
template <int CW>
TCE_DEVINL void init_barriers_warp(const Smem &sm, int lane) {
    if (lane < sm.nst) {
        mbar_init(&sm.full_bar[lane], 1);
        mbar_init(&sm.empty_bar[lane], CW);
    } else if (lane >= 16 && lane < 16 + kRedBufs) {
        mbar_init(&sm.red_full[lane - 16], CW);
        mbar_init(&sm.red_empty[lane - 16], 1);
    }
    mbar_fence_init();
    __syncwarp();
}

// pipeline positions; every role keeps its own copy and all copies advance identically because every role walks the
// same (tile, stage) sequence
struct RingState {
    int stage = 0;
    uint32_t phase = 0;
    int mslot = 0;
};
struct RedState {
    int rb = 0;
    uint32_t rphase = 0;
};

TCE_DEVINL StreamK make_sk(const KArgs &a, int ncta) {
    StreamK sk;
    sk.U = (long long)a.num_tiles * a.NG;
    sk.nc = ncta;
    sk.NG = a.NG;
    sk.aligned = a.aligned;
    sk.T = a.num_tiles;
    sk.gran = a.full ? kStageGroups : 1;  // whole 16-group stages per CTA: consume1<FULL> never sees a partial stage
    return sk;
}

// ------------------------------------------------------------------------------------------------------------------
// producer warp: streams this CTA's unit range into the ring.  Warp-convergent, lane 0 issues.  `a` must be the
// original argument block (kernel parameter or global memory), never a local copy: the TMA unit reads the tensor map
// through its address.
// ------------------------------------------------------------------------------------------------------------------
TCE_DEVINL void produce(const KArgs &a, const Smem &sm, RingState &rs, int cta, int ncta, int lane, uint64_t policy) {
    const StreamK sk = make_sk(a, ncta);
    const uint32_t leader = (lane == 0) ? 1u : 0u;
    const uint32_t meta_bytes_cur = 320u * a.zeros_w;  // bytes actually copied for this IC (<= sm.meta_bytes)
    const uint32_t box_bytes = 16u * a.sg * 64u;       // a stage always receives the full box (out-of-range parts are zero-filled)
    int u = (int)sk.start(cta);
    const int uend = (int)sk.start(cta + 1);
    int rt = u / a.NG;
    int gb = u - rt * a.NG;
    while (u < uend) {
        const int ge = min(a.NG, gb + (uend - u));
        // segment / row of the tile (warp-uniform)
        int si0 = 0, row0 = rt * 16, si1 = 0, row1 = 0;
        if (a.pair_mode) {
            row0 = rt * 8;
            si1 = 1;
            row1 = rt * 8;
        } else if (a.nseg > 1 && row0 >= a.seg[0].rows) {
            row0 -= a.seg[0].rows;
            si0 = 1;
            if (a.nseg > 2 && row0 >= a.seg[1].rows) {
                row0 -= a.seg[1].rows;
                si0 = 2;
            }
        }
        const RowRef r0 = tile_row(a, rt, 0), r8 = tile_row(a, rt, 8);
        uint8_t *mdst = sm.meta + (size_t)rs.mslot * sm.meta_bytes;
        bool first = true;
        for (int g0 = gb; g0 < ge; g0 += a.sg) {
            mbar_wait(&sm.empty_bar[rs.stage], rs.phase ^ 1);
            uint64_t *bar = &sm.full_bar[rs.stage];
            mbar_arrive_expect_tx_pred(bar, box_bytes + (first ? meta_bytes_cur : 0u), leader);
            uint8_t *dst = sm.stages + (size_t)rs.stage * kStageBytes;
            if (a.pair_mode) {
                tma_load_2d_pred(dst, &a.tmap[si0], g0 * 16, row0, bar, policy, leader);
                tma_load_2d_pred(dst + 8 * a.sg * 64, &a.tmap[si1], g0 * 16, row1, bar, policy, leader);
            } else {
                tma_load_2d_pred(dst, &a.tmap[si0], g0 * 16, row0, bar, policy, leader);
            }
            if (first) {
                // this tile's scales / zeros slabs ride on the full barrier of its first stage
                const uint32_t sb = 8u * a.sf_w * 2u, zb = 8u * a.zeros_w * 4u;
                bulk_g2s_pred(mdst, r0.s, sb, bar, policy, leader);
                bulk_g2s_pred(mdst + sb, r8.s, sb, bar, policy, leader);
                bulk_g2s_pred(mdst + 2 * sb, r0.z, zb, bar, policy, leader);
                bulk_g2s_pred(mdst + 2 * sb + zb, r8.z, zb, bar, policy, leader);
            }
            __syncwarp();
            first = false;
            if (++rs.stage == sm.nst) {
                rs.stage = 0;
                rs.phase ^= 1;
            }
        }
        if (++rs.mslot == sm.nst + 1) rs.mslot = 0;
        u += ge - gb;
        rt++;
        gb = 0;
    }
}

// the finished sums of one row tile (lane l holds values idx = l + 32*i, idx = row*NCOLS + col): the fused epilogue
template <int NCOLS, int VPL>
TCE_DEVINL void finish_tile(const KArgs &a, const float (&v)[VPL], int rt, int lane) {
    constexpr int kVals = 16 * NCOLS;
    if (a.pair_mode) {
        // rows 0-7 = gate, rows 8-15 = up of the same output channel: y = SiLU(gate) * up
        // (reference SiLuMul_half, llm/src/nn_modules/cuda/Int4llamaDecoderLayer.cu:21-30; fp32 here)
        if (NCOLS == 1) {
            const float up = __shfl_down_sync(0xffffffffu, v[0], 8);
            if (lane < 8) {
                const float gte = v[0];
                const float act = gte / (1.f + __expf(-gte));
                reinterpret_cast<__half *>(a.y)[(size_t)rt * 8 + lane] = __float2half(act * up);
            }
        } else {
            // idx = row*8 + col: lane holds rows 4i + lane/8; the partner row+8 is slot i+2 of the same lane
#pragma unroll
            for (int i = 0; i < VPL / 2; i++) {
                const int row = 4 * i + (lane >> 3), col = lane & 7;
                if (col < a.M) {
                    const float gte = v[i], up = v[i + VPL / 2];
                    const float act = gte / (1.f + __expf(-gte));
                    reinterpret_cast<__half *>(a.y)[(size_t)col * a.ldy + (size_t)rt * 8 + row] = __float2half(act * up);
                }
            }
        }
    } else {
#pragma unroll
        for (int i = 0; i < VPL; i++) {
            const int idx = lane + 32 * i;
            const int row = idx / NCOLS, col = idx % NCOLS;
            if (idx < kVals && col < a.M) {
                const size_t o = (size_t)col * a.ldy + (size_t)rt * 16 + row;
                if (a.epi == EPI_STORE_HALF)
                    reinterpret_cast<__half *>(a.y)[o] = __float2half(v[i]);
                else if (a.epi == EPI_STORE_F32)
                    reinterpret_cast<float *>(a.y)[o] = v[i];
                else
                    reinterpret_cast<float *>(a.y)[o] += v[i];
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------------------------
// epilogue warp: reduces the CW consumer partials of every tile this CTA touches, then either finishes the tile or
// takes part in the stream-K fix-up.  Lane l owns values idx = l + 32*i  (idx = row*NCOLS + col).
// ------------------------------------------------------------------------------------------------------------------
template <int NCOLS, int CW>
TCE_DEVINL void epilogue(const KArgs &a, const Smem &sm, RedState &es, int cta, int ncta, int lane) {
    constexpr int kVals = 16 * NCOLS;
    constexpr int VPL = (kVals + 31) / 32;  // values per lane
    const StreamK sk = make_sk(a, ncta);
    const long long u0 = sk.start(cta);
    int u = (int)u0;
    const int uend = (int)sk.start(cta + 1);
    int rt = u / a.NG;
    int gb = u - rt * a.NG;
    while (u < uend) {
        const int ge = min(a.NG, gb + (uend - u));
        const bool full_tile = (gb == 0 && ge == a.NG);
        mbar_wait(&sm.red_full[es.rb], es.rphase);
        const float *rbuf = sm.red + (size_t)es.rb * CW * kVals;
        float v[VPL];
#pragma unroll
        for (int i = 0; i < VPL; i++) {
            const int idx = lane + 32 * i;
            float acc = 0.f;
            if (idx < kVals) {
#pragma unroll
                for (int w = 0; w < CW; w++) acc += rbuf[w * kVals + idx];
            }
            v[i] = acc;
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&sm.red_empty[es.rb]);
        if (++es.rb == kRedBufs) {
            es.rb = 0;
            es.rphase ^= 1;
        }
        bool do_final = full_tile;
        if (!full_tile && a.atomic_add) {
            // residual accumulate: every contributor of a split tile adds its partial straight into the fp32 residual
            // with RED.ADD (fire and forget: no fence, no counter, nothing on the critical path).  The order of the
            // <= 3 partial adds is not fixed, so the last bit of the residual may vary run to run.
#pragma unroll
            for (int i = 0; i < VPL; i++) {
                const int idx = lane + 32 * i;
                const int row = idx / NCOLS, col = idx % NCOLS;
                if (idx < kVals && col < a.M) atomicAdd(reinterpret_cast<float *>(a.y) + (size_t)col * a.ldy + (size_t)rt * 16 + row, v[i]);
            }
        } else if (!full_tile) {
            // stream-K fix-up: park the partial; the last contributor to arrive sums all of them in CTA order
            const long long tb = (long long)rt * a.NG;
            const int c_first = sk.cta_of(tb);
            const int c_last = sk.cta_of(tb + a.NG - 1);
            const int rec = (u0 >= tb) ? 0 : 1;  // 0: this tile holds my first unit, 1: it is my tail tile
            float *mine = a.partials + ((size_t)cta * 2 + rec) * kVals;
#pragma unroll
            for (int i = 0; i < VPL; i++)
                if (lane + 32 * i < kVals) mine[lane + 32 * i] = v[i];
            __threadfence();
            __syncwarp();
            int last = 0;
            if (lane == 0) {
                const unsigned prev = atomicAdd(&a.counters[rt], 1u);
                last = (prev == (unsigned)(c_last - c_first)) ? 1 : 0;
                if (last) a.counters[rt] = 0;  // every contributor has arrived: re-arm for the next launch
            }
            last = __shfl_sync(0xffffffffu, last, 0);
            do_final = last != 0;
            if (do_final) {
                __threadfence();
#pragma unroll
                for (int i = 0; i < VPL; i++) {
                    const int idx = lane + 32 * i;
                    float acc = 0.f;
                    if (idx < kVals) {
                        for (int c = c_first; c <= c_last; c++) {
                            const int r = (sk.start(c) >= tb) ? 0 : 1;
                            acc += ldg_cg_f32(a.partials + ((size_t)c * 2 + r) * kVals + idx);
                        }
                    }
                    v[i] = acc;
                }
            }
        }
        if (do_final) finish_tile<NCOLS>(a, v, rt, lane);
        u += ge - gb;
        rt++;
        gb = 0;
    }
}

// quantise + stage one 8-element unit (v) of one activation column: xcol = the column's plane buffer, gx / gsum = the column's per-group
// step and integer sums.  Must be called by all 32 lanes of a warp (half-warp shuffles); `valid` masks the stores.
// Mirror of a unit into the partner CTA of a cluster (persistent decode kernel, pair staging): shared::cluster addresses of the partner's
// plane buffer, group steps / sums and of the mbarrier that counts the bytes it receives (st.async completes them as transactions).
struct PairDst {
    uint32_t xs, gx, gsum, bar;
};
TCE_DEVINL void st_async_b32(uint32_t raddr, uint32_t v, uint32_t rbar) {
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];" ::"r"(raddr), "r"(v), "r"(rbar) : "memory");
}

template <int NCOLS, bool PAIR = false>
TCE_DEVINL void emit_unit(uint8_t *xcol, int IC, float *gx, int *gsum, int ui, bool valid, const float (&v)[8], int lane, const PairDst *pd = nullptr) {
    // Activations enter the integer tensor path as 32-bit block fixed point: per 128-group,
    // X = rint(x * Q / max|x|), Q = 127 * 2^24, X = 2^24*p3 + 2^16*p2 + 2^8*p1 + p0  (four int8 planes = the balanced base-256 digits of
    // X, p3 in [-127,127], the others in [-128,127]).  |x - step*X| <= max(|x| * 2^-24, max|x_group| * 2^-32): every fp16 activation whose
    // magnitude is within 2^20 of the largest of its group keeps all of its 11 significand bits, i.e. the planes carry what the reference's
    // exact fp16 -> fp32 conversion carries (gemv_cuda.cu:181-184) unless a group spans more than 6 decades.  The integer dot products that follow are
    // exact.  The extra planes cost no MMA: the four planes ride in MMA columns 0..3 of the same instruction.
    float amax = 0.f;
#pragma unroll
    for (int i = 0; i < 8; i++) amax = fmaxf(amax, fabsf(v[i]));
    // group maximum over the 16 lanes that hold the group: non-negative floats order like their bit patterns
    const unsigned half_mask = 0xFFFFu << (lane & 16);
    amax = __uint_as_float(__reduce_max_sync(half_mask, __float_as_uint(amax)));
    const float qinv = (amax > 0.f) ? (kActQ / amax) : 0.f;
    // balanced base-256 digits of X in one go: (X + 0x80808080) ^ 0x80808080 holds p3..p0 as signed bytes (the carries between the
    // digits are the carries of the addition)
    uint32_t Z[8];
#pragma unroll
    for (int i = 0; i < 8; i++) Z[i] = ((uint32_t)__float2int_rn(v[i] * qinv) + 0x80808080u) ^ 0x80808080u;
    // B-fragment order of mma.m16n8k32: k-slots 4t..4t+3 <- elements (0,2,4,6) of the word (the bytes of
    // w & 0x0f0f0f0f), k-slots 16+4t.. <- elements (1,3,5,7) (the bytes of (w>>4) & 0x0f0f0f0f).  4x4 byte transposes:
    uint32_t o3e, o2e, o1e, o0e, o3o, o2o, o1o, o0o;
    {
        const uint32_t t0 = __byte_perm(Z[0], Z[2], 0x6240), t1 = __byte_perm(Z[0], Z[2], 0x7351);  // (p0a p0b p2a p2b), (p1a p1b p3a p3b)
        const uint32_t u0 = __byte_perm(Z[4], Z[6], 0x6240), u1 = __byte_perm(Z[4], Z[6], 0x7351);
        o0e = __byte_perm(t0, u0, 0x5410); o2e = __byte_perm(t0, u0, 0x7632);
        o1e = __byte_perm(t1, u1, 0x5410); o3e = __byte_perm(t1, u1, 0x7632);
    }
    {
        const uint32_t t0 = __byte_perm(Z[1], Z[3], 0x6240), t1 = __byte_perm(Z[1], Z[3], 0x7351);
        const uint32_t u0 = __byte_perm(Z[5], Z[7], 0x6240), u1 = __byte_perm(Z[5], Z[7], 0x7351);
        o0o = __byte_perm(t0, u0, 0x5410); o2o = __byte_perm(t0, u0, 0x7632);
        o1o = __byte_perm(t1, u1, 0x5410); o3o = __byte_perm(t1, u1, 0x7632);
    }
    // digit sums of the unit (signed byte dot products with 1)
    const int s3 = __dp4a((int)o3e, 0x01010101, __dp4a((int)o3o, 0x01010101, 0)), s2 = __dp4a((int)o2e, 0x01010101, __dp4a((int)o2o, 0x01010101, 0));
    const int s1 = __dp4a((int)o1e, 0x01010101, __dp4a((int)o1o, 0x01010101, 0)), s0 = __dp4a((int)o0e, 0x01010101, __dp4a((int)o0o, 0x01010101, 0));
    int sxh = s3 * 256 + s2, sxl = s1 * 256 + s0;
    const int G = ui >> 4, tj = ui & 15;  // ui = G*16 + 4*t + j
    if (NCOLS == 1) {
        // single-column layout (consume1).  Region A (planes p3 | p2) and region B (at byte IC*2, planes p1 | p0), each per group
        // 256 B = [parity: even | odd nibble slots][t][plane][word j].  One LDS.128 hands lane (t, plane) the B operands of both MMAs of a
        // parity; the chunks a quarter-warp loads are contiguous (conflict free).
        if (valid) {
            uint32_t *dst = reinterpret_cast<uint32_t *>(xcol + (size_t)G * 256 + (size_t)(tj >> 2) * 32) + (tj & 3);
            dst[0] = o3e;       // even slots, p3
            dst[4] = o2e;       // even slots, p2
            dst[32] = o3o;      // odd slots, p3
            dst[36] = o2o;      // odd slots, p2
            uint32_t *dl = reinterpret_cast<uint32_t *>(xcol + (size_t)IC * 2 + (size_t)G * 256 + (size_t)(tj >> 2) * 32) + (tj & 3);
            dl[0] = o1e;
            dl[4] = o0e;
            dl[32] = o1o;
            dl[36] = o0o;
            if (PAIR) {  // the same eight words into the partner's buffer
                const uint32_t ra = pd->xs + (uint32_t)G * 256u + (uint32_t)(tj >> 2) * 32u + (uint32_t)(tj & 3) * 4u, rb = ra + (uint32_t)IC * 2u;
                st_async_b32(ra, o3e, pd->bar);
                st_async_b32(ra + 16u, o2e, pd->bar);
                st_async_b32(ra + 128u, o3o, pd->bar);
                st_async_b32(ra + 144u, o2o, pd->bar);
                st_async_b32(rb, o1e, pd->bar);
                st_async_b32(rb + 16u, o0e, pd->bar);
                st_async_b32(rb + 128u, o1o, pd->bar);
                st_async_b32(rb + 144u, o0o, pd->bar);
            }
        }
    } else {
        // units of a group are stored j-major so that the four t-lanes of one LDS.128 hit consecutive slots
        const int pos = G * 16 + (tj & 3) * 4 + (tj >> 2);
        if (valid) {
            *reinterpret_cast<uint4 *>(xcol + (size_t)pos * 16) = make_uint4(o3e, o3o, o2e, o2o);
            *reinterpret_cast<uint4 *>(xcol + (size_t)IC * 2 + (size_t)pos * 16) = make_uint4(o1e, o1o, o0e, o0o);
        }
    }
    sxh = __reduce_add_sync(half_mask, sxh);
    sxl = __reduce_add_sync(half_mask, sxl);
    if (valid && (lane & 15) == 0) {
        const float step = (amax > 0.f) ? (amax / kActQ) : 0.f;
        gx[G] = step;              // step of the group
        gsum[G * 2] = sxh;         // 256 * sum(p3) + sum(p2) over the group
        gsum[G * 2 + 1] = sxl;     // 256 * sum(p1) + sum(p0)
        if (PAIR) {
            st_async_b32(pd->gx + (uint32_t)G * 4u, __float_as_uint(step), pd->bar);
            st_async_b32(pd->gsum + (uint32_t)G * 8u, (uint32_t)sxh, pd->bar);
            st_async_b32(pd->gsum + (uint32_t)G * 8u + 4u, (uint32_t)sxl, pd->bar);
        }
    }
}

// ------------------------------------------------------------------------------------------------------------------
// consumer prologue: activations -> (optional RMSNorm) -> four int8 planes per 128-group in MMA-B order, plus the
// per-group step and integer sums.  Ends with a consumer-wide named barrier (id 1).
// ------------------------------------------------------------------------------------------------------------------
template <int NCOLS, int CW>
TCE_DEVINL void stage_activations(const KArgs &a, const Smem &sm, int x_pitch, int ctid, int cw, int lane) {
    constexpr int kConsumerThreads = CW * 32;
    const int units = a.IC / 8;
#pragma unroll 1
    for (int col = 0; col < NCOLS; col++) {
        uint8_t *xcol = sm.xs + (size_t)col * x_pitch;
        float inv = 1.f;
        const float *xsrc = reinterpret_cast<const float *>(a.x);
        if (a.x_mode == X_RMSNORM_F32 && col < a.M) {
            const float *xr = xsrc + (size_t)col * a.ldx;
            float ss = 0.f;
            for (int ui = ctid; ui < units; ui += kConsumerThreads) {
                float4 v0 = *reinterpret_cast<const float4 *>(xr + ui * 8);
                float4 v1 = *reinterpret_cast<const float4 *>(xr + ui * 8 + 4);
                ss += v0.x * v0.x + v0.y * v0.y + v0.z * v0.z + v0.w * v0.w;
                ss += v1.x * v1.x + v1.y * v1.y + v1.z * v1.z + v1.w * v1.w;
            }
            ss = warp_sum(ss);
            if (lane == 0) sm.rms[col * CW + cw] = ss;
            named_bar_sync(1, kConsumerThreads);
            float tot = 0.f;
#pragma unroll
            for (int w = 0; w < CW; w++) tot += sm.rms[col * CW + w];
            inv = rsqrtf(tot / (float)a.IC + a.eps);
        }
        auto emit = [&](int ui, bool valid, const float(&v)[8]) {
            emit_unit<NCOLS>(xcol, a.IC, sm.gx + (size_t)col * a.NG, sm.gsum + (size_t)col * a.NG * 2, ui, valid, v, lane);
        };
        // `units` is a multiple of 16, not of 32: trip counts are warp-uniform so that the half-warp shuffles in emit()
        // always run with all 32 lanes.  Loads of several iterations are issued before any is consumed.
        if (a.x_mode == X_RMSNORM_F32) {
            constexpr int PRE = 2;
            for (int ui0 = 0; ui0 < units; ui0 += PRE * kConsumerThreads) {
                float4 r0[PRE], r1[PRE], g0[PRE], g1[PRE];
#pragma unroll
                for (int k = 0; k < PRE; k++) {
                    const int ui = ui0 + k * kConsumerThreads + ctid;
                    if (ui < units && col < a.M) {
                        const float *xr = xsrc + (size_t)col * a.ldx + ui * 8;
                        r0[k] = *reinterpret_cast<const float4 *>(xr);
                        r1[k] = *reinterpret_cast<const float4 *>(xr + 4);
                        g0[k] = *reinterpret_cast<const float4 *>(a.gamma + ui * 8);
                        g1[k] = *reinterpret_cast<const float4 *>(a.gamma + ui * 8 + 4);
                    } else {
                        r0[k] = r1[k] = g0[k] = g1[k] = make_float4(0.f, 0.f, 0.f, 0.f);
                    }
                }
#pragma unroll
                for (int k = 0; k < PRE; k++) {
                    if (ui0 + k * kConsumerThreads >= units) break;  // warp-uniform
                    const int ui = ui0 + k * kConsumerThreads + ctid;
                    float v[8];
                    v[0] = (r0[k].x * inv) * g0[k].x; v[1] = (r0[k].y * inv) * g0[k].y; v[2] = (r0[k].z * inv) * g0[k].z; v[3] = (r0[k].w * inv) * g0[k].w;
                    v[4] = (r1[k].x * inv) * g1[k].x; v[5] = (r1[k].y * inv) * g1[k].y; v[6] = (r1[k].z * inv) * g1[k].z; v[7] = (r1[k].w * inv) * g1[k].w;
                    emit(ui, ui < units, v);
                }
            }
        } else {
            constexpr int PRE = 4;
            for (int ui0 = 0; ui0 < units; ui0 += PRE * kConsumerThreads) {
                uint4 raw[PRE];
#pragma unroll
                for (int k = 0; k < PRE; k++) {
                    const int ui = ui0 + k * kConsumerThreads + ctid;
                    raw[k] = make_uint4(0u, 0u, 0u, 0u);
                    if (ui < units && col < a.M) raw[k] = *reinterpret_cast<const uint4 *>(reinterpret_cast<const __half *>(a.x) + (size_t)col * a.ldx + ui * 8);
                }
#pragma unroll
                for (int k = 0; k < PRE; k++) {
                    if (ui0 + k * kConsumerThreads >= units) break;  // warp-uniform
                    const int ui = ui0 + k * kConsumerThreads + ctid;
                    const __half2 *h2 = reinterpret_cast<const __half2 *>(&raw[k]);
                    float v[8];
#pragma unroll
                    for (int i = 0; i < 4; i++) {
                        const float2 f = __half22float2(h2[i]);
                        v[2 * i] = f.x;
                        v[2 * i + 1] = f.y;
                    }
                    emit(ui, ui < units, v);
                }
            }
        }
    }
    named_bar_sync(1, kConsumerThreads);
}

// ------------------------------------------------------------------------------------------------------------------
// consumer main loop
// ------------------------------------------------------------------------------------------------------------------
// Single activation column (decode).  Per (16-row tile, 128-k group) a warp issues FOUR integer MMAs instead of twelve:
//   * the four activation planes ride in MMA columns 0..3: lane (g, t) supplies the B operand of column g, so lanes g = 0..3 load planes
//     p3..p0, thread t = 0 of every row pair receives the (p3, p2) plane sums (c0, c1) and thread t = 1 the (p1, p0) sums; columns
//     4..7 are don't-cares;
//   * nibbles become bytes with ONE mask each: w & 0x0f0f0f0f (even slots) and w & 0xf0f0f0f0 (odd slots, = 16 x nibble, still
//     u8).  Even and odd slots accumulate separately (accL, accH); accH is an exact multiple of 16 and is shifted back at the end.
// Two MMAs per parity take words (0,1) and (2,3) of the lane's 16-byte weight load as their two k halves.
struct Lane1 {  // lane-constant operands of the single-column consumer
    const uint8_t *xlane;  // this lane's activation chunk of group 0 (256 B per group)
    float lscale;          // t = 0: 2^16 (columns 0,1 = planes p3,p2), t = 1: 1 (columns 2,3 = planes p1,p0), else 0 (don't-care columns)
    int gsel;              // which of the two group sums this lane subtracts (t & 1)
};
TCE_DEVINL Lane1 make_lane1(const uint8_t *xs, int IC, int g, int t) {
    Lane1 L;
    L.xlane = xs + (size_t)((g >> 1) & 1) * IC * 2 + (size_t)(t * 2 + (g & 1)) * 16;  // column g & 3 supplies plane 3 - (g & 3)
    L.lscale = (t == 0) ? 65536.f : (t == 1 ? 1.f : 0.f);
    L.gsel = t & 1;
    return L;
}
// one (16 rows x 128 k) unit: wa/wb = the lane's 16 B of rows g / g+8; returns the lane's share of the two row sums
TCE_DEVINL void unit1(const Lane1 &L, const uint4 wa, const uint4 wb, int G, float sAq, float sBq, int zAq, int zBq, const float *gx, const int *gsum,
                      float &totA, float &totB) {
    const uint4 xe = *reinterpret_cast<const uint4 *>(L.xlane + (size_t)G * 256);
    const uint4 xo = *reinterpret_cast<const uint4 *>(L.xlane + (size_t)G * 256 + 128);
    constexpr uint32_t ML = 0x0f0f0f0fu, MH = 0xf0f0f0f0u;
    int accL[4], accH[4];
    mma_m16n8k32_u8s8_z(accL, wa.x & ML, wb.x & ML, wa.y & ML, wb.y & ML, xe.x, xe.y);
    mma_m16n8k32_u8s8_z(accH, wa.x & MH, wb.x & MH, wa.y & MH, wb.y & MH, xo.x, xo.y);
    mma_m16n8k32_u8s8(accL, wa.z & ML, wb.z & ML, wa.w & ML, wb.w & ML, xe.z, xe.w);
    mma_m16n8k32_u8s8(accH, wa.z & MH, wb.z & MH, wa.w & MH, wb.w & MH, xo.z, xo.w);
    // X = 2^24*p3 + 2^16*p2 + 2^8*p1 + p0; odd slots carry 16 x nibble: exact integer group result sum_k q*X - z*sum_k X, held as a
    // (p3,p2) part on t = 0 (in units of 2^16) and a (p1,p0) part on t = 1
    const int sxv = gsum[2 * G + L.gsel];
    const float st = gx[G] * L.lscale;
    const int vA = ((accL[0] + (accH[0] >> 4)) << 8) + (accL[1] + (accH[1] >> 4)) - zAq * sxv;
    const int vB = ((accL[2] + (accH[2] >> 4)) << 8) + (accL[3] + (accH[3] >> 4)) - zBq * sxv;
    totA += (sAq * st) * (float)vA;
    totB += (sBq * st) * (float)vB;
}

template <int CW, bool FULL>
TCE_DEVINL void consume1(const KArgs &a, const Smem &sm, RingState &rs, RedState &cs, int cta, int ncta, int cw, int lane) {
    constexpr int GPW = kStageGroups / CW;
    const int g = lane >> 2, t = lane & 3;
    const StreamK sk = make_sk(a, ncta);
    int u = (int)sk.start(cta);
    const int uend = (int)sk.start(cta + 1);
    int gb = u - (u / a.NG) * a.NG;
    const int sg = FULL ? kStageGroups : a.sg;
    const int rp = sg * 64;  // dense row pitch of the TMA box
    // lane-constant offsets: weight rows g / g+8 of the group slot, activation chunk (t, plane = column g)
    const uint32_t w_off = (uint32_t)(g * rp + t * 16);
    const Lane1 L = make_lane1(sm.xs, a.IC, g, t);
    while (u < uend) {
        const int ge = min(a.NG, gb + (uend - u));
        const uint8_t *mbase = sm.meta + (size_t)rs.mslot * sm.meta_bytes;
        const __half *msA = reinterpret_cast<const __half *>(mbase) + g * a.sf_w;
        const __half *msB = msA + 8 * a.sf_w;
        const uint32_t *mzA = reinterpret_cast<const uint32_t *>(mbase + 16 * a.sf_w * 2) + g * a.zeros_w;
        const uint32_t *mzB = mzA + 8 * a.zeros_w;
        float totA = 0.f, totB = 0.f;
        for (int g0 = gb; g0 < ge; g0 += sg) {
            const int n = FULL ? kStageGroups : min(sg, ge - g0);
            mbar_wait(&sm.full_bar[rs.stage], rs.phase);
            const uint8_t *sbase = sm.stages + (size_t)rs.stage * kStageBytes + w_off;
#pragma unroll
            for (int q = 0; q < GPW; q++) {
                const int gi = cw + q * CW;
                if (FULL || gi < n) {
                    const int G = g0 + gi;
                    const uint4 wa = *reinterpret_cast<const uint4 *>(sbase + gi * 64);
                    const uint4 wb = *reinterpret_cast<const uint4 *>(sbase + gi * 64 + 8 * rp);
                    const float sAq = __half2float(msA[G]), sBq = __half2float(msB[G]);
                    const int zsh = (G & 7) * 4;
                    const int zAq = (int)((mzA[G >> 3] >> zsh) & 0xFu);
                    const int zBq = (int)((mzB[G >> 3] >> zsh) & 0xFu);
                    unit1(L, wa, wb, G, sAq, sBq, zAq, zBq, sm.gx, sm.gsum, totA, totB);
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&sm.empty_bar[rs.stage]);
            if (++rs.stage == sm.nst) {
                rs.stage = 0;
                rs.phase ^= 1;
            }
        }
        // ---- hand the tile partial to the epilogue warp (no consumer-to-consumer wait) ----
        totA += __shfl_xor_sync(0xffffffffu, totA, 1);  // (p3, p2) share of t = 0 + (p1, p0) share of t = 1
        totB += __shfl_xor_sync(0xffffffffu, totB, 1);
        mbar_wait(&sm.red_empty[cs.rb], cs.rphase ^ 1);
        float *rbuf = sm.red + ((size_t)cs.rb * CW + cw) * 16;
        if (t == 0) {
            rbuf[g] = totA;
            rbuf[g + 8] = totB;
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&sm.red_full[cs.rb]);
        if (++cs.rb == kRedBufs) {
            cs.rb = 0;
            cs.rphase ^= 1;
        }
        if (++rs.mslot == sm.nst + 1) rs.mslot = 0;
        u += ge - gb;
        gb = 0;
    }
}

template <int NCOLS, int CW>
TCE_DEVINL void consume(const KArgs &a, const Smem &sm, RingState &rs, RedState &cs, int x_pitch, int cta, int ncta, int cw, int lane) {
    static_assert(NCOLS == 1, "the multi-column kernel runs consume_cols");
    if (a.full)
        consume1<CW, true>(a, sm, rs, cs, cta, ncta, cw, lane);
    else
        consume1<CW, false>(a, sm, rs, cs, cta, ncta, cw, lane);
}

// ------------------------------------------------------------------------------------------------------------------
// multi-column kernel (M = 2..8 activation rows).  The 8 MMA columns carry the rows, each plane in its own MMA.  The units are ordered
// slice-major (KArgs::sl): each CTA stages the activation K-slices its unit range touches, one at a time, so the kernel reads every weight
// byte once whatever IC is.  With one slice (the whole row fits) the order is the tile-major order of the single-column kernel.
// ------------------------------------------------------------------------------------------------------------------
struct SliceWalk {
    int T, NG, sl, nsl;
    TCE_DEVINL int len(int s) const { return s < nsl - 1 ? sl : NG - s * sl; }
    // unit u -> slice s, row tile rt, first group gb of the piece, first unit seg0 of the (slice, tile) segment
    TCE_DEVINL void locate(int u, int &s, int &rt, int &gb, int &seg0) const {
        s = min(u / (T * sl), nsl - 1);
        const int base = s * T * sl, L = len(s);
        rt = (u - base) / L;
        seg0 = base + rt * L;
        gb = s * sl + (u - seg0);
    }
    // first unit of segment k (k = s * T + rt; the last slice may be shorter)
    TCE_DEVINL int seg_unit(long long k) const {
        const long long kf = (long long)T * (nsl - 1);
        return (int)(k <= kf ? k * sl : kf * sl + (k - kf) * (NG - (nsl - 1) * sl));
    }
    // first unit of CTA c: with several slices the ranges are cut at segment boundaries, so every piece is a whole (slice, tile) segment
    TCE_DEVINL int start(const StreamK &sk, int c) const {
        if (nsl == 1) return (int)sk.start(c);
        return seg_unit((long long)T * nsl * c / sk.nc);
    }
};
TCE_DEVINL SliceWalk make_walk(const KArgs &a) { return SliceWalk{a.num_tiles, a.NG, a.sl, a.nsl}; }

// producer of the multi-column kernel: one piece = the units of one (slice, tile) segment in this CTA's range
TCE_DEVINL void produce_cols(const KArgs &a, const Smem &sm, RingState &rs, int cta, int ncta, int lane, uint64_t policy) {
    const StreamK sk = make_sk(a, ncta);
    const SliceWalk W = make_walk(a);
    const uint32_t leader = (lane == 0) ? 1u : 0u;
    const uint32_t meta_bytes_cur = 320u * a.zeros_w;
    const uint32_t box_bytes = 16u * a.sg * 64u;
    // A tile's scales / zeros slab is copied whole with every piece: a bulk copy needs a 16-B aligned source, and one slice's part of a
    // zeros row (zeros_w words per row) is not.  With several slices the slab is cached normally in L2 for the tile's later pieces (some
    // microseconds later, on other CTAs); the weights, read once, stay evict-first.
    const uint64_t meta_policy = a.nsl > 1 ? l2_policy_evict_normal() : policy;
    int u = W.start(sk, cta);
    const int uend = W.start(sk, cta + 1);
    while (u < uend) {
        int s, rt, gb, seg0;
        W.locate(u, s, rt, gb, seg0);
        const int pe = min(uend, seg0 + W.len(s));
        const int ge = gb + (pe - u);
        int si0 = 0, row0 = rt * 16, si1 = 0, row1 = 0;
        if (a.pair_mode) {
            row0 = rt * 8;
            si1 = 1;
            row1 = rt * 8;
        } else if (a.nseg > 1 && row0 >= a.seg[0].rows) {
            row0 -= a.seg[0].rows;
            si0 = 1;
            if (a.nseg > 2 && row0 >= a.seg[1].rows) {
                row0 -= a.seg[1].rows;
                si0 = 2;
            }
        }
        const RowRef r0 = tile_row(a, rt, 0), r8 = tile_row(a, rt, 8);
        uint8_t *mdst = sm.meta + (size_t)rs.mslot * sm.meta_bytes;
        bool first = true;
        for (int g0 = gb; g0 < ge; g0 += a.sg) {
            mbar_wait(&sm.empty_bar[rs.stage], rs.phase ^ 1);
            uint64_t *bar = &sm.full_bar[rs.stage];
            mbar_arrive_expect_tx_pred(bar, box_bytes + (first ? meta_bytes_cur : 0u), leader);
            uint8_t *dst = sm.stages + (size_t)rs.stage * kStageBytes;
            tma_load_2d_pred(dst, &a.tmap[si0], g0 * 16, row0, bar, policy, leader);
            if (a.pair_mode) tma_load_2d_pred(dst + 8 * a.sg * 64, &a.tmap[si1], g0 * 16, row1, bar, policy, leader);
            if (first) {  // the tile's scales / zeros slabs
                const uint32_t sb = 8u * a.sf_w * 2u, zb = 8u * a.zeros_w * 4u;
                bulk_g2s_pred(mdst, r0.s, sb, bar, meta_policy, leader);
                bulk_g2s_pred(mdst + sb, r8.s, sb, bar, meta_policy, leader);
                bulk_g2s_pred(mdst + 2 * sb, r0.z, zb, bar, meta_policy, leader);
                bulk_g2s_pred(mdst + 2 * sb + zb, r8.z, zb, bar, meta_policy, leader);
            }
            __syncwarp();
            first = false;
            if (++rs.stage == sm.nst) {
                rs.stage = 0;
                rs.phase ^= 1;
            }
        }
        if (++rs.mslot == sm.nst + 1) rs.mslot = 0;
        u = pe;
    }
}

// epilogue warp of the multi-column kernel.  With several slices every tile is made of nsl pieces, one per slice: each piece parks its
// partial in the record of its (slice, tile) and the last piece to arrive sums them in slice order, so the result does not depend on which
// CTA finished first.  EPI_ADD_F32 with atomic_add adds the pieces with RED.ADD instead.
template <int NCOLS, int CW>
TCE_DEVINL void epilogue_cols(const KArgs &a, const Smem &sm, RedState &es, int cta, int ncta, int lane) {
    constexpr int kVals = 16 * NCOLS;
    constexpr int VPL = kVals / 32;
    static_assert(kVals % 32 == 0, "every lane holds VPL whole values");
    const StreamK sk = make_sk(a, ncta);
    const SliceWalk W = make_walk(a);
    const long long u0 = W.start(sk, cta);
    int u = (int)u0;
    const int uend = W.start(sk, cta + 1);
    while (u < uend) {
        int s, rt, gb, seg0;
        W.locate(u, s, rt, gb, seg0);
        const int pe = min(uend, seg0 + W.len(s));
        const bool full_tile = (a.nsl == 1 && u == seg0 && pe == seg0 + a.NG);
        mbar_wait(&sm.red_full[es.rb], es.rphase);
        const float *rbuf = sm.red + (size_t)es.rb * CW * kVals;
        float v[VPL];
#pragma unroll
        for (int i = 0; i < VPL; i++) {
            const int idx = lane + 32 * i;
            float acc = 0.f;
#pragma unroll
            for (int w = 0; w < CW; w++) acc += rbuf[w * kVals + idx];
            v[i] = acc;
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&sm.red_empty[es.rb]);
        if (++es.rb == kRedBufs) {
            es.rb = 0;
            es.rphase ^= 1;
        }
        bool do_final = full_tile;
        if (!full_tile && a.atomic_add) {
#pragma unroll
            for (int i = 0; i < VPL; i++) {
                const int idx = lane + 32 * i;
                const int row = idx / NCOLS, col = idx % NCOLS;
                if (col < a.M) atomicAdd(reinterpret_cast<float *>(a.y) + (size_t)col * a.ldy + (size_t)rt * 16 + row, v[i]);
            }
        } else if (!full_tile) {
            int last = 0;
            if (a.nsl == 1) {  // one slice: the per-CTA records of the single-column kernel (first tile / tail tile of each CTA)
                const long long tb = (long long)rt * a.NG;
                const int c_first = sk.cta_of(tb), c_last = sk.cta_of(tb + a.NG - 1);
                float *mine = a.partials + ((size_t)cta * 2 + ((u0 >= tb) ? 0 : 1)) * kVals;
#pragma unroll
                for (int i = 0; i < VPL; i++) mine[lane + 32 * i] = v[i];
                __threadfence();
                __syncwarp();
                if (lane == 0) {
                    const unsigned prev = atomicAdd(&a.counters[rt], 1u);
                    last = (prev == (unsigned)(c_last - c_first)) ? 1 : 0;
                    if (last) a.counters[rt] = 0;
                }
                last = __shfl_sync(0xffffffffu, last, 0);
                if (last) {
                    __threadfence();
#pragma unroll
                    for (int i = 0; i < VPL; i++) {
                        float acc = 0.f;
                        for (int c = c_first; c <= c_last; c++)
                            acc += ldg_cg_f32(a.partials + ((size_t)c * 2 + ((sk.start(c) >= tb) ? 0 : 1)) * kVals + lane + 32 * i);
                        v[i] = acc;
                    }
                }
            } else {  // one record per (slice, tile): the last of the tile's nsl pieces to arrive sums them in slice order
                auto rec = [&](int q) { return a.partials + ((size_t)q * a.num_tiles + rt) * kVals; };
                float *mine = rec(s);
#pragma unroll
                for (int i = 0; i < VPL; i++) mine[lane + 32 * i] = v[i];
                __threadfence();
                __syncwarp();
                if (lane == 0) {
                    const unsigned prev = atomicAdd(&a.counters[rt], 1u);
                    last = (prev == (unsigned)(a.nsl - 1)) ? 1 : 0;
                    if (last) a.counters[rt] = 0;
                }
                last = __shfl_sync(0xffffffffu, last, 0);
                if (last) {
                    __threadfence();
                    float p[kMaxSlices][VPL];
#pragma unroll
                    for (int q = 0; q < kMaxSlices; q++)
#pragma unroll
                        for (int i = 0; i < VPL; i++) p[q][i] = q < a.nsl ? ldg_cg_f32(rec(q) + lane + 32 * i) : 0.f;
#pragma unroll
                    for (int i = 0; i < VPL; i++) {
                        float acc = 0.f;
#pragma unroll
                        for (int q = 0; q < kMaxSlices; q++) acc += p[q][i];
                        v[i] = acc;
                    }
                }
            }
            do_final = last != 0;
        }
        if (do_final) finish_tile<NCOLS>(a, v, rt, lane);
        u = pe;
    }
}

// sum of squares of every column's full row (RMSNorm prologue), per consumer warp in sm.rms[col][warp]; ends with a consumer barrier
template <int NCOLS, int CW>
TCE_DEVINL void rms_partials(const KArgs &a, const Smem &sm, int ctid, int cw, int lane) {
    constexpr int kConsumerThreads = CW * 32;
    const int units = a.IC / 8;
    const float *xsrc = reinterpret_cast<const float *>(a.x);
#pragma unroll 1
    for (int col = 0; col < NCOLS; col++) {
        float ss = 0.f;
        if (col < a.M) {
            const float *xr = xsrc + (size_t)col * a.ldx;
            for (int ui = ctid; ui < units; ui += kConsumerThreads) {
                float4 v0 = *reinterpret_cast<const float4 *>(xr + ui * 8);
                float4 v1 = *reinterpret_cast<const float4 *>(xr + ui * 8 + 4);
                ss += v0.x * v0.x + v0.y * v0.y + v0.z * v0.z + v0.w * v0.w;
                ss += v1.x * v1.x + v1.y * v1.y + v1.z * v1.z + v1.w * v1.w;
            }
        }
        ss = warp_sum(ss);
        if (lane == 0) sm.rms[col * CW + cw] = ss;
    }
    named_bar_sync(1, kConsumerThreads);
}

// stage K-slice s of every column (fp16 input, or RMSNorm of the fp32 residual with the full-row sums of rms_partials) as four int8 planes
// in MMA-B order, at group index G - s*sl; the group steps / sums go to their global group index.  Ends with a consumer barrier.
template <int NCOLS, int CW>
TCE_DEVINL void stage_slice(const KArgs &a, const Smem &sm, int x_pitch, int s, int ctid, int cw, int lane) {
    constexpr int kConsumerThreads = CW * 32;
    const int xw = a.sl * 128;                               // plane buffer width of a column (region B starts at xw * 2)
    const int g0 = s * a.sl, units = min(a.sl, a.NG - g0) * 16;  // 8-element units of the slice (a multiple of 16)
#pragma unroll 1
    for (int col = 0; col < NCOLS; col++) {
        uint8_t *xcol = sm.xs + (size_t)col * x_pitch;
        float *gx = sm.gx + (size_t)col * a.NG + g0;
        int *gsum = sm.gsum + ((size_t)col * a.NG + g0) * 2;
        const bool live = col < a.M;
        if (a.x_mode == X_RMSNORM_F32) {
            float tot = 0.f;
#pragma unroll
            for (int w = 0; w < CW; w++) tot += sm.rms[col * CW + w];
            const float inv = rsqrtf(tot / (float)a.IC + a.eps);
            const float *xr = reinterpret_cast<const float *>(a.x) + (size_t)col * a.ldx + (size_t)g0 * 128;
            const float *gm = a.gamma + (size_t)g0 * 128;
            constexpr int PRE = 2;
            for (int ui0 = 0; ui0 < units; ui0 += PRE * kConsumerThreads) {
                float4 r0[PRE], r1[PRE], q0[PRE], q1[PRE];
#pragma unroll
                for (int k = 0; k < PRE; k++) {
                    const int ui = ui0 + k * kConsumerThreads + ctid;
                    if (ui < units && live) {
                        r0[k] = *reinterpret_cast<const float4 *>(xr + ui * 8);
                        r1[k] = *reinterpret_cast<const float4 *>(xr + ui * 8 + 4);
                        q0[k] = *reinterpret_cast<const float4 *>(gm + ui * 8);
                        q1[k] = *reinterpret_cast<const float4 *>(gm + ui * 8 + 4);
                    } else {
                        r0[k] = r1[k] = q0[k] = q1[k] = make_float4(0.f, 0.f, 0.f, 0.f);
                    }
                }
#pragma unroll
                for (int k = 0; k < PRE; k++) {
                    if (ui0 + k * kConsumerThreads >= units) break;  // warp-uniform
                    const int ui = ui0 + k * kConsumerThreads + ctid;
                    float v[8];
                    v[0] = (r0[k].x * inv) * q0[k].x; v[1] = (r0[k].y * inv) * q0[k].y; v[2] = (r0[k].z * inv) * q0[k].z; v[3] = (r0[k].w * inv) * q0[k].w;
                    v[4] = (r1[k].x * inv) * q1[k].x; v[5] = (r1[k].y * inv) * q1[k].y; v[6] = (r1[k].z * inv) * q1[k].z; v[7] = (r1[k].w * inv) * q1[k].w;
                    emit_unit<NCOLS>(xcol, xw, gx, gsum, ui, ui < units, v, lane);
                }
            }
        } else {
            const __half *xr = reinterpret_cast<const __half *>(a.x) + (size_t)col * a.ldx + (size_t)g0 * 128;
            constexpr int PRE = 4;
            for (int ui0 = 0; ui0 < units; ui0 += PRE * kConsumerThreads) {
                uint4 raw[PRE];
#pragma unroll
                for (int k = 0; k < PRE; k++) {
                    const int ui = ui0 + k * kConsumerThreads + ctid;
                    raw[k] = make_uint4(0u, 0u, 0u, 0u);
                    if (ui < units && live) raw[k] = *reinterpret_cast<const uint4 *>(xr + ui * 8);
                }
#pragma unroll
                for (int k = 0; k < PRE; k++) {
                    if (ui0 + k * kConsumerThreads >= units) break;  // warp-uniform
                    const int ui = ui0 + k * kConsumerThreads + ctid;
                    const __half2 *h2 = reinterpret_cast<const __half2 *>(&raw[k]);
                    float v[8];
#pragma unroll
                    for (int i = 0; i < 4; i++) {
                        const float2 f = __half22float2(h2[i]);
                        v[2 * i] = f.x;
                        v[2 * i + 1] = f.y;
                    }
                    emit_unit<NCOLS>(xcol, xw, gx, gsum, ui, ui < units, v, lane);
                }
            }
        }
    }
    named_bar_sync(1, kConsumerThreads);
}

// first slice of this CTA's unit range (the kernel stages it before the barrier hand-off, like the single-column kernel stages its row)
TCE_DEVINL int first_slice(const KArgs &a, int cta, int ncta) {
    const int u = make_walk(a).start(make_sk(a, ncta), cta);
    return min(u / (a.num_tiles * a.sl), a.nsl - 1);
}

// consumers of the multi-column kernel; `staged` = the slice already in shared memory
template <int NCOLS, int CW>
TCE_DEVINL void consume_cols(const KArgs &a, const Smem &sm, RingState &rs, RedState &cs, int x_pitch, int staged, int cta, int ncta, int ctid, int cw,
                             int lane) {
    constexpr int kVals = 16 * NCOLS;
    constexpr int GPW = kStageGroups / CW;  // groups per consumer warp per stage
    const int g = lane >> 2, t = lane & 3;
    const StreamK sk = make_sk(a, ncta);
    const SliceWalk W = make_walk(a);
    const int xw = a.sl * 128;
    int u = W.start(sk, cta);
    const int uend = W.start(sk, cta + 1);
    while (u < uend) {
        int s, rt, gb, seg0;
        W.locate(u, s, rt, gb, seg0);
        const int pe = min(uend, seg0 + W.len(s));
        const int ge = gb + (pe - u);
        if (s != staged) {
            named_bar_sync(1, CW * 32);  // every consumer warp is done with the previous slice
            stage_slice<NCOLS, CW>(a, sm, x_pitch, s, ctid, cw, lane);
            staged = s;
        }
        const int gs = s * a.sl;  // first group of the staged slice
        // this tile's scales / zeros slab (it lands together with the piece's first weight stage)
        const uint8_t *mbase = sm.meta + (size_t)rs.mslot * sm.meta_bytes;
        const __half *msA = reinterpret_cast<const __half *>(mbase) + g * a.sf_w;
        const __half *msB = msA + 8 * a.sf_w;
        const uint32_t *mzA = reinterpret_cast<const uint32_t *>(mbase + 16 * a.sf_w * 2) + g * a.zeros_w;
        const uint32_t *mzB = mzA + 8 * a.zeros_w;
        constexpr int NT = 4;
        float tot[NT];
#pragma unroll
        for (int i = 0; i < NT; i++) tot[i] = 0.f;

        const int rp = a.sg * 64;  // dense row pitch of the TMA box (2-way bank conflict on the weight LDS, see DESIGN.md)
        for (int g0 = gb; g0 < ge; g0 += a.sg) {
            const int n = min(a.sg, ge - g0);
            mbar_wait(&sm.full_bar[rs.stage], rs.phase);
            const uint8_t *sbase = sm.stages + (size_t)rs.stage * kStageBytes;
#pragma unroll
            for (int q = 0; q < GPW; q++) {
                const int gi = cw + q * CW;
                if (gi < n) {
                    const int G = g0 + gi;
                    // per-group scale and zero point of rows g and g+8
                    const float sAq = __half2float(msA[G]), sBq = __half2float(msB[G]);
                    const int zsh = (G & 7) * 4;
                    const int zAq = (int)((mzA[G >> 3] >> zsh) & 0xFu);
                    const int zBq = (int)((mzB[G >> 3] >> zsh) & 0xFu);
                    const uint8_t *sp = sbase + gi * 64 + t * 16;
                    const uint4 wa = *reinterpret_cast<const uint4 *>(sp + g * rp);
                    const uint4 wb = *reinterpret_cast<const uint4 *>(sp + (g + 8) * rp);
                    const uint32_t wav[4] = {wa.x, wa.y, wa.z, wa.w};
                    const uint32_t wbv[4] = {wb.x, wb.y, wb.z, wb.w};
                    const uint8_t *xp = sm.xs + (size_t)g * x_pitch + ((size_t)(G - gs) * 16 + t) * 16;
                    // nibbles -> bytes: w & 0x0f0f0f0f = (n0,n2,n4,n6), (w>>4) & 0x0f0f0f0f = (n1,n3,n5,n7): 3 ALU ops per
                    // 8 weights.  One accumulator set per activation plane (p3..p0).
                    const uint8_t *xl = xp + (size_t)xw * 2;
                    int c3[4], c2[4], c1[4], c0[4];
#pragma unroll
                    for (int i = 0; i < 4; i++) c3[i] = c2[i] = c1[i] = c0[i] = 0;
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        const uint4 xv = *reinterpret_cast<const uint4 *>(xp + j * 64);
                        const uint4 xq = *reinterpret_cast<const uint4 *>(xl + j * 64);
                        const uint32_t a0 = wav[j] & 0x0f0f0f0fu, a2 = (wav[j] >> 4) & 0x0f0f0f0fu;
                        const uint32_t a1 = wbv[j] & 0x0f0f0f0fu, a3 = (wbv[j] >> 4) & 0x0f0f0f0fu;
                        mma_m16n8k32_u8s8(c3, a0, a1, a2, a3, xv.x, xv.y);
                        mma_m16n8k32_u8s8(c2, a0, a1, a2, a3, xv.z, xv.w);
                        mma_m16n8k32_u8s8(c1, a0, a1, a2, a3, xq.x, xq.y);
                        mma_m16n8k32_u8s8(c0, a0, a1, a2, a3, xq.z, xq.w);
                    }
                    // exact integer group result: sum_k q*X - z*sum_k X, X = 2^24*p3 + 2^16*p2 + 2^8*p1 + p0, kept as a (p3,p2) part in
                    // units of 2^16 and a (p1,p0) part (the full integer does not fit 32 bits)
                    {
                        const int *gs0 = sm.gsum + ((2 * t) * a.NG + G) * 2, *gs1 = sm.gsum + ((2 * t + 1) * a.NG + G) * 2;
                        const float st0 = sm.gx[(2 * t) * a.NG + G], st1 = sm.gx[(2 * t + 1) * a.NG + G];
                        auto comb = [](int h3, int h2, int l1, int l0, int z, const int *gsp) {
                            return 65536.f * (float)((h3 << 8) + h2 - z * gsp[0]) + (float)((l1 << 8) + l0 - z * gsp[1]);
                        };
                        tot[0] += (sAq * st0) * comb(c3[0], c2[0], c1[0], c0[0], zAq, gs0);
                        tot[1] += (sAq * st1) * comb(c3[1], c2[1], c1[1], c0[1], zAq, gs1);
                        tot[2] += (sBq * st0) * comb(c3[2], c2[2], c1[2], c0[2], zBq, gs0);
                        tot[3] += (sBq * st1) * comb(c3[3], c2[3], c1[3], c0[3], zBq, gs1);
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&sm.empty_bar[rs.stage]);
            if (++rs.stage == sm.nst) {
                rs.stage = 0;
                rs.phase ^= 1;
            }
        }

        // ---- hand the piece's partial to the epilogue warp (no consumer-to-consumer wait) ----
        mbar_wait(&sm.red_empty[cs.rb], cs.rphase ^ 1);
        float *rbuf = sm.red + ((size_t)cs.rb * CW + cw) * kVals;
        rbuf[g * NCOLS + 2 * t] = tot[0];
        rbuf[g * NCOLS + 2 * t + 1] = tot[1];
        rbuf[(g + 8) * NCOLS + 2 * t] = tot[2];
        rbuf[(g + 8) * NCOLS + 2 * t + 1] = tot[3];
        __syncwarp();
        if (lane == 0) mbar_arrive(&sm.red_full[cs.rb]);
        if (++cs.rb == kRedBufs) {
            cs.rb = 0;
            cs.rphase ^= 1;
        }
        if (++rs.mslot == sm.nst + 1) rs.mslot = 0;
        u = pe;
    }
}


}  // namespace gemv
}  // namespace tce
