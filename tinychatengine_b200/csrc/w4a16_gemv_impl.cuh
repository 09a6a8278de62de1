// w4a16_gemv_impl.cuh -- device-side roles of the stand-alone W4A16 group-128 GEMV (w4a16_gemv.cu): producer, consumers and epilogue
// of one kernel body for 1..8 activation rows.  The persistent decode kernel shares only the activation number format
// (w4a16_act_planes.cuh) with it.
//
// Data contract = the reference's QM_CUDA layout (kernels/cuda/gemv_cuda.cu:140-260, quantize_methods.py:370-442):
//     w uint32[OC][IC/8] sequential nibbles, zeros uint32[OC][zeros_w] (nibble g = zero of group g),
//     scales half[OC][zeros_w*8];   y[m][oc] = sum_ic s[oc,g] * (q[oc,ic] - z[oc,g]) * x[m][ic]
//
//  * work unit = (16-row tile, one 128-k group) = 1 KiB of packed weights, in the order of SliceWalk (kernels.h): slice-major over
//    K-slices of KArgs::sl groups, which with one slice (always at M = 1) is tile-major.  The units of a launch are cut into equal
//    contiguous per-CTA ranges (stream-K), at row-tile boundaries for epilogues that need one ordered writer, or at (slice, tile)
//    segment boundaries with several slices.
//  * producer (1 warp, 1 elected lane): ONE 2-D TMA tensor copy (UTMALDG) per stage moves the [16 rows x <=16 groups]
//    weight box into a ring of KArgs::nst stages guarded by full/empty mbarriers, L2 evict-first; the tile's
//    scales/zeros slabs (1-D bulk copies, UBLKCP) ride on the first stage's barrier.  Producers depend on nothing but the weights,
//    so they run ahead of everything else (in particular of the consumers' activation staging).
//  * consumers (CW warps): 128-bit LDS of the packed nibbles; activations held as four int8 planes (32-bit block fixed point per
//    128-group, exact integer accumulation, w4a16_act_planes.cuh); mma.sync.m16n8k32 u8 x s8 -> s32; per-group epilogue
//    tot += (s * step) * (acc - z * sum_X).  One activation row (consume1): the four planes ride in MMA columns 0..3 and
//    nibbles become bytes with one mask each (even slots w & 0x0f0f0f0f, odd slots w & 0xf0f0f0f0 = 16 x nibble, shifted back
//    after accumulation): 4 IMMAs per (16 rows x 128 k).  Up to 8 rows (consume_cols): the 8 MMA columns carry the rows, planes in
//    separate MMAs, (w >> 4) & 0x0f0f0f0f for the odd slots.  Both run in the same loop (consume).
//  * tile partials go to the epilogue warp through a triple-buffered smem slot + mbarrier (consumers never wait for
//    each other); the epilogue warp runs the fused epilogue (fp16/fp32 store, residual +=, SiLU(gate)*up), the
//    RED.ADD residual path or the ordered stream-K fix-up.
//  * fused prologue: RMSNorm of an fp32 residual stream (LlamaRMSNorm semantics) + activation quantisation.
#pragma once
#include "common.cuh"
#include "kernels.h"
#include "w4a16_act_planes.cuh"

namespace tce {
namespace gemv {

constexpr int kStageGroups = 16;               // 128-k groups per pipeline stage (per row: up to 1024 B)
constexpr int kStageBytes = 16 * kStageGroups * 64;  // 16 KiB: dense [16 rows][sg*64 B] box written by ONE 2-D TMA instruction
constexpr int kStages = 4;         // the shallowest ring a launch plans for (fit check, K-slice choice); KArgs::nst is the deepest that fits
constexpr int kMaxStages = 12;
constexpr int kRedBufs = 3;
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
    int nst;         // TMA ring depth of this launch (2..kMaxStages stages of 16 KiB)
    int pdl_early;   // 1: griddepcontrol.launch_dependents at kernel entry instead of after the last weight request
    // the activation columns are staged one K-slice of `sl` groups (a multiple of kStageGroups, or NG) at a time, in the unit order of
    // SliceWalk: a CTA stages only the slices its range touches.  M = 1 launches stage the whole row (sl = NG, nsl = 1)
    int sl, nsl;
    // one 2-D tensor map per weight segment: uint32 [rows][IC/8], box = [16 (8 in pair mode) rows][sg*16 words]
    alignas(64) CUtensorMap tmap[3];
};

// weight segment `si` and row `r` in it of source row `l` (0..15) of row tile `rt`
struct SegRow {
    int si, r;
};
TCE_DEVINL SegRow seg_row(const KArgs &a, int rt, int l) {
    SegRow p{0, 0};
    if (a.pair_mode) {
        p.si = l >> 3;
        p.r = rt * 8 + (l & 7);
    } else {
        p.r = rt * 16 + l;
        if (a.nseg > 1 && p.r >= a.seg[0].rows) {
            p.r -= a.seg[0].rows;
            p.si = 1;
            if (a.nseg > 2 && p.r >= a.seg[1].rows) {
                p.r -= a.seg[1].rows;
                p.si = 2;
            }
        }
    }
    return p;
}

struct RowRef {
    const uint8_t *w;
    const uint32_t *z;
    const __half *s;
};

// source row `l` (0..15) of row tile `rt`
TCE_DEVINL RowRef tile_row(const KArgs &a, int rt, int l) {
    const SegRow p = seg_row(a, rt, l);
    const W4Seg &s = a.seg[p.si];
    RowRef ref;
    ref.w = reinterpret_cast<const uint8_t *>(s.w) + (size_t)p.r * (a.IC / 2);
    ref.z = s.zeros + (size_t)p.r * a.zeros_w;
    ref.s = s.scales + (size_t)p.r * a.sf_w;
    return ref;
}

TCE_DEVINL void dbg_stamp(const KArgs &a, int cta, int k) {
    if (a.dbg) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        a.dbg[(size_t)cta * 8 + k] = t;
    }
}

// shared-memory layout (offsets from a 128-B aligned base); `xw` = activation elements staged per column (one K-slice)
template <int NCOLS, int CW>
struct Layout {
    static constexpr int kXPad = (NCOLS > 1) ? 64 : 0;  // column pitch = 64 (mod 128) B for the per-column B loads
    static constexpr int kVals = 16 * NCOLS;
    // four int8 planes per activation (32-bit block fixed point): planes (p3, p2) interleaved in region A (2 B per element),
    // planes (p1, p0) in region B that follows region A of the same column
    static __host__ __device__ int x_pitch(int xw) { return xw * 4 + kXPad; }
    // one meta slot = scales half[16][zeros_w*8] followed by zeros uint32[16][zeros_w] = 320 * zeros_w bytes
    static __host__ __device__ int meta_slot_bytes(int IC) { return 320 * (((IC / 128) + 7) / 8); }
    static __host__ __device__ size_t off_meta(int nst) { return (size_t)nst * kStageBytes; }
    static __host__ __device__ size_t off_xs(int IC, int nst) { return off_meta(nst) + (size_t)(nst + 1) * meta_slot_bytes(IC); }
    static __host__ __device__ size_t off_gx(int IC, int nst, int xw) { return off_xs(IC, nst) + (size_t)NCOLS * x_pitch(xw); }
    // gx: float step[NCOLS][NG] followed by int gsum[NCOLS][NG][2] = {256 * sum(p3) + sum(p2), 256 * sum(p1) + sum(p0)}
    static __host__ __device__ size_t off_red(int IC, int nst, int xw) { return off_gx(IC, nst, xw) + (size_t)3 * NCOLS * (IC / 128) * sizeof(float); }
    static __host__ __device__ size_t off_rms(int IC, int nst, int xw) { return off_red(IC, nst, xw) + (size_t)kRedBufs * CW * kVals * sizeof(float); }
    static __host__ __device__ size_t off_bar(int IC, int nst, int xw) { return (off_rms(IC, nst, xw) + (size_t)NCOLS * CW * sizeof(float) + 15) & ~(size_t)15; }
    static __host__ __device__ size_t bytes(int IC, int nst, int xw) { return off_bar(IC, nst, xw) + (2 * nst + 2 * kRedBufs) * sizeof(uint64_t) + 16; }
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

// spread over the lanes of one warp: one barrier pair per lane instead of ~14 dependent inits on one thread
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
// same (piece, stage) sequence
struct RingState {
    int stage = 0;
    uint32_t phase = 0;
    int mslot = 0;
    TCE_DEVINL void next_stage(int nst) {
        if (++stage == nst) {
            stage = 0;
            phase ^= 1;
        }
    }
    TCE_DEVINL void next_piece(int nst) {  // one scales / zeros slot per piece, ring depth + 1 of them
        if (++mslot == nst + 1) mslot = 0;
    }
};
struct RedState {
    int rb = 0;
    uint32_t rphase = 0;
    TCE_DEVINL void next() {
        if (++rb == kRedBufs) {
            rb = 0;
            rphase ^= 1;
        }
    }
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
// the single-column kernel always stages the whole row: its walk is the one-slice case, fixed at compile time so that the
// multi-slice paths of the roles drop out of it
template <int NCOLS>
TCE_DEVINL SliceWalk make_walk(const KArgs &a) {
    return NCOLS == 1 ? SliceWalk{a.num_tiles, a.NG, a.NG, 1} : SliceWalk{a.num_tiles, a.NG, a.sl, a.nsl};
}

// ------------------------------------------------------------------------------------------------------------------
// producer warp: streams this CTA's pieces into the ring.  Warp-convergent, lane 0 issues.  `a` must be the
// original argument block (kernel parameter or global memory), never a local copy: the TMA unit reads the tensor map
// through its address.
// ------------------------------------------------------------------------------------------------------------------
template <int NCOLS>
TCE_DEVINL void produce(const KArgs &a, const Smem &sm, int cta, int ncta, int lane, uint64_t policy) {
    const StreamK sk = make_sk(a, ncta);
    const SliceWalk W = make_walk<NCOLS>(a);
    const uint32_t leader = (lane == 0) ? 1u : 0u;
    const uint32_t meta_bytes_cur = 320u * a.zeros_w;  // bytes actually copied for this IC (<= sm.meta_bytes)
    const uint32_t box_bytes = 16u * a.sg * 64u;       // a stage always receives the full box (out-of-range parts are zero-filled)
    // A tile's scales / zeros slab is copied whole with every piece: a bulk copy needs a 16-B aligned source, and one slice's part of a
    // zeros row (zeros_w words per row) is not.  With several slices the slab is cached normally in L2 for the tile's later pieces (some
    // microseconds later, on other CTAs); the weights, read once, stay evict-first.
    const uint64_t meta_policy = W.nsl > 1 ? l2_policy_evict_normal() : policy;
    RingState rs;
    int u = W.start(sk, cta);
    const int uend = W.start(sk, cta + 1);
    while (u < uend) {
        int s, rt, gb, seg0;
        W.locate(u, s, rt, gb, seg0);
        const int pe = min(uend, seg0 + W.len(s));
        const int ge = gb + (pe - u);
        // box origins: rows 0..15 of the tile, or in pair mode rows 0..7 (gate) and 8..15 (up)
        const SegRow p0 = seg_row(a, rt, 0), p8 = seg_row(a, rt, 8);
        const RowRef r0 = tile_row(a, rt, 0), r8 = tile_row(a, rt, 8);
        uint8_t *mdst = sm.meta + (size_t)rs.mslot * sm.meta_bytes;
        bool first = true;
        for (int g0 = gb; g0 < ge; g0 += a.sg) {
            mbar_wait(&sm.empty_bar[rs.stage], rs.phase ^ 1);
            uint64_t *bar = &sm.full_bar[rs.stage];
            mbar_arrive_expect_tx_pred(bar, box_bytes + (first ? meta_bytes_cur : 0u), leader);
            uint8_t *dst = sm.stages + (size_t)rs.stage * kStageBytes;
            tma_load_2d_pred(dst, &a.tmap[p0.si], g0 * 16, p0.r, bar, policy, leader);
            if (a.pair_mode) tma_load_2d_pred(dst + 8 * a.sg * 64, &a.tmap[p8.si], g0 * 16, p8.r, bar, policy, leader);
            if (first) {  // the tile's scales / zeros slabs
                const uint32_t sb = 8u * a.sf_w * 2u, zb = 8u * a.zeros_w * 4u;
                bulk_g2s_pred(mdst, r0.s, sb, bar, meta_policy, leader);
                bulk_g2s_pred(mdst + sb, r8.s, sb, bar, meta_policy, leader);
                bulk_g2s_pred(mdst + 2 * sb, r0.z, zb, bar, meta_policy, leader);
                bulk_g2s_pred(mdst + 2 * sb + zb, r8.z, zb, bar, meta_policy, leader);
            }
            __syncwarp();
            first = false;
            rs.next_stage(sm.nst);
        }
        rs.next_piece(sm.nst);
        u = pe;
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
// epilogue warp: reduces the CW consumer partials of every piece this CTA walks, then either finishes the tile or takes
// part in the fix-up of a split tile.  With one slice the fix-up records are per CTA ({first tile, tail tile}) and the last
// contributor sums them in CTA order; with several every tile is made of nsl pieces, each parks its partial in the record of
// its (slice, tile) and the last piece to arrive sums them in slice order.  Either way the result does not depend on which
// CTA finished first.  EPI_ADD_F32 with atomic_add adds the pieces with RED.ADD instead.
// Lane l owns values idx = l + 32*i  (idx = row*NCOLS + col).
// ------------------------------------------------------------------------------------------------------------------
template <int NCOLS, int CW>
TCE_DEVINL void epilogue(const KArgs &a, const Smem &sm, int cta, int ncta, int lane) {
    constexpr int kVals = 16 * NCOLS;
    constexpr int VPL = (kVals + 31) / 32;  // values per lane
    // a single-column tile is 16 values over 32 lanes: lanes 16..31 hold none
    auto held = [lane](int i) { return kVals % 32 == 0 || lane + 32 * i < kVals; };
    const StreamK sk = make_sk(a, ncta);
    const SliceWalk W = make_walk<NCOLS>(a);
    RedState es;
    const long long u0 = W.start(sk, cta);
    int u = (int)u0;
    const int uend = W.start(sk, cta + 1);
    while (u < uend) {
        int s, rt, gb, seg0;
        W.locate(u, s, rt, gb, seg0);
        const int pe = min(uend, seg0 + W.len(s));
        const bool full_tile = (W.nsl == 1 && u == seg0 && pe == seg0 + a.NG);
        mbar_wait(&sm.red_full[es.rb], es.rphase);
        const float *rbuf = sm.red + (size_t)es.rb * CW * kVals;
        float v[VPL];
#pragma unroll
        for (int i = 0; i < VPL; i++) {
            float acc = 0.f;
            if (held(i)) {
#pragma unroll
                for (int w = 0; w < CW; w++) acc += rbuf[w * kVals + lane + 32 * i];
            }
            v[i] = acc;
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&sm.red_empty[es.rb]);
        es.next();
        bool do_final = full_tile;
        if (!full_tile && a.atomic_add) {
            // residual accumulate: every contributor of a split tile adds its partial straight into the fp32 residual
            // with RED.ADD (fire and forget: no fence, no counter, nothing on the critical path).  The order of the
            // partial adds is not fixed, so the last bit of the residual may vary run to run.
#pragma unroll
            for (int i = 0; i < VPL; i++) {
                const int idx = lane + 32 * i;
                const int row = idx / NCOLS, col = idx % NCOLS;
                if (held(i) && col < a.M) atomicAdd(reinterpret_cast<float *>(a.y) + (size_t)col * a.ldy + (size_t)rt * 16 + row, v[i]);
            }
        } else if (!full_tile) {
            int last = 0;
            if (W.nsl == 1) {  // one record per CTA and role: 0 = the tile holds the CTA's first unit, 1 = it is the CTA's tail tile
                const long long tb = (long long)rt * a.NG;
                const int c_first = sk.cta_of(tb), c_last = sk.cta_of(tb + a.NG - 1);
                float *mine = a.partials + ((size_t)cta * 2 + ((u0 >= tb) ? 0 : 1)) * kVals;
#pragma unroll
                for (int i = 0; i < VPL; i++)
                    if (held(i)) mine[lane + 32 * i] = v[i];
                __threadfence();
                __syncwarp();
                if (lane == 0) {
                    const unsigned prev = atomicAdd(&a.counters[rt], 1u);
                    last = (prev == (unsigned)(c_last - c_first)) ? 1 : 0;
                    if (last) a.counters[rt] = 0;  // every contributor has arrived: re-arm for the next launch
                }
                last = __shfl_sync(0xffffffffu, last, 0);
                if (last) {
                    __threadfence();
#pragma unroll
                    for (int i = 0; i < VPL; i++) {
                        float acc = 0.f;
                        if (held(i)) {
                            for (int c = c_first; c <= c_last; c++)
                                acc += ldg_cg_f32(a.partials + ((size_t)c * 2 + ((sk.start(c) >= tb) ? 0 : 1)) * kVals + lane + 32 * i);
                        }
                        v[i] = acc;
                    }
                }
            } else {  // one record per (slice, tile): the last of the tile's nsl pieces to arrive sums them in slice order
                auto rec = [&](int q) { return a.partials + ((size_t)q * a.num_tiles + rt) * kVals; };
                float *mine = rec(s);
#pragma unroll
                for (int i = 0; i < VPL; i++)
                    if (held(i)) mine[lane + 32 * i] = v[i];
                __threadfence();
                __syncwarp();
                if (lane == 0) {
                    const unsigned prev = atomicAdd(&a.counters[rt], 1u);
                    last = (prev == (unsigned)(W.nsl - 1)) ? 1 : 0;
                    if (last) a.counters[rt] = 0;
                }
                last = __shfl_sync(0xffffffffu, last, 0);
                if (last) {
                    __threadfence();
                    float p[kMaxSlices][VPL];
#pragma unroll
                    for (int q = 0; q < kMaxSlices; q++)
#pragma unroll
                        for (int i = 0; i < VPL; i++) p[q][i] = (q < W.nsl && held(i)) ? ldg_cg_f32(rec(q) + lane + 32 * i) : 0.f;
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

// ------------------------------------------------------------------------------------------------------------------
// consumer prologue: activations -> (optional RMSNorm) -> four int8 planes per 128-group in MMA-B order, plus the
// per-group step and integer sums, one K-slice at a time.
// ------------------------------------------------------------------------------------------------------------------
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
        // `units` is a multiple of 16, not of 32: trip counts are warp-uniform so that the half-warp shuffles in emit_unit()
        // always run with all 32 lanes.  Loads of several iterations are issued before any is consumed.
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

// first slice of this CTA's unit range (the kernel stages it before the barrier hand-off)
template <int NCOLS>
TCE_DEVINL int first_slice(const KArgs &a, int cta, int ncta) {
    const SliceWalk W = make_walk<NCOLS>(a);
    return W.slice(W.start(make_sk(a, ncta), cta));
}

// ------------------------------------------------------------------------------------------------------------------
// consumer main loop, shared by both consumers: the piece walk, slice staging, the ring and meta-slot steps and the hand-off of
// every piece's partial to the epilogue warp (no consumer-to-consumer wait).  The consumer's own arithmetic comes in as
//   unit(tot, w): accumulate one (16-row tile, group) unit of this warp into the lane's NT partial sums tot[NT];
//   hand(rbuf, tot): store them into the warp's [16 rows][NCOLS] slot of the reduction buffer.
// FULL: every stage carries kStageGroups whole groups (KArgs::full), so the group loop has no bounds checks.
// `staged` = the slice already in shared memory.
// ------------------------------------------------------------------------------------------------------------------
struct UnitIn {    // one (16-row tile, group) unit as lane (g, t) sees it
    uint4 wa, wb;  // the lane's 16 B of weight rows g and g+8
    int G, gl;     // group index in the row and in the staged slice
    float sA, sB;  // scales of rows g and g+8
    int zA, zB;    // their zero points
};

template <int NCOLS, int CW, bool FULL, int NT, class Unit, class Hand>
TCE_DEVINL void consume(const KArgs &a, const Smem &sm, int x_pitch, int staged, int cta, int ncta, int ctid, int cw, int lane, Unit &&unit,
                        Hand &&hand) {
    constexpr int GPW = kStageGroups / CW;  // groups per consumer warp per stage
    const int g = lane >> 2, t = lane & 3;
    const StreamK sk = make_sk(a, ncta);
    const SliceWalk W = make_walk<NCOLS>(a);
    const int sg = FULL ? kStageGroups : a.sg;
    const int rp = sg * 64;  // dense row pitch of the TMA box (2-way bank conflict on the weight LDS, see DESIGN.md)
    const uint32_t w_off = (uint32_t)(g * rp + t * 16);  // the lane's 16 B of weight row g in a group slot
    RingState rs;
    RedState cs;
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
        float tot[NT];
#pragma unroll
        for (int i = 0; i < NT; i++) tot[i] = 0.f;
        for (int g0 = gb; g0 < ge; g0 += sg) {
            const int n = FULL ? kStageGroups : min(sg, ge - g0);
            mbar_wait(&sm.full_bar[rs.stage], rs.phase);
            const uint8_t *sbase = sm.stages + (size_t)rs.stage * kStageBytes + w_off;
#pragma unroll
            for (int q = 0; q < GPW; q++) {
                const int gi = cw + q * CW;
                if (FULL || gi < n) {
                    UnitIn w;
                    w.G = g0 + gi;
                    w.gl = w.G - gs;
                    w.wa = *reinterpret_cast<const uint4 *>(sbase + gi * 64);
                    w.wb = *reinterpret_cast<const uint4 *>(sbase + gi * 64 + 8 * rp);
                    w.sA = __half2float(msA[w.G]);
                    w.sB = __half2float(msB[w.G]);
                    const int zsh = (w.G & 7) * 4;
                    w.zA = (int)((mzA[w.G >> 3] >> zsh) & 0xFu);
                    w.zB = (int)((mzB[w.G >> 3] >> zsh) & 0xFu);
                    unit(tot, w);
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&sm.empty_bar[rs.stage]);
            rs.next_stage(sm.nst);
        }
        mbar_wait(&sm.red_empty[cs.rb], cs.rphase ^ 1);
        hand(sm.red + ((size_t)cs.rb * CW + cw) * 16 * NCOLS, tot);
        __syncwarp();
        if (lane == 0) mbar_arrive(&sm.red_full[cs.rb]);
        cs.next();
        rs.next_piece(sm.nst);
        u = pe;
    }
}

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

// The single-column kernel stages the whole row (nsl == 1), so a unit's activations sit at its group index G.
template <int CW, bool FULL>
TCE_DEVINL void consume1(const KArgs &a, const Smem &sm, int x_pitch, int staged, int cta, int ncta, int ctid, int cw, int lane) {
    const int g = lane >> 2, t = lane & 3;
    const Lane1 L = make_lane1(sm.xs, a.IC, g, t);
    consume<1, CW, FULL, 2>(
        a, sm, x_pitch, staged, cta, ncta, ctid, cw, lane,
        [&](float(&tot)[2], const UnitIn &w) { unit1(L, w.wa, w.wb, w.G, w.sA, w.sB, w.zA, w.zB, sm.gx, sm.gsum, tot[0], tot[1]); },
        [&](float *rbuf, float(&tot)[2]) {
            const float totA = tot[0] + __shfl_xor_sync(0xffffffffu, tot[0], 1);  // (p3, p2) share of t = 0 + (p1, p0) share of t = 1
            const float totB = tot[1] + __shfl_xor_sync(0xffffffffu, tot[1], 1);
            if (t == 0) {
                rbuf[g] = totA;
                rbuf[g + 8] = totB;
            }
        });
}

// Up to 8 activation rows: the 8 MMA columns carry the rows, each plane in its own MMA.  Lane (g, t) accumulates rows g, g+8 of
// columns 2t, 2t+1.
template <int NCOLS, int CW>
TCE_DEVINL void consume_cols(const KArgs &a, const Smem &sm, int x_pitch, int staged, int cta, int ncta, int ctid, int cw, int lane) {
    const int g = lane >> 2, t = lane & 3;
    const int xw = a.sl * 128;
    consume<NCOLS, CW, false, 4>(
        a, sm, x_pitch, staged, cta, ncta, ctid, cw, lane,
        [&](float(&tot)[4], const UnitIn &w) {
            const uint32_t wav[4] = {w.wa.x, w.wa.y, w.wa.z, w.wa.w};
            const uint32_t wbv[4] = {w.wb.x, w.wb.y, w.wb.z, w.wb.w};
            const uint8_t *xp = sm.xs + (size_t)g * x_pitch + ((size_t)w.gl * 16 + t) * 16;
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
            const int G = w.G;
            const int *gs0 = sm.gsum + ((2 * t) * a.NG + G) * 2, *gs1 = sm.gsum + ((2 * t + 1) * a.NG + G) * 2;
            const float st0 = sm.gx[(2 * t) * a.NG + G], st1 = sm.gx[(2 * t + 1) * a.NG + G];
            auto comb = [](int h3, int h2, int l1, int l0, int z, const int *gsp) {
                return 65536.f * (float)((h3 << 8) + h2 - z * gsp[0]) + (float)((l1 << 8) + l0 - z * gsp[1]);
            };
            tot[0] += (w.sA * st0) * comb(c3[0], c2[0], c1[0], c0[0], w.zA, gs0);
            tot[1] += (w.sA * st1) * comb(c3[1], c2[1], c1[1], c0[1], w.zA, gs1);
            tot[2] += (w.sB * st0) * comb(c3[2], c2[2], c1[2], c0[2], w.zB, gs0);
            tot[3] += (w.sB * st1) * comb(c3[3], c2[3], c1[3], c0[3], w.zB, gs1);
        },
        [&](float *rbuf, float(&tot)[4]) {
            rbuf[g * NCOLS + 2 * t] = tot[0];
            rbuf[g * NCOLS + 2 * t + 1] = tot[1];
            rbuf[(g + 8) * NCOLS + 2 * t] = tot[2];
            rbuf[(g + 8) * NCOLS + 2 * t + 1] = tot[3];
        });
}

}  // namespace gemv
}  // namespace tce
