// persistent.h -- host/device interface of the persistent Llama decode kernel (decode_persistent.cu).
//
// One kernel per decoded token, one CTA per SM, launched as clusters of two CTAs: both CTAs of a cluster walk the same GEMV tiles, each
// over its half of the 128-groups (k_range), and one CTA per tile adds its partner's 32 row sums (st.async over DSMEM).  Everything a
// token needs from HBM -- packed weights, their repacked scales/zeros, and the K/V cache rows -- flows through ONE ring of TMA stages per
// CTA that is filled by a producer warp which depends on nothing but static data, so it runs ahead across all phase boundaries.  Phases
// hand their results to each other through flag-carrying 8-byte words (value + phase tag, stored and loaded as one unit): there is no
// grid barrier, fence or counter between the five phases of a layer -- a consumer simply spins on the words it needs.
#pragma once
#include "kernels.h"

namespace tce {
namespace pk {

constexpr int kCW = 16;                          // consumer warps
constexpr int kAuxWarps = 4;                     // warpgroup 0: loader warp, epilogue warp, two spare warps that only donate their registers
constexpr int kThreads = 32 * (kAuxWarps + kCW); // 640
constexpr int kConsumerThreads = 32 * kCW;       // 512
constexpr int kHalfBytes = 16384;                // 64 K rows or 64 V rows (one half of an attention stage)
constexpr int kTileRows = 32;                    // rows of a GEMV tile (gate | up: 16 gate rows + 16 up rows of the same 16 channels)
constexpr int kBoxGroups = 16;                   // 128-k groups per weight box; a stage carries one box (16 groups x 32 rows x 64 B = 32 KiB)
constexpr int kMetaOff = 2 * kHalfBytes;         // the box's record: scales half[16 groups][8][4] (rows g, g+8, g+16, g+24 adjacent) then zero points u8[16][8][4]
constexpr int kBoxMetaBytes = 1536;
constexpr int kStageBytes = 34816;               // 32 KiB + 1.5 KiB meta (+ pad), 1 KiB multiple (128B-swizzle atoms of the K/V boxes)
constexpr int kMaxStages = 6;
constexpr int kRedBufs = 3;
constexpr int kPairSlots = 8;                    // tile partials in flight from one CTA to its partner
constexpr int kKvChunk = 64;                     // cached positions per ring stage (K rows in the first half, V rows in the second)

enum XMode : int { PX_HALF = 0, PX_RMS_F32 = 1 };
enum Epi : int { PE_HALF_LL = 0, PE_DELTA_LL = 1, PE_SILU_LL = 2, PE_LOGITS = 3 };
enum OpIdx : int { OPI_QKV = 0, OPI_O = 1, OPI_GATEUP = 2, OPI_DOWN = 3, OPI_LMHEAD = 4, OPI_COUNT = 5 };

// shape of one GEMV op; identical for every layer, so it lives in the kernel parameter block.
struct GemvOp {
    int IC, NG;          // input channels, 128-groups per row
    int num_tiles;       // 32-row tiles (gate | up: 16 gate rows + 16 up rows)
    int nseg, gate_up;   // row segments (q|k|v = 3); gate_up: tiles interleave 16 rows of each of the two segments
    int rows0, rows1;    // rows of segments 0 and 1 (tile -> segment)
    int x_mode, epi;
};

// The K range a CTA reduces over: cluster rank 0 the first ceil(NG / 2) groups, rank 1 the rest.  Contiguous halves keep every TMA box a
// plain range of groups of one tensor map, encoded over the half (box width bw), so a box never reads the partner's groups.  The range is
// walked as `nb` boxes of 16 groups per tile, tile by tile, one box per ring stage: at NG = 32 (IC = 4096) a stage is a whole tile.  Group gi
// of a box sits at gi * 2 KiB (gate | up: the 16 gate rows at gi KiB, the 16 up rows 16 KiB further); a box that runs past the range is
// zero-filled by TMA and still counts its full bytes.  Scales and zeros follow the same walk: one 1536-byte record per (tile, box).
struct KRange {
    int g0, ng;  // first group, groups
    int nb, bw;  // boxes per tile, TMA box width in groups
};
__host__ __device__ inline KRange k_range(int NG, int rank) {
    KRange k;
    const int h = (NG + 1) / 2;
    k.g0 = rank ? h : 0;
    k.ng = rank ? NG - h : h;
    k.nb = (k.ng + kBoxGroups - 1) / kBoxGroups;
    k.bw = k.ng < kBoxGroups ? k.ng : kBoxGroups;
    return k;
}
// input channels of the activation-plane buffer of one op (planes of the CTA's K range, the larger one of rank 0; region B starts at twice
// this many bytes)
__host__ __device__ inline int plane_ic(int NG) { return k_range(NG, 0).ng * 128; }

struct LayerDesc {       // per layer, global memory
    const uint8_t *meta[2][4];   // repacked scales|zeros of qkv, o, gate_up, down over the K range of cluster rank 0 / 1: [tile][box][1536 B]
    const float *input_norm, *post_norm;
    __half *k_cache, *v_cache;   // [KVH][max_ctx][128] of this layer (append)
    int k_row0, v_row0;          // first row of this layer's K / V slab in the cache tensor map
    int pad[2];
};

struct Args {
    GemvOp op[OPI_COUNT];
    const LayerDesc *layers;
    int num_layers;
    const CUtensorMap *maps;     // [2][num_layers * 7 (q k v o gate up down) + 1 (lm_head)] weight maps over the K range of cluster rank 0 / 1,
                                 // then the KV cache map
    const uint8_t *lm_meta[2];
    const float *final_norm;
    const __half *embed;         // [rows][E]
    int embed_rows;
    // phase-to-phase hand-off buffers: 8-byte words {payload, tag}
    uint2 *delta_ll[2];          // [tp][E] o_proj (0) / down_proj (1) outputs per rank slot: fp32 payload (added to the residual by every reader)
    uint2 *qkv_ll;               // [(H + 2 KVH) * 64]  half2 payload
    uint2 *attn_ll;              // [H * 64]            half2 payload
    uint2 *act_ll;               // [F / 2]             half2 payload
    uint2 *part_ll;              // [H][nsplit_max][130] fp32 payload: flash-decode partials (o[128], m, l)
    float *logits;
    const int *tokpos;           // {token, position}
    int *next_token;
    unsigned long long *argmax_cell;
    unsigned *done;              // monotonic arrival counter of the final phase
    unsigned *epoch;             // launches completed so far
    int *error;                  // device error word (bad token / position)
    const float *cos, *sin;      // [max_ctx][128]
    float alpha, eps;
    int H, KVH, nrep, max_ctx, E, V, F;
    int nsplit_max;
    int nst;                     // ring depth
    int xs_bytes;                // activation-plane buffer (also the attention scratch)
    int max_ng;
    // tensor parallel (tp_size > 1): every rank writes its o_proj / down_proj outputs into slot `tp_rank` of every rank's delta buffers
    int tp_size, tp_rank;
    uint2 *tp_delta[2][kMaxTP];  // [which][peer]: that peer's delta_ll[which] base
    uint2 *tp_keys[kMaxTP];      // every rank's arg-max key words [P][2]
    int vocab_base;              // global index of this rank's first vocabulary row
    unsigned long long *dbg;     // optional (TCE_PK_DEBUG=1): globaltimer stamps [cta][phase][8]: 0 phase entered, 1 staged, 2 consumed, 3 results written, 4.. sub-steps
};

size_t smem_bytes(const Args &a);
// shared-memory plan: the activation-plane buffer and the ring depth that fits `smem_optin` next to the fixed buffers (a.nst = 0:
// does not fit).  Needs a.op, a.nrep, a.E and a.max_ng.
void plan_smem(Args &a, int smem_optin);
int attn_scratch_bytes(int nrep);
int attn_nsplit_max(int ncta, int KVH, int max_ctx);
cudaError_t launch(Ctx *ctx, const Args &a, cudaStream_t stream);
bool pair_supported(Ctx *ctx, const Args &a);  // the grid fits as co-resident clusters of two CTAs
// one-off repack of a (possibly multi-segment / gate|up interleaved) matrix's scales and zeros over the K range `kr` into per-(tile, box)
// records (num_tiles * kr.nb * kBoxMetaBytes bytes)
cudaError_t repack_meta(Ctx *ctx, const W4Seg *segs, int nseg, int gate_up, int IC, const KRange &kr, uint8_t *out, cudaStream_t stream);
cudaError_t encode_kv_tmap(CUtensorMap *out, const void *kv, long long rows);

}  // namespace pk
}  // namespace tce
