// kernels.h -- internal C++ launch interface of libtce_b200 (the public face is include/tce_b200.h).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>

namespace tce {

// One context per (device, stream).  Owns the small workspaces the kernels need; never owns caller data.
struct Ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    int num_sms = 0;
    int smem_optin = 0;
    // stream-K fix-up workspace of the W4A16 GEMV: partial records of 16 x 8 floats (2 per CTA, or 1 per (K-slice, row tile) in the
    // multi-column kernel, grown on demand by gemv_partials_reserve) + one arrival counter per row tile
    float *gemv_partials = nullptr;
    int gemv_partial_records = 0;
    unsigned *gemv_counters = nullptr;
    int gemv_max_ctas = 0;
    int gemv_max_tiles = 0;
    unsigned long long *gemv_dbg = nullptr;  // optional phase timestamps (option "gemv_debug")
    unsigned long long *gemv_dbg_keep = nullptr;  // its allocation (kept until the context is destroyed)
    unsigned option_gen = 0;       // bumped by every tce_ctx_set_option / set_stream: captured CUDA graphs hold the context by value and are rebuilt
    // the int8 OPT attention's in-kernel seed hand-off: [0] the seed value of the current call, [1] its epoch flag (zeroed at creation)
    float *opt_seed = nullptr;
    unsigned attn_seed_epoch = 0;  // calls of the int8 OPT attention so far (tags the in-kernel seed hand-off)
    // tunables (env overridable, see ctx.cu)
    int gemv_impl = 1;      // 0 = simple warp-per-row, 1 = TMA + mma.sync stream-K
    int gemv_ctas_per_sm = 1;
    int gemv_consumer_warps = 8;   // 8 or 16 consumer warps per CTA; 0 = chosen per shape
    int gemv_stages = 8;           // TMA ring depth (16 KiB stages, capped by the per-CTA shared-memory share); 0 = deepest that fits
    bool use_pdl = false;
    int pdl_early = 0;  // with use_pdl: 1 = dependents may become resident from the first instruction of each GEMV (2: and no 2-CTA/SM mode)
    // large-M (prefill) path: fp16 expansion of one int4 weight matrix, grown on demand; M >= gemm_min_m goes to the wgmma GEMM
    __half *w16_scratch = nullptr;
    size_t w16_scratch_elems = 0;
    int gemm_min_m = 16;
};

// One-time kernel attribute setup (cudaFuncSetAttribute) is per (kernel, DEVICE): a process may hold contexts on several devices, so each launch site
// keeps one bit per device instead of one flag per process.  Setting the attribute twice from two racing threads is harmless.
struct DeviceOnce {
    std::atomic<unsigned long long> mask{0};
    bool pending(int device) const { return !((mask.load(std::memory_order_acquire) >> (device & 63)) & 1ull); }
    void done(int device) { mask.fetch_or(1ull << (device & 63), std::memory_order_release); }
};

constexpr int kW4Group = 128;  // QK for QM_CUDA (llm/include/common.h:17-21)

inline int zeros_width(int ic, int group) {  // llm/src/nn_modules/cuda/utils.cu:162-178
    int mult = group >= 128 ? 1 : (group == 64 ? 2 : 4);
    int base = (ic / group + 7) / 8;
    return (base + mult - 1) / mult * mult;
}

enum XMode : int { X_HALF = 0, X_RMSNORM_F32 = 1 };
enum EpiMode : int { EPI_STORE_HALF = 0, EPI_STORE_F32 = 1, EPI_ADD_F32 = 2, EPI_SILU_MUL_HALF = 3 };
constexpr int kMaxTP = 8;

struct W4Seg {
    const uint32_t *w;       // [rows][IC/8]
    const uint32_t *zeros;   // [rows][zeros_w]
    const __half *scales;    // [rows][zeros_w*8]
    int rows;                // multiple of 16 (8 in pair mode)
};

struct W4GemvParams {
    W4Seg seg[3];
    int nseg = 1;
    int pair_mode = 0;  // 1: row tile = 8 rows of seg[0] (-> MMA rows 0-7) + the same 8 rows of seg[1] (rows 8-15)
    int IC = 0;
    int M = 1;          // activation rows (<= 8 per launch)
    const void *x = nullptr;
    int x_mode = X_HALF;
    int ldx = 0;        // elements between activation rows
    const float *gamma = nullptr;
    float eps = 0.f;
    void *y = nullptr;
    int epi = EPI_STORE_HALF;
    int ldy = 0;        // elements between output rows
    bool pdl = false;   // launch with programmatic stream serialization
    bool atomic_residual = false;  // EPI_ADD_F32 only: allow RED.ADD for split tiles (non-deterministic last bit)
};

// M = 2..8 at long rows needs one stream-K fix-up record per (K-slice, row tile); the launch grows ctx->gemv_partials when it has too few
// (outside of stream capture only; the context's option generation moves, so captured graphs are rebuilt)
cudaError_t launch_w4a16_gemv(Ctx *ctx, const W4GemvParams &p);
long long w4a16_gemv_fixup_records(const Ctx *ctx, const W4GemvParams &p);  // records a launch of p needs beyond the per-CTA ones
cudaError_t gemv_partials_reserve(Ctx *ctx, long long records);
cudaError_t launch_w4a16_gemv_simple(Ctx *ctx, const W4GemvParams &p);
cudaError_t launch_w4a16_gemv_g64(Ctx *ctx, const __half *x, const uint32_t *w, const uint32_t *zeros, const __half *scales, __half *y, int M, int IC, int OC);
cudaError_t encode_w4_tmap(CUtensorMap *out, const void *w, int rows, int IC, int sg, int box_rows);
// [group][row][64 B] boxes over the groups [g0, g0 + ng) of each row (ng = 0: all IC / 128)
cudaError_t encode_w4_tmap_units(CUtensorMap *out, const void *w, int rows, int IC, int sg, int box_rows, int g0 = 0, int ng = 0);

cudaError_t launch_naive_fp16_int4(Ctx *ctx, const __half *A, const int32_t *B, const __half *scales, __half *C, int M, int IC, int OC, int block);
cudaError_t launch_f32_matmul_transposed(Ctx *ctx, const float *A, const float *B, float *C, int M, int N, int K);

cudaError_t launch_w4_expand(Ctx *ctx, const uint32_t *w, const uint32_t *zeros, const __half *scales, __half *out, int OC, int IC);
// the W4A16 large-M GEMM on the expanded fp16 weights (gemm_tc2.cu): 2-CTA clusters on 256-row tiles, weight tiles multicast
cudaError_t launch_gemm_f16_pair(Ctx *ctx, const __half *X, long long ldx, const __half *W, long long ldw, void *C, long long ldc, int M, int N, int K, int add_f32);
cudaError_t launch_gemm_f16_pair_silu(Ctx *ctx, const __half *X, long long ldx, const __half *W, long long ldw, __half *act, long long ldc, int M, int F, int K);
cudaError_t w4_scratch_reserve(Ctx *ctx, size_t elems);  // grows ctx->w16_scratch (may synchronise the device)

// lm_head scoring: log-softmax statistics of 128 logits of one row (m = max, s = sum of exp(x - m), id = lowest vocabulary id of the max)
struct alignas(16) LmStat {
    float m, s;
    int id, unused;
};
// the lm_head GEMM of one vocabulary chunk (W = its fp16 rows [N][K], vocabulary ids col0 .. col0 + N - 1) with the log-softmax epilogue:
// stats[row][c / 128] for every 128 columns, tgt[row] = the logit of target[row] when the target falls in this chunk, and, when logits is
// not null, logits[row * ld_logits + col0 + c] = every logit.  The [M][N] logits never reach HBM otherwise.
cudaError_t launch_gemm_f16_pair_stats(Ctx *ctx, const __half *X, long long ldx, const __half *W, long long ldw, int M, int N, int K, int col0, LmStat *stats,
                                       int stats_ld, const int *target, float *tgt, float *logits, long long ld_logits);
// folds the n_rec records of each row (in column order) into the running state[row]; with `last`, also writes logprob[row] =
// tgt[row] - logsumexp (NaN where target[row] < 0), greedy[row] and greedy_logprob[row]
cudaError_t launch_lm_stats_merge(Ctx *ctx, const LmStat *stats, int stats_ld, int n_rec, int rows, bool first, bool last, LmStat *state, const int *target,
                                  const float *tgt, float *logprob, int *greedy, float *greedy_logprob);

// host-side mirror of the stream-K partition used by the kernel (unit-tested on the CPU)
struct StreamK {
    long long U;   // total units = tiles * groups
    int nc;        // CTAs
    int NG;        // groups per row tile
    int aligned = 0;  // cut at row-tile boundaries instead of unit boundaries
    int T = 0;        // row tiles (aligned mode)
    int gran = 1;     // unaligned mode: cuts fall on multiples of `gran` units (16 = whole pipeline stages; U % gran == 0)
    __host__ __device__ long long start(int c) const {
        const long long n = aligned ? (long long)T : U / gran;  // cut positions are n * c / nc, in tiles or in `gran` units
        const long long q = (n * nc < 0x7fffffffLL) ? (long long)(((unsigned)n * (unsigned)c) / (unsigned)nc) : (n * (long long)c) / nc;  // 32-bit divide when it fits
        return q * (aligned ? NG : gran);
    }
    // owner of unit u in unaligned mode: the largest c with start(c) <= u
    __host__ __device__ int cta_of(long long u) const {
        const long long Ug = U / gran, ug = u / gran;
        return (int)(((ug + 1) * nc + Ug - 1) / Ug - 1);
    }
};

// Unit order of the W4A16 GEMV over T row tiles of NG groups, cut into K-slices of `sl` groups (the last slice may be shorter): units are
// ordered slice-major, u = T*sl*s + rt*len(s) + (g - s*sl), and a (slice, tile) segment is len(s) consecutive units.  With one slice
// (sl = NG) this is the tile-major stream-K order u = rt*NG + g.  A piece is the part of one segment inside one CTA's range.
struct SliceWalk {
    int T, NG, sl, nsl;
    __host__ __device__ int len(int s) const { return s < nsl - 1 ? sl : NG - s * sl; }
    __host__ __device__ int slice(int u) const {
        if (nsl == 1) return 0;
        const int s = u / (T * sl);
        return s < nsl - 1 ? s : nsl - 1;
    }
    // unit u -> slice s, row tile rt, first group gb of the piece, first unit seg0 of the (slice, tile) segment
    __host__ __device__ void locate(int u, int &s, int &rt, int &gb, int &seg0) const {
        s = slice(u);
        const int base = s * T * sl, L = len(s);
        rt = (u - base) / L;
        seg0 = base + rt * L;
        gb = s * sl + (u - seg0);
    }
    // first unit of segment k (k = s * T + rt; the last slice may be shorter)
    __host__ __device__ int seg_unit(long long k) const {
        const long long kf = (long long)T * (nsl - 1);
        return (int)(k <= kf ? k * sl : kf * sl + (k - kf) * (NG - (nsl - 1) * sl));
    }
    // first unit of CTA c: one slice keeps the stream-K cuts of `sk`; with several the ranges are cut at segment boundaries, so every
    // piece is a whole (slice, tile) segment
    __host__ __device__ int start(const StreamK &sk, int c) const {
        if (nsl == 1) return (int)sk.start(c);
        return seg_unit((long long)T * nsl * c / sk.nc);
    }
};

}  // namespace tce
