// kv_copy.cu -- KV-cache row copies between positions and slots, with the K rows re-rotated by the position change.
//
// The cache stores keys after RoPE, so a K row that moves from position p to p + d is rotated by d (rotate-half, dim j with j + 64, the
// pairing of rope_kv_append_kernel): with c = cos[|d|], s = sign(d) * sin[|d|] from the model's own tables,
//   r_j = x_j c_j - x_{j+64} s_j,   r_{j+64} = x_{j+64} c_{j+64} + x_j s_{j+64},
// each product and each sum rounded on its own in fp32 (no FMA contraction), then rounded to fp16: a numpy restatement reproduces it bit
// for bit.  V rows, and K rows with d = 0, are byte copies.  The kernel is HBM-bound: every source row is read once with 16-byte loads and
// written to every destination.
#include "common.cuh"
#include "kernels_attn.h"

namespace tce {
namespace {

constexpr int kHD = 128;                       // head_dim (LlamaDecoder::create requires it)
constexpr int kThreads = 256;
constexpr int kRowsPerPass = kThreads / 8;     // 8 threads per row: thread p holds dims 8p..8p+7 and 64+8p..64+8p+7
constexpr int kUnroll = 4;
constexpr int kTileRows = kRowsPerPass * kUnroll;

TCE_DEVINL void rotate8(const uint4 &lo, const uint4 &hi, const float *c, const float *s, uint4 &out_lo, uint4 &out_hi) {
    const __half *xl = reinterpret_cast<const __half *>(&lo), *xh = reinterpret_cast<const __half *>(&hi);
    __half *rl = reinterpret_cast<__half *>(&out_lo), *rh = reinterpret_cast<__half *>(&out_hi);
#pragma unroll
    for (int e = 0; e < 8; e++) {
        const float xj = __half2float(xl[e]), xk = __half2float(xh[e]);
        rl[e] = __float2half_rn(__fsub_rn(__fmul_rn(xj, c[e]), __fmul_rn(xk, s[e])));
        rh[e] = __float2half_rn(__fadd_rn(__fmul_rn(xk, c[8 + e]), __fmul_rn(xj, s[8 + e])));
    }
}

}  // namespace

// Outside the anonymous namespace so that its symbol, tce::kv_copy_kernel, is the same in every build (profiles key on it).
// grid (tiles, slabs): blockIdx.y is one (layer, K|V, head) slab of max_ctx contiguous rows.  Without in_place every CTA owns tiles
// blockIdx.x, blockIdx.x + gridDim.x, ... of the n rows.  With in_place (one destination overlapping the source in its slot) the grid has
// one CTA per slab, which walks the tiles away from the overlap (ascending when the rows move down, descending when they move up) and
// reads a whole tile before writing any of it: a tile never overwrites a source row that is still to be read.
__global__ void __launch_bounds__(kThreads) kv_copy_kernel(const KvCopyArgs a) {
    __shared__ __align__(16) float tab[kMaxKvCopyDst][2][kHD];  // per destination: cos[|d|] | sign(d) * sin[|d|]
    const int slab = blockIdx.y;
    const bool is_k = ((slab / a.num_kv_heads) & 1) == 0;
    if (is_k) {
        for (int i = threadIdx.x; i < a.n_dst * 2 * kHD; i += kThreads) {
            const int d = i / (2 * kHD), e = i % (2 * kHD), delta = a.dst_pos[d] - a.src_pos, ad = delta < 0 ? -delta : delta;
            tab[d][e / kHD][e % kHD] = e < kHD ? a.cos[(size_t)ad * kHD + e] : (delta < 0 ? -a.sin[(size_t)ad * kHD + e - kHD] : a.sin[(size_t)ad * kHD + e - kHD]);
        }
        __syncthreads();
    }
    const size_t base = (size_t)slab * a.max_ctx * kHD;
    const int p = threadIdx.x & 7, r = threadIdx.x >> 3;
    const int n_tiles = (a.n + kTileRows - 1) / kTileRows;
    for (int it = blockIdx.x; it < n_tiles; it += gridDim.x) {
        const int t = a.reverse ? n_tiles - 1 - it : it;
        uint4 lo[kUnroll], hi[kUnroll];
#pragma unroll
        for (int u = 0; u < kUnroll; u++) {
            const int row = t * kTileRows + u * kRowsPerPass + r;
            if (row < a.n) {
                const __half *x = a.src + base + (size_t)(a.src_pos + row) * kHD;
                lo[u] = *reinterpret_cast<const uint4 *>(x + 8 * p);
                hi[u] = *reinterpret_cast<const uint4 *>(x + 64 + 8 * p);
            }
        }
        if (a.in_place) __syncthreads();  // the whole tile is read before any row of it is overwritten
        for (int d = 0; d < a.n_dst; d++) {
            const bool rot = is_k && a.dst_pos[d] != a.src_pos;
            float c[16], s[16];  // [0, 8): dims 8p.., [8, 16): dims 64 + 8p..
            if (rot) {
#pragma unroll
                for (int q = 0; q < 2; q++) {
                    const float4 *tc = reinterpret_cast<const float4 *>(&tab[d][0][q * 64 + 8 * p]), *ts = reinterpret_cast<const float4 *>(&tab[d][1][q * 64 + 8 * p]);
                    *reinterpret_cast<float4 *>(&c[q * 8]) = tc[0];
                    *reinterpret_cast<float4 *>(&c[q * 8 + 4]) = tc[1];
                    *reinterpret_cast<float4 *>(&s[q * 8]) = ts[0];
                    *reinterpret_cast<float4 *>(&s[q * 8 + 4]) = ts[1];
                }
            }
#pragma unroll
            for (int u = 0; u < kUnroll; u++) {
                const int row = t * kTileRows + u * kRowsPerPass + r;
                if (row >= a.n) continue;
                __half *y = a.dst[d] + base + (size_t)(a.dst_pos[d] + row) * kHD;
                uint4 ol = lo[u], oh = hi[u];
                if (rot) rotate8(lo[u], hi[u], c, s, ol, oh);
                *reinterpret_cast<uint4 *>(y + 8 * p) = ol;
                *reinterpret_cast<uint4 *>(y + 64 + 8 * p) = oh;
            }
        }
    }
}

cudaError_t launch_kv_copy(Ctx *ctx, const KvCopyArgs &a, int n_slabs) {
    if (a.n <= 0) return cudaSuccess;
    if (a.n_dst < 1 || a.n_dst > kMaxKvCopyDst || n_slabs < 1) return cudaErrorInvalidValue;
    const int n_tiles = (a.n + kTileRows - 1) / kTileRows;
    kv_copy_kernel<<<dim3(a.in_place ? 1 : n_tiles, n_slabs), kThreads, 0, ctx->stream>>>(a);
    return cudaGetLastError();
}

}  // namespace tce
