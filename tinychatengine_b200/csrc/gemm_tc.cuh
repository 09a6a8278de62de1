// gemm_tc.cuh -- the large-M GEMM of the path on the Hopper tensor cores (wgmma):  C[M][N] = A[M][K] * B[N][K]^T with both operands
// K-major, which is the natural layout of the activations ([tokens][IC]) and of the weights ([OC][IC]) on this path.
//
//   * operands reach shared memory by 2-D TMA (128-byte swizzle, one 128-byte swizzle atom of K per stage row: 64 fp16 or 128 int8),
//   * two consumer warpgroups each own 64 rows of the 128-row tile and issue wgmma.mma_async (m64n128, K = 32 bytes per instruction)
//     straight from the swizzled tiles through shared-memory matrix descriptors; the fp32 / int32 accumulator lives in registers
//     (BLOCK_N / 2 per thread) and the op's epilogue is applied to the fragment in place,
//   * one producer thread keeps the TMA ring full, also while the consumers are in their epilogue.
// Persistent: one CTA per SM walks tiles m-fastest so that concurrently running CTAs share the same B (weight) tile in L2.
//
// CL = 2 (CTA pairs): the two CTAs of a cluster own two vertically adjacent 128-row tiles of the same N block.  Each CTA fetches half
// of the B tile and multicasts it into both CTAs' shared memory, so every weight byte leaves L2 once per 256 output rows.
//
// FUSED: B is the packed QM_CUDA int4 matrix.  TMA brings BLOCK_N rows x 32 bytes of nibbles per k-block; dequant warps (one thread per
// weight row) turn them into the fp16 SWIZZLE_128B operand tile ((q - z) * s, one rounding), fence.proxy.async, arrive on the operand ring.
//
// Roles: warps 0-7 = consumers (warpgroup w owns tile rows 64w..64w+63), warp 8 = TMA producer, FUSED: warps 9.. = dequant.
#pragma once
#include <cuda.h>

#include <type_traits>

#include "common.cuh"
#include "kernels.h"

namespace tce {
namespace tc {

constexpr int kBlockM = 128;
constexpr int kAtomBytes = 128;  // bytes of K per row per stage = one SWIZZLE_128B atom
constexpr int kABytes = kBlockM * kAtomBytes;  // 16 KiB
constexpr int kConsumerThreads = 256;
constexpr int kOpStages = 3;     // FUSED: ring of dequantised fp16 weight tiles

struct GemmArgs {
    alignas(64) CUtensorMap tmA;  // [M][K] box {128 B, 128 rows}, SWIZZLE_128B
    alignas(64) CUtensorMap tmB;  // [N][K] box {128 B, BLOCK_N / 2 rows}, SWIZZLE_128B; FUSED: uint32 [N][K/8], box {8, BLOCK_N / 2}, no swizzle
    int M, N;
    int k_blocks;                 // K * sizeof(element) / 128
    int m_blocks, n_blocks;       // m_blocks counts rows of 128 * CL
    int silu_F;                   // > 0: B = [gate (F rows); up (F rows)]; tile columns 0..127 = gate, 128..255 = up of the SAME 128 channels
    // FUSED
    const __half *scales;
    const uint32_t *zeros;
    int sf_w, zeros_w;
    // epilogue
    void *C;
    long long ldc;                // elements between output rows
    const int8_t *bias8;
    const float *biasf;
    float alpha, beta;
    int q_min, q_max;
};

TCE_DEVINL void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
TCE_DEVINL void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
TCE_DEVINL void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

#define TCE_ACC8(C, d, i) C(d[i]), C(d[i + 1]), C(d[i + 2]), C(d[i + 3]), C(d[i + 4]), C(d[i + 5]), C(d[i + 6]), C(d[i + 7])
#define TCE_ACC64(C, d) \
    TCE_ACC8(C, d, 0), TCE_ACC8(C, d, 8), TCE_ACC8(C, d, 16), TCE_ACC8(C, d, 24), TCE_ACC8(C, d, 32), TCE_ACC8(C, d, 40), TCE_ACC8(C, d, 48), TCE_ACC8(C, d, 56)
#define TCE_D64                                                                                                                                          \
    "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, " \
    "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, "  \
    "%62, %63}"

// D(64 x 128, f32) (+)= A(64 x 16 fp16, smem) * B(128 x 16 fp16, smem)^T
TCE_DEVINL void wgmma_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\twgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " TCE_D64 ", %64, %65, p, 1, 1, 0, 0;\n\t}"
                 : TCE_ACC64("+f", d)
                 : "l"(adesc), "l"(bdesc), "r"(accumulate)
                 : "memory");
}
// D(64 x 128, s32) (+)= A(64 x 32 int8, smem) * B(128 x 32 int8, smem)^T
TCE_DEVINL void wgmma_n128(int (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\twgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 " TCE_D64 ", %64, %65, p;\n\t}"
                 : TCE_ACC64("+r", d)
                 : "l"(adesc), "l"(bdesc), "r"(accumulate)
                 : "memory");
}
// the accumulator is defined only after wgmma.wait_group: keeps the compiler from reading it earlier
TCE_DEVINL void acc_fence(float (&d)[64]) { asm volatile("" : TCE_ACC64("+f", d)::"memory"); }
TCE_DEVINL void acc_fence(int (&d)[64]) { asm volatile("" : TCE_ACC64("+r", d)::"memory"); }

TCE_DEVINL void tma_load_2d(void *dst_smem, const void *tmap, int x, int y, uint64_t *bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(smem_u32(dst_smem)),
                 "l"(tmap), "r"(x), "r"(y), "r"(smem_u32(bar))
                 : "memory");
}
// the box lands at the same shared-memory offset in every CTA of `mask`, and its bytes are counted on the barrier at `bar`'s offset there
TCE_DEVINL void tma_load_2d_multicast(void *dst_smem, const void *tmap, int x, int y, uint64_t *bar, uint16_t mask) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%2, %3}], [%4], %5;" ::"r"(
            smem_u32(dst_smem)),
        "l"(tmap), "r"(x), "r"(y), "r"(smem_u32(bar)), "h"(mask)
        : "memory");
}
TCE_DEVINL void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// arrive on the mbarrier at the same shared-memory offset in CTA `rank` of the cluster (CTA-scope release: a slot is handed back, no data)
TCE_DEVINL void mbar_arrive_cluster(uint64_t *bar, uint32_t rank) {
    uint32_t remote;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(bar)), "r"(rank));
    asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}
// hand a ring slot back to the producers of every CTA that writes into it
template <int CL>
TCE_DEVINL void mbar_release(uint64_t *bar) {
    if constexpr (CL == 1) {
        mbar_arrive(bar);
    } else {
#pragma unroll
        for (uint32_t r = 0; r < (uint32_t)CL; r++) mbar_arrive_cluster(bar, r);
    }
}

// K-major, SWIZZLE_128B shared-memory matrix descriptor (wgmma format): start address >> 4 in bits [0,14), leading byte offset (unused
// for swizzled K-major, set to 1) in [16,30), stride byte offset = 8 rows * 128 B = 1024 B (>> 4) in [32,46), layout type 1
// (SWIZZLE_128B) in [62,64).  Tiles are 1024-byte aligned, so base_offset stays 0.
TCE_DEVINL uint64_t make_sw128_desc(uint32_t smem_addr) {
    const uint32_t lo = ((smem_addr >> 4) & 0x3FFFu) | (1u << 16);
    const uint32_t hi = 64u | (1u << 30);
    return ((uint64_t)hi << 32) | lo;
}

template <int BLOCK_N, bool FUSED>
constexpr int b_stage_bytes() {
    return BLOCK_N * (FUSED ? 32 : kAtomBytes);
}
template <int BLOCK_N, int STAGES, bool FUSED>
constexpr size_t smem_bytes() {
    return 1024 + (size_t)STAGES * (kABytes + b_stage_bytes<BLOCK_N, FUSED>()) + (FUSED ? (size_t)kOpStages * BLOCK_N * kAtomBytes : 0);
}
template <int BLOCK_N, bool FUSED>
constexpr int num_threads() {
    return FUSED ? kConsumerThreads + 32 + BLOCK_N : kConsumerThreads + 128;
}

// 8 nibbles -> 8 fp16 (q - z) * s in k order
TCE_DEVINL uint4 dequant_word(uint32_t w, uint32_t zmagic, __half2 s2) {
    constexpr uint32_t Mk = 0x000F000Fu, MG = 0x64006400u;
    const __half2 zm = *reinterpret_cast<const __half2 *>(&zmagic);
    // (1024 + e0, 1024 + e4), (e1, e5), (e2, e6), (e3, e7)
    uint32_t q[4] = {lop3_and_or(w, Mk, MG), lop3_and_or(w >> 4, Mk, MG), lop3_and_or(w >> 8, Mk, MG), lop3_and_or(w >> 12, Mk, MG)};
    uint32_t p[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const __half2 v = __hmul2(__hsub2(*reinterpret_cast<const __half2 *>(&q[i]), zm), s2);  // exact difference, one rounding
        p[i] = *reinterpret_cast<const uint32_t *>(&v);
    }
    return make_uint4(__byte_perm(p[0], p[1], 0x5410), __byte_perm(p[2], p[3], 0x5410), __byte_perm(p[0], p[1], 0x7632), __byte_perm(p[2], p[3], 0x7632));
}

// Epilogues see the wgmma fragment two columns at a time: Epi::apply(args, row, col, v0, v1) owns C[row][col], C[row][col + 1] (col even,
// col < N).  Epi::kSilu: apply(args, row, col, g0, g1, u0, u1) with the gate / up accumulators of channels col, col + 1.
template <int BLOCK_N, int STAGES, bool I8, bool FUSED, int CL, class Epi>
__global__ void __launch_bounds__(num_threads<BLOCK_N, FUSED>(), 1) gemm_wg_kernel(const __grid_constant__ GemmArgs a) {
    static_assert(BLOCK_N == 128 || BLOCK_N == 256, "BLOCK_N");
    static_assert(!FUSED || (BLOCK_N == 128 && !I8), "the fused unpack is built for 128-row fp16 operand tiles");
    static_assert(!Epi::kSilu || BLOCK_N == 256, "gate and up share a 256-column tile");
    static_assert(CL == 1 || CL == 2, "CL");
    using Acc = typename std::conditional<I8, int, float>::type;
    constexpr int NH = BLOCK_N / 128;                      // 128-column halves of the tile, one wgmma each
    constexpr int kHalfRows = BLOCK_N / 2;                 // rows per B load (one per CTA of a pair)
    constexpr int kBBytes = b_stage_bytes<BLOCK_N, FUSED>();
    constexpr int kLdBytes = kABytes + kBBytes;
    constexpr int kOpBytes = BLOCK_N * kAtomBytes;
    constexpr int kDqWarps = FUSED ? BLOCK_N / 32 : 0;
    constexpr int OS = FUSED ? kOpStages : 1;
    extern __shared__ uint8_t smem_raw[];
    // barriers live at identical offsets in both CTAs of a pair (multicast loads and remote arrives address "the same barrier in the other CTA")
    __shared__ __align__(8) uint64_t full_bar[STAGES], empty_bar[STAGES], op_full[OS], op_empty[OS];

    const uint32_t raw = smem_u32(smem_raw);
    uint8_t *tiles = smem_raw + (((raw + 1023u) & ~1023u) - raw);  // SWIZZLE_128B tiles need 1024-byte alignment
    uint8_t *sLd = tiles;                                           // [STAGES][A 16 KiB | B]
    uint8_t *sOp = tiles + (size_t)STAGES * kLdBytes;               // FUSED: [OS][dequantised B]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t rank = CL == 1 ? 0u : blockIdx.x % CL;
    const int cl = blockIdx.x / CL, ncl = gridDim.x / CL;
    const int tiles_total = a.m_blocks * a.n_blocks;

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; s++) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], CL * (8 + kDqWarps));  // every warp that reads the slot, in every CTA that is written with it
        }
        for (int s = 0; s < OS; s++) {
            mbar_init(&op_full[s], kDqWarps);
            mbar_init(&op_empty[s], 8);
        }
        mbar_fence_init();
    }
    if constexpr (CL == 1) __syncthreads();
    else cluster_sync_all();  // barriers of both CTAs exist before anyone signals across

    if (warp < 8) {
        // ------------------------------------------------------------------------------- consumers: MMA + epilogue
        const int wg = warp >> 2;
        int s = 0, os = 0;
        uint32_t ph = 0, oph = 0;
        Acc acc[NH][64];
        for (int t = cl; t < tiles_total; t += ncl) {
            const int mb = (t % a.m_blocks) * CL + (int)rank, nb = t / a.m_blocks;
            for (int kb = 0; kb < a.k_blocks; kb++) {
                mbar_wait(&full_bar[s], ph);
                if (FUSED) mbar_wait(&op_full[os], oph);
                const uint32_t aaddr = smem_u32(sLd + (size_t)s * kLdBytes) + (uint32_t)wg * 64u * kAtomBytes;
                const uint32_t baddr = FUSED ? smem_u32(sOp + (size_t)os * kOpBytes) : smem_u32(sLd + (size_t)s * kLdBytes + kABytes);
                wg_fence();
#pragma unroll
                for (int h = 0; h < NH; h++) {
                    const uint64_t adesc = make_sw128_desc(aaddr), bdesc = make_sw128_desc(baddr + (uint32_t)h * 128u * kAtomBytes);
#pragma unroll
                    for (int k = 0; k < kAtomBytes / 32; k++)  // 32 bytes of K per instruction; +2 in the (>>4) address field
                        wgmma_n128(acc[h], adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), (kb | k) != 0 ? 1u : 0u);
                }
                wg_commit();
                wg_wait0();  // the other warpgroup's MMAs fill the tensor pipe meanwhile
                if (lane == 0) {
                    mbar_release<CL>(&empty_bar[s]);
                    if (FUSED) mbar_arrive(&op_empty[os]);
                }
                if (++s == STAGES) {
                    s = 0;
                    ph ^= 1u;
                }
                if (FUSED && ++os == OS) {
                    os = 0;
                    oph ^= 1u;
                }
            }
#pragma unroll
            for (int h = 0; h < NH; h++) acc_fence(acc[h]);
            // fragment: thread (warp w, lane l) holds rows 16w + l/4 (+8), n-tile i: columns 8i + 2(l%4) + {0,1}
            const int row0 = mb * kBlockM + wg * 64 + (warp & 3) * 16 + (lane >> 2);
            const int cq = 2 * (lane & 3);
            if constexpr (Epi::kSilu) {
#pragma unroll
                for (int i = 0; i < 16; i++) {
                    const int col = nb * 128 + 8 * i + cq;
                    if (col < a.silu_F) {
                        if (row0 < a.M) Epi::apply(a, row0, col, acc[0][4 * i], acc[0][4 * i + 1], acc[NH - 1][4 * i], acc[NH - 1][4 * i + 1]);
                        if (row0 + 8 < a.M) Epi::apply(a, row0 + 8, col, acc[0][4 * i + 2], acc[0][4 * i + 3], acc[NH - 1][4 * i + 2], acc[NH - 1][4 * i + 3]);
                    }
                }
            } else {
#pragma unroll
                for (int h = 0; h < NH; h++) {
#pragma unroll
                    for (int i = 0; i < 16; i++) {
                        const int col = nb * BLOCK_N + h * 128 + 8 * i + cq;
                        if (col < a.N) {
                            if (row0 < a.M) Epi::apply(a, row0, col, acc[h][4 * i], acc[h][4 * i + 1]);
                            if (row0 + 8 < a.M) Epi::apply(a, row0 + 8, col, acc[h][4 * i + 2], acc[h][4 * i + 3]);
                        }
                    }
                }
            }
        }
    } else if (warp == 8) {
        // ------------------------------------------------------------------------------- TMA producer
        if (lane == 0) {
            asm volatile("prefetch.tensormap [%0];" ::"l"(&a.tmA) : "memory");
            asm volatile("prefetch.tensormap [%0];" ::"l"(&a.tmB) : "memory");
            int s = 0;
            uint32_t ph = 0;
            for (int t = cl; t < tiles_total; t += ncl) {
                const int mb = (t % a.m_blocks) * CL + (int)rank, nb = t / a.m_blocks;
                for (int kb = 0; kb < a.k_blocks; kb++) {
                    mbar_wait(&empty_bar[s], ph ^ 1u);
                    mbar_arrive_expect_tx(&full_bar[s], kLdBytes);
                    uint8_t *dst = sLd + (size_t)s * kLdBytes;
                    tma_load_2d(dst, &a.tmA, kb * (I8 ? kAtomBytes : kAtomBytes / 2), mb * kBlockM, &full_bar[s]);
                    const int bx = FUSED ? kb * 8 : kb * (I8 ? kAtomBytes : kAtomBytes / 2);  // element coordinate along K
#pragma unroll
                    for (int h = 0; h < 2; h++) {
                        if (CL == 2 && h != (int)rank) continue;  // a pair splits the B tile and multicasts the halves
                        const int by = a.silu_F > 0 ? nb * 128 + h * a.silu_F : nb * BLOCK_N + h * kHalfRows;
                        uint8_t *bdst = dst + kABytes + (size_t)h * (kBBytes / 2);
                        if constexpr (CL == 2) tma_load_2d_multicast(bdst, &a.tmB, bx, by, &full_bar[s], (uint16_t)3);
                        else tma_load_2d(bdst, &a.tmB, bx, by, &full_bar[s]);
                    }
                    if (++s == STAGES) {
                        s = 0;
                        ph ^= 1u;
                    }
                }
            }
        }
        __syncwarp();
    } else if (FUSED) {
        // ------------------------------------------------------------------------------- dequant warps: thread r owns weight row r of the tile
        const int r = threadIdx.x - 32 * 9;
        int ls = 0, os = 0;
        uint32_t lph = 0, oph = 0;
        // destination of chunk c (8 fp16) of row r inside a 128B-swizzled K-major tile: 8-row groups of 1024 B, chunk index XOR (row & 7)
        const uint32_t row_off = (uint32_t)(r >> 3) * 1024u + (uint32_t)(r & 7) * 128u;
        const uint32_t sw = (uint32_t)(r & 7);
        for (int t = cl; t < tiles_total; t += ncl) {
            const int nb = t / a.m_blocks;
            const int grow = nb * BLOCK_N + r;
            const bool live = grow < a.N;
            const __half *srow = a.scales + (size_t)(live ? grow : 0) * a.sf_w;
            const uint32_t *zrow = a.zeros + (size_t)(live ? grow : 0) * a.zeros_w;
            // scale / zero point of a 128-k group are requested one group (two k-blocks) before they are used, off the critical path of the ring
            const int ngroups = a.k_blocks >> 1;
            uint32_t zword = 0u, zword_nxt = live ? zrow[0] : 0u, zmagic = 0x64006400u;
            __half s_nxt = live ? srow[0] : __float2half(0.f);
            __half2 s2 = __float2half2_rn(0.f);
            for (int kb = 0; kb < a.k_blocks; kb++) {
                if ((kb & 1) == 0) {  // a new group (rows past N: scale 0 -> zero weights)
                    const int g = kb >> 1;
                    if ((g & 7) == 0) {
                        zword = zword_nxt;
                        if (live && g + 8 < ngroups) zword_nxt = zrow[(g >> 3) + 1];
                    }
                    const uint32_t z = (zword >> (4 * (g & 7))) & 0xFu;
                    zmagic = 0x64006400u | z | (z << 16);
                    s2 = __half2half2(s_nxt);
                    if (live && g + 1 < ngroups) s_nxt = srow[g + 1];
                }
                mbar_wait(&full_bar[ls], lph);
                const uint8_t *src = sLd + (size_t)ls * kLdBytes + kABytes + (size_t)r * 32;
                const uint4 w0 = *reinterpret_cast<const uint4 *>(src), w1 = *reinterpret_cast<const uint4 *>(src + 16);
                __syncwarp();
                if (lane == 0) mbar_release<CL>(&empty_bar[ls]);  // the packed tile is in registers
                if (++ls == STAGES) {
                    ls = 0;
                    lph ^= 1u;
                }
                const uint32_t ww[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
                uint4 o[8];
#pragma unroll
                for (int c = 0; c < 8; c++) o[c] = dequant_word(ww[c], zmagic, s2);
                mbar_wait(&op_empty[os], oph ^ 1u);
                uint8_t *dst = sOp + (size_t)os * kOpBytes + row_off;
#pragma unroll
                for (int c = 0; c < 8; c++) *reinterpret_cast<uint4 *>(dst + (((uint32_t)c ^ sw) << 4)) = o[c];
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes, read by the tensor core (async proxy)
                __syncwarp();
                if (lane == 0) mbar_arrive(&op_full[os]);
                if (++os == OS) {
                    os = 0;
                    oph ^= 1u;
                }
            }
        }
    }
    if constexpr (CL == 2) cluster_sync_all();  // the peer may still write this CTA's shared memory and barriers until it is done too
}

// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*EncodeFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *, const cuuint32_t *,
                             const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeFn encoder() {
    static EncodeFn fn = nullptr;
    if (!fn) {
        void *sym = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &q) == cudaSuccess && sym) fn = reinterpret_cast<EncodeFn>(sym);
    }
    return fn;
}

// [rows][K] K-major operand (fp16 or int8), box {128 B, box_rows}, SWIZZLE_128B
inline cudaError_t encode_kmajor(CUtensorMap *out, const void *base, bool i8, long long rows, long long K, long long ld_elems, int box_rows) {
    EncodeFn fn = encoder();
    if (!fn) return cudaErrorNotSupported;
    const int es = i8 ? 1 : 2;
    const cuuint64_t gdim[2] = {(cuuint64_t)K, (cuuint64_t)rows};
    const cuuint64_t gstride[1] = {(cuuint64_t)(ld_elems * es)};
    const cuuint32_t box[2] = {(cuuint32_t)(kAtomBytes / es), (cuuint32_t)box_rows};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = fn(out, i8 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void *>(base), gdim, gstride, box, estr,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? cudaSuccess : cudaErrorInvalidValue;
}

// packed QM_CUDA int4 weights: uint32 [N][K/8], box {8 words = 64 k, box_rows}, no swizzle
inline cudaError_t encode_w4_packed(CUtensorMap *out, const uint32_t *w, long long N, long long K, int box_rows) {
    EncodeFn fn = encoder();
    if (!fn) return cudaErrorNotSupported;
    const cuuint64_t gdim[2] = {(cuuint64_t)(K / 8), (cuuint64_t)N};
    const cuuint64_t gstride[1] = {(cuuint64_t)(K / 8) * 4};
    const cuuint32_t box[2] = {8u, (cuuint32_t)box_rows};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_UINT32, 2, const_cast<uint32_t *>(w), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                          CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? cudaSuccess : cudaErrorInvalidValue;
}

// a.tmA / a.tmB, M, N, k_blocks and the epilogue fields are set by the caller; fills the block counts and launches the persistent grid
template <int BLOCK_N, int STAGES, bool I8, bool FUSED, int CL, class Epi>
cudaError_t launch_wg(Ctx *ctx, GemmArgs &a) {
    a.m_blocks = (a.M + kBlockM * CL - 1) / (kBlockM * CL);
    a.n_blocks = a.silu_F > 0 ? a.silu_F / 128 : (a.N + BLOCK_N - 1) / BLOCK_N;
    auto kern = gemm_wg_kernel<BLOCK_N, STAGES, I8, FUSED, CL, Epi>;
    constexpr size_t smem = smem_bytes<BLOCK_N, STAGES, FUSED>();
    static DeviceOnce attr_once;  // per instantiation
    if (attr_once.pending(ctx->device)) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        attr_once.done(ctx->device);
    }
    const int tiles = a.m_blocks * a.n_blocks;
    const int clusters = tiles < ctx->num_sms / CL ? tiles : ctx->num_sms / CL;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(clusters * CL));
    cfg.blockDim = dim3((unsigned)num_threads<BLOCK_N, FUSED>());
    cfg.dynamicSmemBytes = smem;
    cfg.stream = ctx->stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = CL;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = CL > 1 ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kern, a);
}

// ------------------------------------------------------------------------------------------------ epilogues shared by the fp16 GEMMs
struct EpiHalf {  // fp32 accumulator -> fp16 C
    static constexpr bool kSilu = false;
    TCE_DEVINL static void apply(const GemmArgs &a, int row, int col, float v0, float v1) {
        __half *dst = reinterpret_cast<__half *>(a.C) + (size_t)row * a.ldc + col;
        if (col + 1 < a.N && (a.ldc & 1) == 0) {
            *reinterpret_cast<uint32_t *>(dst) = pack_half2(v0, v1);
        } else {
            dst[0] = __float2half_rn(v0);
            if (col + 1 < a.N) dst[1] = __float2half_rn(v1);
        }
    }
};

struct EpiAddF32 {  // fp32 accumulator added into an fp32 C (residual stream)
    static constexpr bool kSilu = false;
    TCE_DEVINL static void apply(const GemmArgs &a, int row, int col, float v0, float v1) {
        float *dst = reinterpret_cast<float *>(a.C) + (size_t)row * a.ldc + col;
        if (col + 1 < a.N && (a.ldc & 1) == 0) {
            float2 c = *reinterpret_cast<float2 *>(dst);
            c.x += v0;
            c.y += v1;
            *reinterpret_cast<float2 *>(dst) = c;
        } else {
            dst[0] += v0;
            if (col + 1 < a.N) dst[1] += v1;
        }
    }
};

}  // namespace tc
}  // namespace tce
