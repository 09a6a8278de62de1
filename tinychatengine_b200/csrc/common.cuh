// common.cuh -- device-side building blocks shared by the sm_90a kernels of libtce_b200.
// Raw PTX wrappers only (mbarrier, bulk async copy = TMA 1-D, mma.sync, PDL); no CUTLASS, no Triton.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace tce {

#define TCE_DEVINL __device__ __forceinline__

TCE_DEVINL uint32_t smem_u32(const void *p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

// ---------------------------------------------------------------- mbarrier -------------------------------
TCE_DEVINL void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
TCE_DEVINL void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
TCE_DEVINL void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
TCE_DEVINL void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
TCE_DEVINL bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a protocol bug must surface as a launch failure within seconds, never as a hung GPU.
TCE_DEVINL void mbar_wait(uint64_t *bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > 6000000000LL) __trap();  // ~3 s
    }
}

// ---------------------------------------------------------------- TMA 1-D bulk copy (UBLKCP) --------------
TCE_DEVINL uint64_t l2_policy_evict_first() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
TCE_DEVINL uint64_t l2_policy_evict_normal() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
TCE_DEVINL uint64_t l2_policy_evict_last() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
// global -> shared::cta, completion counted in bytes on `bar`.  dst/src 16-B aligned, bytes % 16 == 0.
TCE_DEVINL void bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar, uint64_t policy) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
            smem_u32(dst_smem)),
        "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
        : "memory");
}

// Predicated forms for warp-convergent producers: every lane evaluates the (warp-uniform) operands, one lane issues.
// Keeping the call site convergent lets ptxas hold the addresses in uniform registers instead of emitting a
// per-lane waterfall loop around UBLKCP.
TCE_DEVINL void bulk_g2s_pred(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar, uint64_t policy, uint32_t pred) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %5, 0;\n\t"
        "@p cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;\n\t}" ::"r"(
            smem_u32(dst_smem)),
        "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)), "l"(policy), "r"(pred)
        : "memory");
}
TCE_DEVINL void mbar_arrive_expect_tx_pred(uint64_t *bar, uint32_t bytes, uint32_t pred) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %2, 0;\n\t@p mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n\t}" ::"r"(
                     smem_u32(bar)),
                 "r"(bytes), "r"(pred)
                 : "memory");
}

// 2-D tiled TMA load (UTMALDG): one instruction moves a [rows x bytes] box; coordinates in elements of the map.
TCE_DEVINL void tma_load_2d_pred(void *dst_smem, const void *tmap, int x, int y, uint64_t *bar, uint64_t policy, uint32_t pred) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %6, 0;\n\t"
        "@p cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%2, %3}], [%4], %5;\n\t}" ::"r"(
            smem_u32(dst_smem)),
        "l"(tmap), "r"(x), "r"(y), "r"(smem_u32(bar)), "l"(policy), "r"(pred)
        : "memory");
}

TCE_DEVINL void tma_load_3d_pred(void *dst_smem, const void *tmap, int x, int y, int z, uint64_t *bar, uint64_t policy, uint32_t pred) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %7, 0;\n\t"
        "@p cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%2, %3, %4}], [%5], %6;\n\t}" ::"r"(
            smem_u32(dst_smem)),
        "l"(tmap), "r"(x), "r"(y), "r"(z), "r"(smem_u32(bar)), "l"(policy), "r"(pred)
        : "memory");
}

TCE_DEVINL void bulk_g2s_nohint(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// ---------------------------------------------------------------- programmatic dependent launch -----------
// wait: blocks until every prerequisite grid has completed and its memory is visible (no-op without PDL).
TCE_DEVINL void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
TCE_DEVINL void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ---------------------------------------------------------------- named barriers --------------------------
TCE_DEVINL void named_bar_sync(uint32_t id, uint32_t nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ---------------------------------------------------------------- cp.async, ldmatrix ----------------------
TCE_DEVINL void cp_async16(void *dst_smem, const void *src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst_smem)), "l"(src) : "memory");
}
TCE_DEVINL void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
TCE_DEVINL void ldmatrix_x4(uint32_t &r0, uint32_t &r1, uint32_t &r2, uint32_t &r3, const void *row) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(smem_u32(row)));
}
TCE_DEVINL void ldmatrix_x4_t(uint32_t &r0, uint32_t &r1, uint32_t &r2, uint32_t &r3, const void *row) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(smem_u32(row)));
}

// ---------------------------------------------------------------- legacy tensor path for skinny shapes ----
// D(16x8,f32) += A(16x16,f16,row) * B(16x8,f16,col)
TCE_DEVINL void mma_m16n8k16(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// D(16x8,s32) += A(16x32,u8,row) * B(32x8,s8,col)
TCE_DEVINL void mma_m16n8k32_u8s8(int (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm(
        "mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// ---------------------------------------------------------------- misc ------------------------------------
// same, accumulating onto zero: the compiler feeds RZ, no accumulator initialisation moves
TCE_DEVINL void mma_m16n8k32_u8s8_z(int (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%10,%10,%10};"
                 : "=r"(c[0]), "=r"(c[1]), "=r"(c[2]), "=r"(c[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1), "r"(0));
}
TCE_DEVINL uint32_t lop3_and_or(uint32_t a, uint32_t mask, uint32_t orv) {
    uint32_t r;
    // (a & mask) | orv   -> immLut 0xEA = (a & b) | c
    asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(r) : "r"(a), "r"(mask), "r"(orv));
    return r;
}
TCE_DEVINL uint32_t hsub2_u32(uint32_t a, uint32_t b) {
    uint32_t r;
    asm("sub.f16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
    return r;
}
TCE_DEVINL uint32_t pack_half2(float lo, float hi) {
    __half2 h = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<uint32_t *>(&h);
}
TCE_DEVINL float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
TCE_DEVINL float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
TCE_DEVINL uint4 ldg_nc_u4(const void *p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
// data written by other CTAs of the same grid (stream-K partials): bypass L1
TCE_DEVINL float ldg_cg_f32(const float *p) {
    float r;
    asm volatile("ld.global.cg.f32 %0, [%1];" : "=f"(r) : "l"(p));
    return r;
}

// ---------------------------------------------------------------- host: TMA descriptors ------------------
// cuTensorMapEncodeTiled is a pure host-side encoder; it is reached through the runtime's driver entry point so the library does not
// link libcuda directly.  Looked up once per process; nullptr when the driver does not provide it.
typedef CUresult (*TmapEncodeFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *, const cuuint32_t *,
                                 const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline TmapEncodeFn tmap_encoder() {
    static const TmapEncodeFn fn = [] {
        void *sym = nullptr;
        cudaDriverEntryPointQueryResult q;
        return cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &q) == cudaSuccess ? reinterpret_cast<TmapEncodeFn>(sym) : nullptr;
    }();
    return fn;
}

}  // namespace tce
