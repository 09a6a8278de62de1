// w4a16_act_planes.cuh -- the activation number format of the W4A16 GEMVs: every 128-group of an activation row enters the integer
// tensor path as four int8 planes (32-bit block fixed point) plus the group's step and integer plane sums.  Shared by the stand-alone
// GEMV (w4a16_gemv_impl.cuh) and the persistent decode kernel (decode_persistent.cu), which stage activations the same way.
#pragma once
#include "common.cuh"

namespace tce {
namespace gemv {

constexpr float kActQ = 2130706432.f;  // 127 * 2^24: activation fixed-point full scale (four balanced base-256 digits = int8 planes)

// quantise + stage one 8-element unit (v) of one activation column: xcol = the column's plane buffer (IC = its width in elements; region B
// starts at byte IC * 2), gx / gsum = the column's per-group step and integer sums.  Must be called by all 32 lanes of a warp (half-warp
// shuffles); `valid` masks the stores.
template <int NCOLS>
TCE_DEVINL void emit_unit(uint8_t *xcol, int IC, float *gx, int *gsum, int ui, bool valid, const float (&v)[8], int lane) {
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
    }
}

}  // namespace gemv
}  // namespace tce
