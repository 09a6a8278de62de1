"""Host-side model of the decode GEMV's arithmetic (tinychatengine_b200/csrc: emit_unit in w4a16_act_planes.cuh, shared by the persistent decode kernel,
and the group combination of unit1 and consume_cols in w4a16_gemv_impl.cuh): fp16 activations -> 32-bit block fixed point per 128-group -> four balanced base-256 int8 digit planes ->
exact integer dot products with the nibbles -> one fp32 FMA per group.  The model restates that arithmetic in numpy with the SAME integer widths and checks,
without a GPU, the properties DESIGN.md 4.1 claims: the digits reconstruct X, nothing overflows 32 bits at the extreme inputs, and the result stays inside
the parity contract (<= 1e-2 per element wherever |y| > 1e-3 max|y|, SURVEY.md 8(d) config 1) on the heavy-tailed activations that broke round 1's 15-bit
scheme.  The CUDA kernel itself is checked against the oracle on the same cases in tests/test_gpu_w4a16.py; this file guards
the DESIGN of the number format."""
import numpy as np
import pytest

from oracle import capi, quant

Q = np.float32(2130706432.0)  # kActQ = 127 * 2^24


def digits_of(x_group):
    """x fp32 [128] -> (X int64 [128], planes int8 [4][128] = p0..p3, step fp32) exactly as emit_unit computes them (fp32 scale, round to nearest even,
    (X + 0x80808080) ^ 0x80808080 in 32-bit wrap-around arithmetic)."""
    x = np.asarray(x_group, np.float32)
    amax = np.float32(np.abs(x).max())
    qinv = np.float32(Q / amax) if amax > 0 else np.float32(0)
    X = np.rint((x * qinv).astype(np.float32)).astype(np.int64)
    Z = ((X.astype(np.uint64) + np.uint64(0x80808080)) & np.uint64(0xFFFFFFFF)) ^ np.uint64(0x80808080)
    planes = np.stack([((Z >> np.uint64(8 * d)) & np.uint64(0xFF)).astype(np.uint8).view(np.int8) for d in range(4)])
    step = np.float32(amax / Q) if amax > 0 else np.float32(0)
    return X, planes, step


def model_gemv(x_half, w, zeros, scales, group=128):
    """y fp32 [OC] for one activation row, following the kernel: per (row, group) hi = 256*sum(q*p3) + sum(q*p2) - z*(256*sum p3 + sum p2), lo likewise
    with p1, p0 (both int32, asserted), v = 65536*float(hi) + float(lo) in fp32, y += (s * step) * v in fp32."""
    x = np.asarray(x_half, np.float16).astype(np.float32).ravel()
    oc, ic = w.shape[0], w.shape[1] * 8
    q = np.stack([(w >> np.uint32(4 * i)) & np.uint32(0xF) for i in range(8)], axis=2).reshape(oc, ic).astype(np.int64)
    ng = ic // group
    z = np.stack([(zeros >> np.uint32(4 * i)) & np.uint32(0xF) for i in range(8)], axis=2).reshape(oc, -1)[:, :ng].astype(np.int64)
    s = np.asarray(scales, np.float16)[:, :ng].astype(np.float32)
    y = np.zeros(oc, np.float32)
    i32 = np.iinfo(np.int32)
    for g in range(ng):
        X, P, step = digits_of(x[g * group:(g + 1) * group])
        p0, p1, p2, p3 = (P[d].astype(np.int64) for d in range(4))
        assert np.array_equal(X, (p3 << 24) + (p2 << 16) + (p1 << 8) + p0), "digit planes do not reconstruct X"
        assert np.abs(p3).max() <= 127
        qg = q[:, g * group:(g + 1) * group]
        hi = ((qg @ p3) << 8) + (qg @ p2) - z[:, g] * ((p3.sum() << 8) + p2.sum())
        lo = ((qg @ p1) << 8) + (qg @ p0) - z[:, g] * ((p1.sum() << 8) + p0.sum())
        assert i32.min <= hi.min() and hi.max() <= i32.max and i32.min <= lo.min() and lo.max() <= i32.max, "32-bit overflow in the group result"
        v = np.float32(65536.0) * hi.astype(np.float32) + lo.astype(np.float32)
        y = (y + (s[:, g] * step).astype(np.float32) * v).astype(np.float32)
    return y


def random_w4(rng, oc, ic):
    w = rng.integers(0, 2 ** 32, (oc, ic // 8), dtype=np.uint64).astype(np.uint32)
    zw = quant.calculate_zeros_width(ic, 128)
    zeros = rng.integers(0, 2 ** 32, (oc, zw), dtype=np.uint64).astype(np.uint32)
    scales = np.zeros((oc, zw * 8), np.float16)
    scales[:, :ic // 128] = ((0.5 + rng.random((oc, ic // 128))) * 0.004).astype(np.float16)
    return w, zeros, scales


def test_digits_reconstruct_and_error_bound():
    rng = np.random.default_rng(0)
    for trial in range(50):
        x = (rng.standard_normal(128) * 10.0 ** rng.integers(-3, 3)).astype(np.float16).astype(np.float32)
        if trial % 5 == 0:
            x[rng.integers(128)] *= 1000.0
            x = x.astype(np.float16).astype(np.float32)
        X, P, step = digits_of(x)
        assert np.array_equal(X, sum(P[d].astype(np.int64) << (8 * d) for d in range(4)))
        amax = np.abs(x).max()
        err = np.abs(x.astype(np.float64) - float(step) * X)
        assert np.all(err <= np.maximum(np.abs(x) * 2.0 ** -22, amax * 2.0 ** -31)), err.max()  # DESIGN 4.1 bound with fp32-scale slack


def test_extreme_inputs_do_not_overflow_32_bits():
    """All nibbles 15 against zero point 0 (and 0 against 15), every activation at +-full scale: the largest |hi|, |lo| the format can produce."""
    oc, ic = 16, 256
    for nib, zp, sign in ((0xFFFFFFFF, 0x00000000, 1.0), (0x00000000, 0xFFFFFFFF, 1.0), (0xFFFFFFFF, 0x00000000, -1.0), (0xFFFFFFFF, 0xFFFFFFFF, -1.0)):
        w = np.full((oc, ic // 8), nib, np.uint32)
        zeros = np.full((oc, 1), zp, np.uint32)
        scales = np.full((oc, 8), 0.01, np.float16)
        x = np.full((1, ic), sign * 3.0, np.float16)
        y = model_gemv(x, w, zeros, scales)  # the overflow assertions live in the model
        ref = capi.w4a16_gemv(x, w, zeros, scales)[0]
        assert np.abs(y - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max())


@pytest.mark.parametrize("factor", [100.0, 1000.0])
@pytest.mark.parametrize("kill", [False, True])
def test_heavy_tailed_activations_stay_inside_the_contract(factor, kill):
    """One massive channel per 128-group (x100 / x1000); with kill=True the weights on that channel equal the zero point, so the whole output comes
    from the 127 small channels the outlier would swamp in a narrow format (round 1: 7e-2).  Per element, against the oracle (exact fp16 -> fp32)."""
    rng = np.random.default_rng(int(factor) + kill)
    oc, ic = 64, 1024
    w, zeros, scales = random_w4(rng, oc, ic)
    x = rng.standard_normal((1, ic)).astype(np.float32)
    hot = np.arange(ic // 128) * 128 + rng.integers(0, 128, ic // 128)
    x[0, hot] *= factor
    x = x.astype(np.float16)
    if kill:
        for g, c in enumerate(hot):  # nibble of channel c := zero point of (row, group g)
            zn = (zeros[:, g // 8] >> np.uint32(4 * (g % 8))) & np.uint32(0xF)
            word, sh = c // 8, np.uint32(4 * (c % 8))
            w[:, word] = (w[:, word] & ~(np.uint32(0xF) << sh)) | (zn << sh)
    ref = capi.w4a16_gemv(x, w, zeros, scales)[0]
    y = model_gemv(x, w, zeros, scales)
    big = np.abs(ref) > 1e-3 * np.abs(ref).max()
    rel = np.abs(y - ref)[big] / np.abs(ref)[big]
    assert rel.max() <= 1e-2, rel.max()
    assert rel.max() <= 1e-4  # what the 32-bit format actually delivers (the remainder is fp32 accumulation order)
