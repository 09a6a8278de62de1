"""The wgmma GEMMs (large-M slots of the path) on the GPU.
W4A16 prefill slot (tce_w4a16_gemm, M >= 16): vs the CPU oracle, <= 1e-2 relative (contract) and the 2e-3 internal bar.
W8A8 (tce_w8a8_matmul, M >= 16, K % 128 == 0): BIT-EXACT vs the oracle, and identical to the DP4A kernel."""
import numpy as np
import pytest
import torch

from helpers import assert_w4_close
from test_gpu_w4a16 import make_case, oracle

pytestmark = pytest.mark.gpu

ALPHA, BETA = 0.00050354, 0.0213013


@pytest.fixture(scope="module")
def ctx():
    from tinychatengine_b200.runtime import Context

    c = Context(0)
    yield c
    c.close()


# ragged M (TMA zero-fills the last row block), ragged OC (not a multiple of the 128/256 tile, not a multiple of 8), several k blocks
@pytest.mark.parametrize("m,oc,ic", [(16, 256, 128), (128, 512, 1024), (200, 1000, 1152), (333, 4096, 4096), (17, 44, 256), (64, 11008, 4096),
                                      (130, 300, 11008)])
def test_w4a16_gemm_matches_oracle(ctx, m, oc, ic):
    for rz in (False, True):
        x, w, z, s = make_case(oc, ic, m, 500 + m + oc, rz)
        y = ctx.w4a16_gemv(x, w, z, s, gemm=True)
        torch.cuda.synchronize()
        assert_w4_close(y.float().cpu().numpy(), oracle(x, w, z, s), f"gemm M={m} {oc}x{ic} rz={rz}")


def test_w4a16_gemm_agrees_with_gemv_passes(ctx):
    """Same inputs through the tensor-core path and through the weight-streaming GEMV passes (gemm_min_m raised)."""
    x, w, z, s = make_case(1024, 2048, 48, 77, True)
    y_tc = ctx.w4a16_gemv(x, w, z, s, gemm=True).float()
    ctx.set_option("gemm_min_m", 1 << 30)
    y_gv = ctx.w4a16_gemv(x, w, z, s, gemm=True).float()
    ctx.set_option("gemm_min_m", 16)
    torch.cuda.synchronize()
    scale = y_gv.abs().max().item()
    assert (y_tc - y_gv).abs().max().item() <= 2e-3 * scale


def test_w4a16_gemm_repeated_calls_and_scratch_growth(ctx):
    """Scratch grows with the largest matrix; results stay right when a small matrix follows a large one and back."""
    cases = [make_case(256, 1024, 32, 1, True), make_case(2048, 2048, 32, 2, True), make_case(256, 1024, 32, 1, True)]
    outs = [ctx.w4a16_gemv(*c, gemm=True).float().cpu().numpy() for c in cases]
    assert np.array_equal(outs[0], outs[2])
    assert_w4_close(outs[1], oracle(*cases[1]), "after growth")


def rnd8(shape, seed):
    return np.random.default_rng(seed).integers(-127, 128, shape, dtype=np.int8)


@pytest.mark.parametrize("M,N,K", [(16, 128, 128), (108, 768, 768), (512, 3072, 768), (300, 1000, 1152), (64, 40, 4096), (129, 257, 256)])
def test_w8a8_tc_bit_exact(ctx, M, N, K):
    from oracle import capi

    A, B = rnd8((M, K), 1), rnd8((N, K), 2)
    b8 = rnd8((N,), 3)
    bf = np.random.default_rng(4).standard_normal(N).astype(np.float32)
    dA, dB = torch.from_numpy(A).cuda(), torch.from_numpy(B).cuda()
    db8, dbf = torch.from_numpy(b8).cuda(), torch.from_numpy(bf).cuda()

    def run_all():
        return [ctx.w8a8_matmul(0, dA, dB, db8, ALPHA, BETA, -128, 127).cpu().numpy(), ctx.w8a8_matmul(0, dA, dB, db8, ALPHA, BETA, 0, 127).cpu().numpy(),
                ctx.w8a8_matmul(1, dA, dB, None, ALPHA, 0.0).cpu().numpy(), ctx.w8a8_matmul(2, dA, dB, dbf, ALPHA, 0.0).cpu().numpy(),
                ctx.w8a8_matmul(3, dA, dB, None, ALPHA, 0.0).cpu().numpy()]

    tc = run_all()
    ctx.set_option("gemm_min_m", 1 << 30)
    dp = run_all()
    ctx.set_option("gemm_min_m", 16)
    want = [capi.int8_matmul(0, A, B, b8, None, ALPHA, BETA, -128, 127), capi.int8_matmul(0, A, B, b8, None, ALPHA, BETA, 0, 127),
            capi.int8_matmul(2, A, B, alpha=ALPHA), capi.int8_matmul(4, A, B, biasf=bf, alpha=ALPHA), capi.int8_matmul(6, A, B, alpha=ALPHA)]
    for i, (t, d, w_) in enumerate(zip(tc, dp, want)):
        assert np.array_equal(t, w_), f"wgmma variant #{i}"
        assert np.array_equal(d, w_), f"dp4a variant #{i}"
