"""The two remaining MatmulOperator methods of the reference's CUDA build (fp16-int4 host reference in the AWQ-GEMM layout,
fp32 transposed matmul): BIT-EXACT against the oracle and against the committed golden vectors produced by the reference."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from tinychatengine_b200.runtime import Context

    c = Context(0)
    yield c
    c.close()


def test_fp16_int4_golden(ctx, golden_dir):
    g = np.load(golden_dir / "kernels_generic.npz")
    A, qs, d = g["f16_A"], g["f16_qs"], g["f16_d"]
    got = ctx.naive_fp16_int4(torch.from_numpy(A.view(np.float16)).cuda(), torch.from_numpy(qs).cuda(), torch.from_numpy(d.view(np.float16)).cuda())
    assert np.array_equal(got.cpu().numpy().view(np.uint16), g["f16_C"].view(np.uint16))


@pytest.mark.parametrize("M,IC,OC", [(1, 128, 8), (3, 256, 64), (2, 1024, 136)])
def test_fp16_int4_vs_oracle(ctx, M, IC, OC):
    from oracle import capi

    rng = np.random.default_rng(M * 7 + OC)
    A = (rng.standard_normal((M, IC)) * 0.5).astype(np.float16)
    qs = rng.integers(-(2**31), 2**31, (IC, OC // 8), dtype=np.int64).astype(np.int32)
    d = (rng.random((IC // 128, OC)) * 0.02 + 0.001).astype(np.float16)
    want = np.zeros((M, OC), np.uint16)
    capi.lib().orc_naive_mat_mul_fp16_int4(A.view(np.uint16), qs, d.view(np.uint16), want, M, IC, OC, 128)
    got = ctx.naive_fp16_int4(torch.from_numpy(A).cuda(), torch.from_numpy(qs).cuda(), torch.from_numpy(d).cuda())
    assert np.array_equal(got.cpu().numpy().view(np.uint16), want)


def test_f32_transposed_golden_and_oracle(ctx, golden_dir):
    from oracle import capi

    g = np.load(golden_dir / "kernels_generic.npz")
    got = ctx.f32_matmul_transposed(torch.from_numpy(g["t_A"]).cuda(), torch.from_numpy(g["t_B"]).cuda())
    assert np.array_equal(got.cpu().numpy(), g["t_C"])
    rng = np.random.default_rng(5)
    A, B = rng.standard_normal((5, 333)).astype(np.float32), rng.standard_normal((129, 333)).astype(np.float32)
    want = np.zeros((5, 129), np.float32)
    capi.lib().orc_mat_mul_transposed(A, B, want, 5, 129, 333)
    got = ctx.f32_matmul_transposed(torch.from_numpy(A).cuda(), torch.from_numpy(B).cuda())
    assert np.array_equal(got.cpu().numpy(), want)


@pytest.mark.parametrize("rows,dim", [(1, 4096), (5, 768), (3, 130), (64, 4096)])
def test_layernorm_q_bit_exact(ctx, rows, dim):
    """tce_layernorm_q == LayerNormQ::forward (llm/src/ops/LayerNormQ.cc:12-52) as restated by the oracle (itself pinned bit-for-bit against
    the compiled reference op, tests/test_oracle_golden.py): int8 outputs identical, including rounding ties."""
    from oracle import capi

    rng = np.random.default_rng(rows * 1000 + dim)
    x = (rng.standard_normal((rows, dim)) * 60).astype(np.float32)
    w = (1 + 0.1 * rng.standard_normal(dim)).astype(np.float32)
    b = rng.standard_normal(dim).astype(np.float32)
    want = np.zeros((rows, dim), np.int8)
    capi.lib().orc_layernorm_q(x, w, b, want, rows, dim)
    dev = torch.device("cuda", 0)
    got = ctx.layernorm_q(torch.from_numpy(x).to(dev), torch.from_numpy(w).to(dev), torch.from_numpy(b).to(dev))
    torch.cuda.synchronize()
    assert np.array_equal(got.cpu().numpy(), want)
    a2 = torch.from_numpy(x).to(dev)
    assert torch.equal(ctx.add_f32(a2, a2), a2 + a2)


@pytest.mark.parametrize("n", [1, 1000, 128256])
def test_argmax_f32_first_index_of_the_maximum(ctx, n):
    """tce_argmax_f32 against numpy: the lowest index wins when the maximum repeats, a maximum at the last index is found, and an input
    with no value above -inf returns 0"""
    rng = np.random.default_rng(n)
    x = rng.standard_normal(n).astype(np.float32)
    cases = [x.copy()]
    rep = x.copy()
    rep[rng.choice(n, size=min(n, 5), replace=False)] = 7.0
    cases.append(rep)
    last = x.copy()
    last[-1] = 9.0
    cases.append(last)
    for c in cases:
        got = ctx.argmax_f32(torch.from_numpy(c).cuda())
        assert int(got.item()) == int(np.argmax(c))
    for fill in (-np.inf, np.nan):
        assert int(ctx.argmax_f32(torch.full((n,), fill, dtype=torch.float32, device="cuda")).item()) == 0
