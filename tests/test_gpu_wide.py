"""The prompt-pass kernels at the widths the benchmark times, against the float64 reference of tests/wide_ref.py (pinned against the oracle
by tests/test_wide_ref.py): the CTA-pair W4A16 GEMM and the W8A8 wgmma GEMM with several tiles per cluster (the persistent tile walk and the
TMA ring carried from one tile into the next), the flash prefill attention at 32 and 40 heads over up to 4095 rows, and whole 2-layer
prompt passes at Llama-3-8B and Llama-2-13B widths with the fused epilogues (residual add, SiLU(gate)*up, lm_head row statistics).
Every case prints its worst ratio to its bound."""
import math

import numpy as np
import pytest
import torch

import wide_ref
from wide_ref import row_rel_err, ulp_f16

pytestmark = pytest.mark.gpu

HD = 128
DEV = torch.device("cuda", 0)


@pytest.fixture(scope="module")
def ctx():
    from tinychatengine_b200.runtime import Context

    c = Context(0)
    yield c
    c.close()


def _randn16(shape, seed, scale=1.0):
    g = torch.Generator(device=DEV)
    g.manual_seed(seed)
    return (torch.randn(shape, device=DEV, generator=g) * scale).to(torch.float16)


# ------------------------------------------------------------------------------------------------ a. W4A16 CTA-pair GEMM (EpiHalf)

W4_SHAPES = {"13b-qkv": (15360, 5120), "13b-gate": (13824, 5120), "13b-down": (5120, 13824), "8b-qkv": (6144, 4096), "8b-down": (4096, 14336),
             "lm-chunk": (27648, 4096)}
# fp32 tensor-core accumulation, per unit of sum |x_k w_k|: the worst element on an H100 SXM (700 W) needed 1.05 * 2^-20 (13824-long sums)
C_ACC = 2.0 ** -19


@pytest.mark.parametrize("M", [2048, 1057, 1281])
@pytest.mark.parametrize("name", list(W4_SHAPES))
def test_w4a16_gemm_prefill_shapes(ctx, name, M):
    """tce_w4a16_gemm, every element against the exact product: |y - ref| <= 1/2 ulp_fp16 + C_ACC * sum_k |x_k w_k|.  The output is a view
    into a NaN-filled buffer whose rows before and after must stay NaN."""
    N, K = W4_SHAPES[name]
    assert math.ceil(M / 256) * math.ceil(N / 256) > ctx.num_sms // 2  # more tiles than CTA pairs: a cluster runs several tiles
    from tinychatengine_b200.runtime import random_w4

    t = random_w4(N, K, DEV, 31 + M + N, 0.02, random_zeros=(M != 2048))
    x = _randn16((M, K), M + K)
    buf = torch.full((M + 3, N), float("nan"), dtype=torch.float16, device=DEV)
    y = ctx.w4a16_gemv(x, *t, out=buf[1:M + 1], gemm=True)
    w16 = wide_ref.expand_w4(*t).double()
    xd = x.double()
    ref = xd @ w16.T
    mag = xd.abs() @ w16.abs().T
    del w16
    torch.cuda.synchronize()
    assert torch.isnan(buf[0]).all() and torch.isnan(buf[M + 1:]).all()
    yd = y.double()
    half_ulp = 0.5 * ulp_f16(torch.maximum(ref.abs(), yd.abs()))
    d = (yd - ref).abs()
    ratio = (d / (half_ulp + C_ACC * mag)).nan_to_num(nan=math.inf)
    worst = ratio.max().item()
    c_needed = ((d - half_ulp).clamp_min(0) / mag).max().item()
    print(f"[w4a16 gemm {name} {N}x{K} M={M}] worst |y - ref| / bound = {worst:.3f}; accumulation needs c = {c_needed / 2 ** -20:.2f} * 2^-20")
    if worst > 1.0:
        r, c = divmod(int((ratio > 1.0).flatten().nonzero()[0].item()), N)
        pytest.fail(f"first bad element row {r} col {c} (128-row block {r // 128}, 256-column block {c // 256}): y {yd[r, c].item()} "
                    f"ref {ref[r, c].item()}; worst ratio {worst:.3f}")


# ------------------------------------------------------------------------------------------------ b. W8A8 wgmma GEMM

W8_CASES = [  # (N, K, ctx.w8a8_matmul variant, q_min) at M = 2048: the linears of tools/w8a8_layer_bench.py
    (4096, 4096, 0, -128), (11008, 4096, 0, -128), (11008, 4096, 0, 0), (4096, 11008, 2, -128)]


@pytest.mark.parametrize("N,K,variant,q_min", W8_CASES)
def test_w8a8_wgmma_layer_shapes(ctx, N, K, variant, q_min):
    """Bit for bit: the whole output against the DP4A kernel, and 64 random rows against the oracle (every row is computed on its own)."""
    from oracle import capi
    from tinychatengine_b200.runtime import Context

    M = 2048
    assert math.ceil(M / 128) * math.ceil(N / 256) > ctx.num_sms  # more tiles than CTAs
    g = torch.Generator(device=DEV)
    g.manual_seed(N + K + variant - q_min)
    A = torch.randint(-127, 128, (M, K), dtype=torch.int8, device=DEV, generator=g)
    B = torch.randint(-127, 128, (N, K), dtype=torch.int8, device=DEV, generator=g)
    if variant == 0:
        bias = torch.randint(-127, 128, (N,), dtype=torch.int8, device=DEV, generator=g)
        alpha, beta = (0.00050354, 0.0213013) if K == 4096 and N == 4096 else (0.00045, 0.02)
    else:
        bias = torch.randn(N, device=DEV, generator=g)
        alpha, beta = 0.0007, 1.0
    got = ctx.w8a8_matmul(variant, A, B, bias, alpha, beta, q_min=q_min)
    dp4a = Context(0)
    dp4a.set_option("gemm_min_m", 1 << 30)
    want = dp4a.w8a8_matmul(variant, A, B, bias, alpha, beta, q_min=q_min)
    torch.cuda.synchronize()
    dp4a.close()
    mism = (got.view(torch.int8) != want.view(torch.int8)) if variant == 0 else (got.view(torch.int32) != want.view(torch.int32))
    if mism.any():
        r, c = divmod(int(mism.flatten().nonzero()[0].item()), N)
        pytest.fail(f"wgmma != DP4A at {int(mism.sum())} elements, first row {r} col {c} (128-row block {r // 128}, 256-column block {c // 256})")
    rows = np.sort(np.random.default_rng(N + K).choice(M, 64, replace=False))
    An, Bn, bn = A[rows].cpu().numpy(), B.cpu().numpy(), bias.cpu().numpy()
    if variant == 0:
        ref = capi.int8_matmul(0, An, Bn, bn, None, alpha, beta, q_min, 127)
        assert np.array_equal(got[rows].cpu().numpy(), ref)
    else:
        ref = capi.int8_matmul(4, An, Bn, biasf=bn, alpha=alpha)
        assert np.array_equal(got[rows].cpu().numpy().view(np.uint32), ref.view(np.uint32))
    if q_min == 0:
        assert (got == 0).float().mean().item() > 0.1  # the clamp at 0 is exercised
    print(f"[w8a8 wgmma {N}x{K} v{variant} q_min={q_min}] bit-exact against DP4A and 64 oracle rows")


# ------------------------------------------------------------------------------------------------ c. flash prefill attention

ATTN_CASES = [(H, KVH, n, pos0) for H, KVH in ((32, 8), (40, 40)) for n, pos0 in ((2048, 0), (1000, 3000), (4095, 0), (1025, 3071))]
ATTN_OUT_BOUND = 1.2e-3  # worst row on an H100 SXM (700 W): 6.0e-4 (fp16 P and output)


@pytest.mark.parametrize("H,KVH,n,pos0", ATTN_CASES)
def test_prefill_attention_benchmarked_heads(ctx, H, KVH, n, pos0):
    """tce_attn_prefill against gqa_causal_attention on the fp16 rotated q / k: per row relative to the row's max; the appended K rows to
    2 fp16 ulps, the V rows bit for bit; the cached prefix and the rows past pos0 + n untouched."""
    from oracle import capi

    max_ctx = 4096
    theta = 500000.0 if KVH != H else 10000.0
    cosb, sinb = capi.rope_tables(max_ctx, HD, theta)
    QKV = (H + 2 * KVH) * HD
    qkv = _randn16((n, QKV), 7 * H + n + pos0)
    g = torch.Generator(device=DEV)
    g.manual_seed(pos0 + 1)
    kc = torch.full((KVH, max_ctx, HD), float("nan"), dtype=torch.float16, device=DEV)
    vc = torch.full_like(kc, float("nan"))
    if pos0:
        kc[:, :pos0] = (torch.randn((KVH, pos0, HD), device=DEV, generator=g) * 0.7).to(torch.float16)
        vc[:, :pos0] = torch.randn((KVH, pos0, HD), device=DEV, generator=g).to(torch.float16)
    prefix_k, prefix_v = kc[:, :pos0].clone(), vc[:, :pos0].clone()
    dcos, dsin = torch.from_numpy(cosb).to(DEV), torch.from_numpy(sinb).to(DEV)
    out = torch.zeros((n, H * HD), dtype=torch.float16, device=DEV)
    alpha = 1.0 / math.sqrt(HD)
    dq = qkv.clone()  # q is rotated in place
    ctx.attn_prefill(dq, kc, vc, dcos, dsin, out, alpha, n, pos0, H, KVH, HD, max_ctx)
    c, s = dcos[pos0:pos0 + n], dsin[pos0:pos0 + n]
    q = wide_ref.f16(wide_ref.rope(qkv[:, :H * HD].reshape(n, H, HD), c, s))
    k = wide_ref.f16(wide_ref.rope(qkv[:, H * HD:(H + KVH) * HD].reshape(n, KVH, HD), c, s))
    v = qkv[:, (H + KVH) * HD:].reshape(n, KVH, HD)
    ref = wide_ref.gqa_causal_attention(q, k, v, prefix_k, prefix_v, pos0, alpha)
    torch.cuda.synchronize()
    assert torch.isfinite(out).all()
    e = row_rel_err(out, ref)
    worst = e.max().item()
    # K rows: 2 fp16 ulps, plus the fp32 rounding of the rotation where x0 c - x1 s cancels (|error| < 2^-23 (|x0| + |x1|))
    kin = qkv[:, H * HD:(H + KVH) * HD].reshape(n, KVH, HD).double().abs()
    pair = kin[..., :HD // 2] + kin[..., HD // 2:]
    kref = k.transpose(0, 1)
    k_bound = 2 * ulp_f16(kref) + 2.0 ** -20 * torch.cat([pair, pair], dim=-1).transpose(0, 1)
    k_ratio = ((kc[:, pos0:pos0 + n].double() - kref).abs() / k_bound).nan_to_num(nan=math.inf).max().item()
    print(f"[prefill attention H={H} KVH={KVH} n={n} pos0={pos0}] worst row rel err {worst:.2e} (bound {ATTN_OUT_BOUND:.1e}), "
          f"K rows |d| / bound {k_ratio:.2f}")
    if worst > ATTN_OUT_BOUND:
        r = int((e > ATTN_OUT_BOUND).nonzero()[0].item())
        pytest.fail(f"first bad row {r} (query block {r // 64}): rel err {e[r].item():.2e}")
    assert k_ratio <= 1.0
    assert torch.equal(vc[:, pos0:pos0 + n], v.transpose(0, 1))
    assert torch.equal(kc[:, :pos0], prefix_k) and torch.equal(vc[:, :pos0], prefix_v)
    assert torch.isnan(kc[:, pos0 + n:]).all() and torch.isnan(vc[:, pos0 + n:]).all()


# ------------------------------------------------------------------------------------------------ d. the prompt pass, every row and every layer

# about twice the worst value of an H100 SXM (700 W) run, given after each bound
LOGITS_BOUND = 4.5e-3      # per row: max |d| / max |ref|; 2.27e-3 (13B), 1.78e-3 (8B)
KV1_BOUND = 4.8e-3         # layer-1 K/V rows, same metric; 2.41e-3 (13B), 1.89e-3 (8B)
KV0_ULPS = 4               # layer-0 K/V rows: max |d| over a row in fp16 ulps of the row's max; 2 (13B), 1 (8B)
PREFILL_LAST_BOUND = 2e-3  # prefill()'s last-row logits (lm_head GEMV from the fp32 residual); 9.1e-4


def _two_layer(name):
    from tinychatengine_b200.llama import GEOMETRIES, LlamaGeometry

    b = GEOMETRIES[name]
    return LlamaGeometry(name + "-2l", 2, b.num_heads, b.num_kv_heads, b.embed_dim, b.hidden_dim, b.vocab_size, b.rms_eps, b.rope_theta, b.head_dim)


def _kv_worst(model, K, V, slots, pos0s, lengths):
    """Worst per-row error of the cached K/V rows against the reference rows: (layer 0 in ulps of the row max, layer 1 relative)."""
    w0, w1 = 0.0, 0.0
    for l in range(model.geom.num_layers):
        for which, R in ((0, K), (1, V)):
            for i, (slot, p0, n) in enumerate(zip(slots, pos0s, lengths)):
                got = model.kv_cache(l, which, slot)[:, p0:p0 + n].double()
                ref = R[l][i]
                d = (got - ref).abs().amax(-1)
                mx = ref.abs().amax(-1)
                if l == 0:
                    w0 = max(w0, (d / ulp_f16(mx)).max().item())
                else:
                    w1 = max(w1, (d / mx.clamp_min(1e-30)).max().item())
    return w0, w1


def _report(tag, worst, bounds):
    print(f"[{tag}] " + ", ".join(f"{k} {v:.3g} (bound {bounds[k]:.3g})" for k, v in worst.items()))
    for k, v in worst.items():
        assert v <= bounds[k], (tag, k, v, bounds[k])


def test_prompt_pass_llama3_8b_widths():
    """8 ragged prompts (1057 rows, up to position 4095) into random-filled slots at Llama-3-8B widths with full vocabulary (5 lm_head
    chunks, so EpiRowStats runs with col0 > 0): every position's logits from score_batch, every layer's K/V rows, and no other cache row
    touched."""
    from oracle import capi
    from test_gpu_score import _check_rows, _fill_caches, _snapshot, _tokens
    from tinychatengine_b200.llama import LlamaModel
    from tinychatengine_b200.runtime import Context

    g = _two_layer("llama3-8b")
    ctx = Context(0)
    model = LlamaModel(ctx, g, max_ctx=4096, seed=11, random_zeros=True)
    model.reserve_slots(9)
    _fill_caches(model, 9, 4)
    before = _snapshot(model, 9)
    lengths = [300, 17, 129, 64, 1, 250, 96, 200]
    pos0s = [0, 100, 0, 3000, 4095, 0, 512, 3896]
    slots = [3, 0, 8, 1, 6, 2, 5, 7]
    prompts = [_tokens(n, g.vocab_size, 70 + i) for i, n in enumerate(lengths)]
    n = sum(lengths)
    assert math.ceil(n / 256) * math.ceil(g.embed_dim / 256) > ctx.num_sms // 2
    logits = torch.empty((n, g.vocab_size), dtype=torch.float32, device=DEV)
    model.score_batch(prompts, slots, pos0s, logits=logits)
    after = _snapshot(model, 9)
    _check_rows(before, after, {s: (p0, len(p)) for p, p0, s in zip(prompts, pos0s, slots)})
    cosb, sinb = capi.rope_tables(4096, HD, g.rope_theta)
    past = [[(before[s][l][0][:, :p0], before[s][l][1][:, :p0]) for l in range(g.num_layers)] if p0 else None for s, p0 in zip(slots, pos0s)]
    ref, K, V = wide_ref.prompt_pass(model.W, g, prompts, pos0s, past, cosb, sinb)
    assert torch.isfinite(logits).all()
    e = row_rel_err(logits, ref)
    w0, w1 = _kv_worst(model, K, V, slots, pos0s, lengths)
    worst = {"logits": e.max().item(), "kv layer0 ulps": w0, "kv layer1": w1}
    if worst["logits"] > LOGITS_BOUND:
        print(f"first bad logits row {int((e > LOGITS_BOUND).nonzero()[0].item())}")
    _report("prompt pass llama3-8b widths, 8 prompts", worst, {"logits": LOGITS_BOUND, "kv layer0 ulps": KV0_ULPS, "kv layer1": KV1_BOUND})
    model.close()
    ctx.close()


def test_prompt_pass_llama2_13b_widths():
    """One 2048-token prompt at Llama-2-13B widths (the benchmark's prompt pass at two layers): every position's logits from score_batch and
    the K/V rows of both layers, then prefill() of the same prompt, whose last-row logits come from the lm_head GEMV (final RMSNorm inside,
    from the fp32 residual: other rounding points than the scoring GEMM)."""
    from oracle import capi
    from test_gpu_score import _tokens
    from tinychatengine_b200.llama import LlamaModel
    from tinychatengine_b200.runtime import Context

    g = _two_layer("llama2-13b")
    ctx = Context(0)
    model = LlamaModel(ctx, g, max_ctx=2048, seed=13, random_zeros=True)
    prompt = _tokens(2048, g.vocab_size, 99)
    logits = torch.empty((2048, g.vocab_size), dtype=torch.float32, device=DEV)
    model.score_batch([prompt], [0], [0], logits=logits)
    torch.cuda.synchronize()
    cosb, sinb = capi.rope_tables(2048, HD, g.rope_theta)
    ref, K, V = wide_ref.prompt_pass(model.W, g, [prompt], [0], None, cosb, sinb)
    assert torch.isfinite(logits).all()
    e = row_rel_err(logits, ref)
    w0, w1 = _kv_worst(model, K, V, [0], [0], [2048])
    last = torch.empty(g.vocab_size, dtype=torch.float32)
    model.prefill(prompt, 0, last)
    e_last = row_rel_err(last.to(DEV), ref[-1]).item()
    worst = {"logits": e.max().item(), "kv layer0 ulps": w0, "kv layer1": w1, "prefill last row": e_last}
    if worst["logits"] > LOGITS_BOUND:
        print(f"first bad logits row {int((e > LOGITS_BOUND).nonzero()[0].item())}")
    _report("prompt pass llama2-13b widths, 2048 tokens", worst,
            {"logits": LOGITS_BOUND, "kv layer0 ulps": KV0_ULPS, "kv layer1": KV1_BOUND, "prefill last row": PREFILL_LAST_BOUND})
    model.close()
    ctx.close()
