"""Per-token KV-cache attention parity on the GPU (tce_attn_decode) vs the fp32 GQA oracle."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HD = 128


@pytest.fixture(scope="module")
def ctx():
    from tinychatengine_b200.runtime import Context

    c = Context(0)
    yield c
    c.close()


@pytest.mark.parametrize("H,KVH", [(8, 2), (4, 4), (8, 1), (16, 8)])
@pytest.mark.parametrize("past", [0, 1, 5, 127, 128, 129, 255, 256, 257, 300, 1023])
def test_decode_attention_matches_oracle(ctx, H, KVH, past):
    from oracle import capi

    max_ctx = 1024
    rng = np.random.default_rng(1000 * H + past)
    cosb, sinb = capi.rope_tables(max_ctx, HD, 500000.0)
    qkv = rng.standard_normal((H + 2 * KVH) * HD).astype(np.float16)
    pk = (rng.standard_normal((KVH, past, HD)) * 0.7).astype(np.float16)
    pv = rng.standard_normal((KVH, past, HD)).astype(np.float16)
    alpha = 1.0 / np.sqrt(HD)
    q = qkv[: H * HD].astype(np.float32)[None]
    k = qkv[H * HD: (H + KVH) * HD].astype(np.float32)[None]
    v = qkv[(H + KVH) * HD:].astype(np.float32)[None]
    want, fk, fv = capi.llama_attention_core(q, k, v, pk.astype(np.float32) if past else None, pv.astype(np.float32) if past else None,
                                             capi.causal_mask(1, past), cosb, sinb, alpha, H, KVH, HD)
    dev = torch.device("cuda", 0)
    kc = torch.zeros((KVH, max_ctx, HD), dtype=torch.float16, device=dev)
    vc = torch.zeros_like(kc)
    # poison the not-yet-written part of the cache: the kernel must never read it
    kc[:, past:, :] = float("nan")
    vc[:, past:, :] = float("nan")
    if past:
        kc[:, :past] = torch.from_numpy(pk).to(dev)
        vc[:, :past] = torch.from_numpy(pv).to(dev)
    out = torch.zeros(H * HD, dtype=torch.float16, device=dev)
    pos = torch.tensor([past], dtype=torch.int32, device=dev)
    ctx.attn_decode(torch.from_numpy(qkv).to(dev), kc, vc, torch.from_numpy(cosb).to(dev), torch.from_numpy(sinb).to(dev), pos, out, alpha, H, KVH, HD, max_ctx)
    torch.cuda.synchronize()
    got = out.float().cpu().numpy()
    assert np.all(np.isfinite(got))
    scale = max(np.abs(want).max(), 1e-6)
    assert np.abs(got - want[0]).max() / scale <= 3e-3  # fp16 q / K / P / V operands of the tensor-core products, fp16 output
    # the appended rows: rotated K (fp16 rounded) and V, bit-for-bit V
    assert np.allclose(kc[:, past].float().cpu().numpy(), fk[:, past], atol=2e-3, rtol=1e-3)
    assert np.array_equal(vc[:, past].cpu().numpy(), fv[:, past].astype(np.float16))
    if past:
        assert torch.equal(kc[:, :past].cpu(), torch.from_numpy(pk))  # the cached prefix is untouched


@pytest.mark.parametrize("past", [1024, 2047, 3000, 4095])
def test_decode_attention_benchmarked_geometry(ctx, past):
    """The configuration bench.py times: Llama-3-8B heads (H = 32, KVH = 8), max_ctx = 4096, long contexts (the many-way
    flash-decode split and its merge)."""
    from oracle import capi

    H, KVH, max_ctx = 32, 8, 4096
    rng = np.random.default_rng(past)
    cosb, sinb = capi.rope_tables(max_ctx, HD, 500000.0)
    qkv = rng.standard_normal((H + 2 * KVH) * HD).astype(np.float16)
    pk = (rng.standard_normal((KVH, past, HD)) * 0.7).astype(np.float16)
    pv = rng.standard_normal((KVH, past, HD)).astype(np.float16)
    alpha = 1.0 / np.sqrt(HD)
    q = qkv[: H * HD].astype(np.float32)[None]
    k = qkv[H * HD: (H + KVH) * HD].astype(np.float32)[None]
    v = qkv[(H + KVH) * HD:].astype(np.float32)[None]
    want, fk, fv = capi.llama_attention_core(q, k, v, pk.astype(np.float32), pv.astype(np.float32), capi.causal_mask(1, past), cosb, sinb, alpha, H, KVH, HD)
    dev = torch.device("cuda", 0)
    kc = torch.full((KVH, max_ctx, HD), float("nan"), dtype=torch.float16, device=dev)
    vc = torch.full_like(kc, float("nan"))
    kc[:, :past] = torch.from_numpy(pk).to(dev)
    vc[:, :past] = torch.from_numpy(pv).to(dev)
    out = torch.zeros(H * HD, dtype=torch.float16, device=dev)
    pos = torch.tensor([past], dtype=torch.int32, device=dev)
    ctx.attn_decode(torch.from_numpy(qkv).to(dev), kc, vc, torch.from_numpy(cosb).to(dev), torch.from_numpy(sinb).to(dev), pos, out, alpha, H, KVH, HD, max_ctx)
    torch.cuda.synchronize()
    got = out.float().cpu().numpy()
    assert np.all(np.isfinite(got))
    assert np.abs(got - want[0]).max() / max(np.abs(want).max(), 1e-6) <= 3e-3
    assert np.allclose(kc[:, past].float().cpu().numpy(), fk[:, past], atol=2e-3, rtol=1e-3)
    assert np.array_equal(vc[:, past].cpu().numpy(), fv[:, past].astype(np.float16))


def test_multi_step_append_is_consistent(ctx):
    """decode 40 tokens one by one through the in-place cache and compare every step with the oracle fed by its
    own accumulated past (reference test: test_Int4llamaAttention sqlen 9 then 1 with past 9)."""
    from oracle import capi

    H, KVH, max_ctx = 8, 2, 256
    rng = np.random.default_rng(77)
    cosb, sinb = capi.rope_tables(max_ctx, HD, 10000.0)
    dev = torch.device("cuda", 0)
    kc = torch.zeros((KVH, max_ctx, HD), dtype=torch.float16, device=dev)
    vc = torch.zeros_like(kc)
    dcos, dsin = torch.from_numpy(cosb).to(dev), torch.from_numpy(sinb).to(dev)
    out = torch.zeros(H * HD, dtype=torch.float16, device=dev)
    pk = pv = None
    alpha = 1.0 / np.sqrt(HD)
    for step in range(40):
        qkv = rng.standard_normal((H + 2 * KVH) * HD).astype(np.float16)
        pos = torch.tensor([step], dtype=torch.int32, device=dev)
        ctx.attn_decode(torch.from_numpy(qkv).to(dev), kc, vc, dcos, dsin, pos, out, alpha, H, KVH, HD, max_ctx)
        q = qkv[: H * HD].astype(np.float32)[None]
        k = qkv[H * HD: (H + KVH) * HD].astype(np.float32)[None]
        v = qkv[(H + KVH) * HD:].astype(np.float32)[None]
        want, fk, fv = capi.llama_attention_core(q, k, v, pk, pv, capi.causal_mask(1, step), cosb, sinb, alpha, H, KVH, HD)
        fk[:, -1] = fk[:, -1].astype(np.float16).astype(np.float32)
        pk, pv = fk, fv
        got = out.float().cpu().numpy()
        assert np.abs(got - want[0]).max() / max(np.abs(want).max(), 1e-6) <= 3e-3, step


@pytest.mark.parametrize("H,KVH,n,pos0", [(8, 2, 1, 0), (8, 2, 70, 0), (4, 4, 64, 0), (8, 1, 33, 100), (16, 8, 130, 61), (4, 2, 5, 1019)])
def test_prefill_attention_matches_oracle(ctx, H, KVH, n, pos0):
    """tce_attn_prefill (sqlen = n > 1, optional past): vs the fp32 GQA oracle; q rotated in place, K/V rows appended."""
    from oracle import capi

    max_ctx = 1024
    rng = np.random.default_rng(7 * H + n + pos0)
    cosb, sinb = capi.rope_tables(max_ctx, HD, 500000.0)
    QKV = (H + 2 * KVH) * HD
    qkv = rng.standard_normal((n, QKV)).astype(np.float16)
    pk = (rng.standard_normal((KVH, pos0, HD)) * 0.7).astype(np.float16)
    pv = rng.standard_normal((KVH, pos0, HD)).astype(np.float16)
    alpha = 1.0 / np.sqrt(HD)
    f = qkv.astype(np.float32)
    want, fk, fv = capi.llama_attention_core(f[:, : H * HD], f[:, H * HD: (H + KVH) * HD], f[:, (H + KVH) * HD:], pk.astype(np.float32) if pos0 else None,
                                             pv.astype(np.float32) if pos0 else None, capi.causal_mask(n, pos0), cosb, sinb, alpha, H, KVH, HD)
    dev = torch.device("cuda", 0)
    kc = torch.full((KVH, max_ctx, HD), float("nan"), dtype=torch.float16, device=dev)
    vc = torch.full_like(kc, float("nan"))
    if pos0:
        kc[:, :pos0] = torch.from_numpy(pk).to(dev)
        vc[:, :pos0] = torch.from_numpy(pv).to(dev)
    out = torch.zeros((n, H * HD), dtype=torch.float16, device=dev)
    dq = torch.from_numpy(qkv).to(dev)
    ctx.attn_prefill(dq, kc, vc, torch.from_numpy(cosb).to(dev), torch.from_numpy(sinb).to(dev), out, alpha, n, pos0, H, KVH, HD, max_ctx)
    torch.cuda.synchronize()
    got = out.float().cpu().numpy()
    assert np.all(np.isfinite(got))
    assert np.abs(got - want).max() / max(np.abs(want).max(), 1e-6) <= 3e-3  # fp16 q/k/p operands of the tensor-core products
    assert np.allclose(kc[:, pos0:pos0 + n].float().cpu().numpy(), fk[:, pos0:], atol=2e-3, rtol=1e-3)
    assert np.array_equal(vc[:, pos0:pos0 + n].cpu().numpy(), fv[:, pos0:].astype(np.float16))
    if pos0:
        assert torch.equal(kc[:, :pos0].cpu(), torch.from_numpy(pk))
    assert torch.isnan(kc[:, pos0 + n:]).all()  # rows past the new ones are never touched


def test_attention_kernels_against_reference_module_fixture(ctx, golden_dir):
    """The prefill kernel (7 tokens) followed by three decode-kernel steps on the inputs of tests/golden/llama_attention_module.npz:
    compared directly with what the compiled reference Int4llamaAttention module returned.  Its o_proj is a channel selection of the
    int8-round-tripped core output, so the comparison holds to half a quantisation step (amax/254 per 32-block) + fp16 rounding."""
    g = np.load(golden_dir / "llama_attention_module.npz")
    H, KVH, prefill, steps, max_sq = (int(g[k]) for k in ("H", "KVH", "prefill", "steps", "max_sq"))
    from oracle import capi

    hidden = g["hidden"]
    E = hidden.shape[1]
    assert E // H == HD
    cosb, sinb = capi.rope_tables(max_sq, HD, float(g["theta"]))
    dev = torch.device("cuda", 0)
    dcos, dsin = torch.from_numpy(cosb).to(dev), torch.from_numpy(sinb).to(dev)
    # exact in fp16; fancy indexing yields column-major pieces, the kernels take row-major buffers
    qkv_all = np.ascontiguousarray(np.concatenate([hidden[:, g["sel_q"]], hidden[:, g["sel_k"]], hidden[:, g["sel_v"]]], axis=1).astype(np.float16))
    kc = torch.zeros((KVH, max_sq, HD), dtype=torch.float16, device=dev)
    vc = torch.zeros_like(kc)
    outs = torch.zeros((prefill + steps, E), dtype=torch.float16, device=dev)
    alpha = float(g["alpha"])
    dq_all = torch.from_numpy(qkv_all).to(dev)  # kept alive until the stream has consumed it (the caller owns every buffer it passes)
    ctx.attn_prefill(dq_all[:prefill], kc, vc, dcos, dsin, outs[:prefill], alpha, prefill, 0, H, KVH, HD, max_sq)
    torch.cuda.synchronize()
    kerr0 = np.abs(kc[:, :prefill].float().cpu().numpy() - g["final_k"][:, :prefill]).max(axis=(0, 2))
    assert kerr0.max() <= 2e-3 * np.abs(g["final_k"]).max(), f"K rows right after the prefill kernel: error per position {kerr0}"
    for s in range(steps):
        pos = torch.tensor([prefill + s], dtype=torch.int32, device=dev)
        ctx.attn_decode(dq_all[prefill + s], kc, vc, dcos, dsin, pos, outs[prefill + s], alpha, H, KVH, HD, max_sq)
    torch.cuda.synchronize()
    T = prefill + steps
    kerr = np.abs(kc[:, :T].float().cpu().numpy() - g["final_k"]).max(axis=(0, 2))  # per position
    assert kerr.max() <= 2e-3 * np.abs(g["final_k"]).max(), f"K cache error per position {kerr}"
    verr = np.abs(vc[:, :T].float().cpu().numpy() - g["final_v"]).max(axis=(0, 2))
    assert verr.max() == 0, f"V cache error per position {verr}"
    core = outs.float().cpu().numpy()
    ref_core = np.zeros_like(core)
    ref_core[:, g["sel_o"]] = g["out"]  # undo the o_proj channel selection: out[:, j] = roundtrip(core)[:, sel_o[j]]
    amax = np.abs(ref_core.reshape(T, -1, 32)).max(-1, keepdims=True)
    tol = (amax / 254 * 1.05 + 2e-3 * np.abs(ref_core).max()) * np.ones((1, 1, 32), np.float32)
    assert np.all(np.abs(core - ref_core).reshape(T, -1, 32) <= tol)


def _decode_case(H, KVH, past, max_ctx, seed):
    """Seeded inputs of one tce_attn_decode call and the fp32 GQA oracle's answer: (qkv, K cache, V cache, cos, sin, want)."""
    from oracle import capi

    rng = np.random.default_rng(seed)
    cosb, sinb = capi.rope_tables(max_ctx, HD, 500000.0)
    qkv = rng.standard_normal((H + 2 * KVH) * HD).astype(np.float16)
    pk = (rng.standard_normal((KVH, past, HD)) * 0.7).astype(np.float16)
    pv = rng.standard_normal((KVH, past, HD)).astype(np.float16)
    f = qkv.astype(np.float32)[None]
    want, _, _ = capi.llama_attention_core(f[:, : H * HD], f[:, H * HD: (H + KVH) * HD], f[:, (H + KVH) * HD:], pk.astype(np.float32) if past else None,
                                           pv.astype(np.float32) if past else None, capi.causal_mask(1, past), cosb, sinb, 1.0 / np.sqrt(HD), H, KVH, HD)
    dev = torch.device("cuda", 0)
    kc = torch.full((KVH, max_ctx, HD), float("nan"), dtype=torch.float16, device=dev)
    vc = torch.full_like(kc, float("nan"))
    kc[:, :past] = torch.from_numpy(pk).to(dev)
    vc[:, :past] = torch.from_numpy(pv).to(dev)
    return torch.from_numpy(qkv).to(dev), kc, vc, torch.from_numpy(cosb).to(dev), torch.from_numpy(sinb).to(dev), want[0]


def _decode(c, case, H, KVH, past, max_ctx):
    qkv, kc, vc, cosb, sinb, _ = case
    out = torch.zeros(H * HD, dtype=torch.float16, device=qkv.device)
    pos = torch.tensor([past], dtype=torch.int32, device=qkv.device)
    c.attn_decode(qkv, kc, vc, cosb, sinb, pos, out, 1.0 / np.sqrt(HD), H, KVH, HD, max_ctx)
    torch.cuda.synchronize()
    return out.cpu()


def test_decode_and_opt_attention_interleaved_on_one_context():
    """tce_opt_int8_attention and a multi-split tce_attn_decode on one context share no memory: each gives the bits it gives on a fresh
    context, before and after the other."""
    from tinychatengine_b200.runtime import Context

    H8, hd, past8 = 12, 64, 300
    rnd = lambda shape, seed: torch.from_numpy(np.random.default_rng(seed).integers(-127, 128, shape, dtype=np.int8)).cuda()
    q, k, v = rnd((1, H8 * hd), 1), rnd((1, H8 * hd), 2), rnd((1, H8 * hd), 3)
    pk, pv = rnd((H8, past8, hd), 4), rnd((H8, past8, hd), 5)

    def opt(c):
        fk = torch.zeros((H8, past8 + 1, hd), dtype=torch.int8, device="cuda")
        return c.opt_int8_attention(q, k, v, pk, pv, fk, torch.zeros_like(fk), None, 0.0007, 0.011, past8, H8, hd).cpu()

    H, KVH, past, max_ctx = 32, 8, 3000, 4096
    case = _decode_case(H, KVH, past, max_ctx, 11)
    fresh = [Context(0) for _ in range(2)]
    try:
        opt_fresh, dec_fresh = opt(fresh[0]), _decode(fresh[1], case, H, KVH, past, max_ctx)
    finally:
        for c in fresh:
            c.close()
    c = Context(0)
    try:
        opt1 = opt(c)
        dec = _decode(c, case, H, KVH, past, max_ctx)
        opt2 = opt(c)
    finally:
        c.close()
    assert torch.equal(opt1, opt_fresh) and torch.equal(opt2, opt_fresh)
    assert torch.equal(dec, dec_fresh)


def test_decode_workspace_grows():
    """A short-context call sizes the context's split workspace; a later long-context call on the same context grows it."""
    from tinychatengine_b200.runtime import Context

    c = Context(0)
    try:
        for H, KVH, past, max_ctx in ((8, 2, 100, 256), (32, 8, 4000, 4096)):
            case = _decode_case(H, KVH, past, max_ctx, past)
            got, want = _decode(c, case, H, KVH, past, max_ctx).float().numpy(), case[-1]
            assert np.all(np.isfinite(got))
            assert np.abs(got - want).max() / max(np.abs(want).max(), 1e-6) <= 3e-3, (H, past)
    finally:
        c.close()


@pytest.mark.parametrize("chunk", [64, 256])
@pytest.mark.parametrize("H,KVH", [(32, 8), (8, 8)])
def test_span_of_one_row_is_the_decode_call(H, KVH, chunk):
    """tce_attn_span at n = 1 and tce_attn_decode on the same inputs give the same output and K / V cache bits: in one split, on the last row
    of a split, on the first row of the next one, and over many splits."""
    from tinychatengine_b200.runtime import Context

    max_ctx = 4096
    bits = lambda t: t.view(torch.int16)  # the unwritten cache rows are NaN
    c = Context(0)
    try:
        c.set_option("attn_chunk", chunk)
        for past in (0, 37, chunk - 1, chunk, 3000):
            case = _decode_case(H, KVH, past, max_ctx, 7 * past + H)
            qkv, kc, vc, cosb, sinb, _ = case
            kc2, vc2 = kc.clone(), vc.clone()
            dec = _decode(c, case, H, KVH, past, max_ctx)
            out = torch.zeros((1, H * HD), dtype=torch.float16, device=qkv.device)
            c.attn_span(qkv, kc2, vc2, cosb, sinb, out, 1.0 / np.sqrt(HD), 1, past, H, KVH, HD, max_ctx)
            torch.cuda.synchronize()
            assert torch.equal(bits(out[0].cpu()), bits(dec)), past
            assert torch.equal(bits(kc2), bits(kc)) and torch.equal(bits(vc2), bits(vc)), past
    finally:
        c.close()


@pytest.mark.parametrize("H,KVH,hd,max_ctx,chunk,status", [
    (8, 2, 64, 64, None, -2),      # head_dim 64: TCE_ERR_UNSUPPORTED
    (6, 4, 128, 64, None, -1),     # H % KVH != 0: TCE_ERR_INVALID
    (6, 2, 128, 64, None, -3),     # 3 query heads per KV head: no kernel, TCE_ERR_CUDA
    (128, 128, 128, 1025, 1, -3),  # H x nsplit = 128 x 1025 split records: more than one call takes, TCE_ERR_CUDA
])
def test_decode_refusals_write_nothing(H, KVH, hd, max_ctx, chunk, status):
    from tinychatengine_b200.runtime import Context, _ptr

    c = Context(0)
    try:
        if chunk is not None:
            c.set_option("attn_chunk", chunk)
        g = torch.Generator(device="cuda").manual_seed(H + max_ctx)
        rnd = lambda *shape: torch.randn(shape, generator=g, device="cuda").half()
        qkv, kc, vc, out = rnd((H + 2 * KVH) * hd), rnd(KVH, max_ctx, hd), rnd(KVH, max_ctx, hd), rnd(H * hd)
        cosb, sinb = torch.ones((max_ctx, hd), device="cuda"), torch.zeros((max_ctx, hd), device="cuda")
        pos = torch.tensor([max_ctx - 1], dtype=torch.int32, device="cuda")
        before = [t.clone() for t in (out, kc, vc)]
        rc = c.L.tce_attn_decode(c.h, _ptr(qkv), _ptr(kc), _ptr(vc), _ptr(cosb), _ptr(sinb), _ptr(pos), _ptr(out), 1.0 / np.sqrt(hd), H, KVH, hd, max_ctx)
        torch.cuda.synchronize()
        assert rc == status, c.L.tce_last_error()
        assert all(torch.equal(a, b) for a, b in zip(before, (out, kc, vc)))
    finally:
        c.close()
