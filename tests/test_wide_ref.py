"""The float64 reference of tests/test_gpu_wide.py (tests/wide_ref.py) pinned on the CPU: the weight expansion bit for bit against the QM_CUDA
unpacking of formats.py, the attention against the oracle's GQA core, and the prompt pass against oracle/llama_ref.py::llama_forward, the
composition that tests/test_oracle_golden.py pins against the compiled reference model."""
import numpy as np
import pytest
import torch

import wide_ref
from oracle import capi

HD = 128


@pytest.mark.parametrize("OC,IC", [(64, 1024), (40, 11008), (16, 4096)])
@pytest.mark.parametrize("random_zeros", [False, True])
def test_expand_w4_bit_exact(OC, IC, random_zeros):
    """fp16((q - z) * s) with numpy from formats.unpack_qm_cuda; IC = 11008 has 86 groups, so its zero and scale rows carry padding."""
    from tinychatengine_b200.formats import unpack_qm_cuda
    from tinychatengine_b200.runtime import random_w4

    w, z, s = random_w4(OC, IC, torch.device("cpu"), 17 + IC + OC, random_zeros=random_zeros)
    q, sc, zz = unpack_qm_cuda(w.numpy().view(np.uint32), z.numpy().view(np.uint32), s.numpy())
    rep = lambda a: np.repeat(a, 128, axis=1)
    want = ((q.astype(np.float32) - rep(zz).astype(np.float32)) * rep(sc).astype(np.float32)).astype(np.float16)
    got = wide_ref.expand_w4(w, z, s).numpy()
    assert got.dtype == np.float16 and got.shape == (OC, IC)
    assert np.array_equal(got.view(np.uint16), want.view(np.uint16))
    if random_zeros:
        assert len(np.unique(zz)) == 16  # the zero points are not all 8


@pytest.mark.parametrize("H,KVH", [(8, 2), (4, 4), (8, 1)])
@pytest.mark.parametrize("n,pos0", [(1, 0), (37, 0), (9, 30)])
def test_gqa_causal_attention_matches_oracle(H, KVH, n, pos0):
    """rope + gqa_causal_attention against capi.llama_attention_core (fp32, RoPE inside) on fp16-valued inputs, with and without past rows."""
    rng = np.random.default_rng(100 * H + 10 * KVH + n + pos0)
    cosb, sinb = capi.rope_tables(128, HD, 500000.0)
    q = rng.standard_normal((n, H * HD)).astype(np.float16).astype(np.float32)
    k = rng.standard_normal((n, KVH * HD)).astype(np.float16).astype(np.float32)
    v = rng.standard_normal((n, KVH * HD)).astype(np.float16).astype(np.float32)
    pk = (rng.standard_normal((KVH, pos0, HD)) * 0.7).astype(np.float16)
    pv = rng.standard_normal((KVH, pos0, HD)).astype(np.float16)
    alpha = 1.0 / np.sqrt(HD)
    want, fk, _ = capi.llama_attention_core(q, k, v, pk.astype(np.float32) if pos0 else None, pv.astype(np.float32) if pos0 else None,
                                            capi.causal_mask(n, pos0), cosb, sinb, alpha, H, KVH, HD)
    c, s = torch.from_numpy(cosb[pos0:pos0 + n]), torch.from_numpy(sinb[pos0:pos0 + n])
    qr = wide_ref.rope(torch.from_numpy(q).reshape(n, H, HD), c, s)
    kr = wide_ref.rope(torch.from_numpy(k).reshape(n, KVH, HD), c, s)
    got = wide_ref.gqa_causal_attention(qr, kr, torch.from_numpy(v).reshape(n, KVH, HD), torch.from_numpy(pk), torch.from_numpy(pv), pos0, alpha)
    assert np.abs(kr.transpose(0, 1).numpy() - fk[:, pos0:]).max() <= 1e-5 * np.abs(fk).max()
    err = wide_ref.row_rel_err(got, torch.from_numpy(want).double()).max().item()
    print(f"[wide_ref attention H={H} KVH={KVH} n={n} pos0={pos0}] worst row rel err {err:.2e}")
    assert err <= 1e-5


@pytest.mark.parametrize("H,KVH", [(8, 2), (4, 4), (8, 1)])
@pytest.mark.parametrize("n,pos0", [(1, 0), (8, 0), (5, 30)])
def test_span_rows_decode_attention_matches_oracle(H, KVH, n, pos0):
    """The span step's attention reference of tests/test_gpu_decode_wide.py: row i is decode_attention of its rotated, scaled query over
    the cached rows and the span's rows 0..i, against capi.llama_attention_core under the causal mask of n rows after pos0."""
    rng = np.random.default_rng(200 * H + 10 * KVH + n + pos0)
    cosb, sinb = capi.rope_tables(128, HD, 10000.0)
    q = rng.standard_normal((n, H * HD)).astype(np.float16).astype(np.float32)
    k = rng.standard_normal((n, KVH * HD)).astype(np.float16).astype(np.float32)
    v = rng.standard_normal((n, KVH * HD)).astype(np.float16).astype(np.float32)
    pk = (rng.standard_normal((KVH, pos0, HD)) * 0.7).astype(np.float16)
    pv = rng.standard_normal((KVH, pos0, HD)).astype(np.float16)
    alpha = 1.0 / np.sqrt(HD)
    want, _, _ = capi.llama_attention_core(q, k, v, pk.astype(np.float32) if pos0 else None, pv.astype(np.float32) if pos0 else None,
                                           capi.causal_mask(n, pos0), cosb, sinb, alpha, H, KVH, HD)
    c, s = torch.from_numpy(cosb[pos0:pos0 + n]), torch.from_numpy(sinb[pos0:pos0 + n])
    qa = wide_ref.rope(torch.from_numpy(q).reshape(n, H, HD), c, s) * alpha
    K = torch.cat([torch.from_numpy(pk).double(), wide_ref.rope(torch.from_numpy(k).reshape(n, KVH, HD), c, s).transpose(0, 1)], dim=1)
    V = torch.cat([torch.from_numpy(pv).double(), torch.from_numpy(v).double().reshape(n, KVH, HD).transpose(0, 1)], dim=1)
    got = torch.stack([wide_ref.decode_attention(qa[i], K[:, :pos0 + i + 1], V[:, :pos0 + i + 1])[0].reshape(-1) for i in range(n)])
    err = wide_ref.row_rel_err(got, torch.from_numpy(want).double()).max().item()
    print(f"[wide_ref span rows H={H} KVH={KVH} n={n} pos0={pos0}] worst row rel err {err:.2e}")
    assert err <= 1e-5


@pytest.mark.parametrize("geom", ["tiny-mha", "tiny-gqa"])
def test_prompt_pass_matches_llama_forward(geom):
    """prompt_pass (rotated q/k unrounded) against llama_forward with the fp32 product of the fp16-expanded weights as its linear and fp16 as
    its rounding: that is the prompt pass's composition, since llama_forward rounds q|k|v and SiLU*up and adds o / down unrounded.  A
    20-token prompt from position 0, then a 13-token continuation at position 20 over the first call's fp16 K/V rows; both calls again
    as one two-prompt pass, which must give the same bits as the calls alone."""
    from oracle import llama_ref
    from tinychatengine_b200.llama import GEOMETRIES, make_random_weights

    g = GEOMETRIES[geom]
    W = make_random_weights(g, torch.device("cpu"), seed=3, random_zeros=True)
    cosb, sinb = capi.rope_tables(64, g.head_dim, g.rope_theta)
    rng = np.random.default_rng(5)
    p1, p2 = [int(t) for t in rng.integers(0, g.vocab_size, 20)], [int(t) for t in rng.integers(0, g.vocab_size, 13)]

    def linear(xh, t):
        return (torch.from_numpy(np.asarray(xh, np.float32)).double() @ wide_ref.expand_w4(*t).double().T).float().numpy()

    layers = [{**{n: L[n] for n in llama_ref.LINEARS}, "input_norm": L["input_norm"].numpy(), "post_norm": L["post_norm"].numpy()} for L in W["layers"]]

    def forward(tokens, pk, pv):
        return llama_ref.llama_forward(tokens, pk, pv, embed_row=lambda t: W["embed"][t].float().numpy(), layers=layers, final_norm=W["final_norm"].numpy(),
                                       lm_head=W["lm_head"], linear=linear, cosb=cosb, sinb=sinb, H=g.num_heads, KVH=g.num_kv_heads, hd=g.head_dim,
                                       eps=g.rms_eps, rnd=lambda a: np.asarray(a).astype(np.float16))

    nl = g.num_layers
    lg1, fk1, fv1 = forward(p1, [None] * nl, [None] * nl)
    pk = [a.astype(np.float16) for a in fk1]  # the cache holds fp16
    pv = [a.astype(np.float16) for a in fv1]
    lg2, fk2, fv2 = forward(p2, [a.astype(np.float32) for a in pk], [a.astype(np.float32) for a in pv])
    past2 = [(torch.from_numpy(pk[l]), torch.from_numpy(pv[l])) for l in range(nl)]

    r1, K1, V1 = wide_ref.prompt_pass(W, g, [p1], [0], None, cosb, sinb, round_qk=False)
    r2, K2, V2 = wide_ref.prompt_pass(W, g, [p2], [20], [past2], cosb, sinb, round_qk=False)
    worst = {"logits": 0.0, "K": 0.0, "V": 0.0}
    for got, want in ((r1, lg1), (r2, lg2)):
        worst["logits"] = max(worst["logits"], wide_ref.row_rel_err(got, torch.from_numpy(want)).max().item())
    for K, V, fk, fv, p0 in ((K1, V1, fk1, fv1, 0), (K2, V2, fk2, fv2, 20)):
        for l in range(nl):
            worst["K"] = max(worst["K"], wide_ref.row_rel_err(K[l][0], torch.from_numpy(fk[l][:, p0:])).max().item())
            worst["V"] = max(worst["V"], wide_ref.row_rel_err(V[l][0], torch.from_numpy(fv[l][:, p0:])).max().item())
    print(f"[wide_ref prompt pass {geom}] worst row rel err: " + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))
    # fp32 against float64 arithmetic between the same fp16 rounding points: the RMSNorm outputs round the other way in a few elements, and
    # from there q|k|v and SiLU*up do too, by one fp16 ulp (~1e-3 of a row's max).  Measured at most 8.4e-4 (logits), 9.6e-4 (K) and 1.04e-3
    # (V, one ulp); a wrong composition (rotation, head mapping, SiLU, a missing or extra rounding of a sum) is off by far more.
    assert worst["logits"] <= 2e-3 and worst["K"] <= 2e-3 and worst["V"] <= 2e-3, worst

    rb, Kb, Vb = wide_ref.prompt_pass(W, g, [p1, p2], [0, 20], [None, past2], cosb, sinb, round_qk=False)
    assert torch.equal(rb, torch.cat([r1, r2]))
    for l in range(nl):
        assert torch.equal(Kb[l][0], K1[l][0]) and torch.equal(Kb[l][1], K2[l][0])
        assert torch.equal(Vb[l][0], V1[l][0]) and torch.equal(Vb[l][1], V2[l][0])


@pytest.mark.parametrize("geom", ["tiny-mha", "tiny-gqa"])
def test_decode_step_matches_oracle_decode_step(geom):
    """decode_step with the RMSNorm outputs rounded to fp16 and the scaled query unrounded (round_norm=True, round_q=False) against
    helpers.oracle_decode_step, the composition tests/test_gpu_llama.py checks the decode steps with: the first step (no cached rows),
    then steps after 30 random fp16 rows, each over the rows the oracle returned (fp16 K rows, fp16 V rows).  The logits, the appended K
    and V rows; and, with the kernels' rounding points (the defaults), the same step differs from the oracle's by about fp16 rounding."""
    from types import SimpleNamespace

    from helpers import oracle_decode_step
    from tinychatengine_b200.llama import GEOMETRIES, make_random_weights

    g = GEOMETRIES[geom]
    W = make_random_weights(g, torch.device("cpu"), seed=9, random_zeros=True)
    model = SimpleNamespace(geom=g, max_ctx=64, embed=W["embed"], final_norm=W["final_norm"], tensors=[W["lm_head"]],
                            layer_tensors=lambda l: W["layers"][l])
    cosb, sinb = capi.rope_tables(64, g.head_dim, g.rope_theta)
    rng = np.random.default_rng(11)
    nl, KVH = g.num_layers, g.num_kv_heads
    worst = {"logits": 0.0, "K": 0.0, "V": 0.0, "logits (kernel points)": 0.0}
    for start in (None, 30):
        if start is None:
            pk, pv, steps = [None] * nl, [None] * nl, [(17, 0)]
        else:
            pk = [(rng.standard_normal((KVH, start, HD)) * 0.7).astype(np.float16).astype(np.float32) for _ in range(nl)]
            pv = [rng.standard_normal((KVH, start, HD)).astype(np.float16).astype(np.float32) for _ in range(nl)]
            steps = [(int(t), start + i) for i, t in enumerate(rng.integers(0, g.vocab_size, 3))]
        for tok, pos in steps:
            past = [(torch.from_numpy(pk[l]), torch.from_numpy(pv[l])) for l in range(nl)] if pos else None
            want, fk, fv = oracle_decode_step(model, tok, pos, pk, pv)
            got, K, V = wide_ref.decode_step(W, g, tok, pos, past, cosb, sinb, round_norm=True, round_q=False)
            kern, _, _ = wide_ref.decode_step(W, g, tok, pos, past, cosb, sinb)
            worst["logits"] = max(worst["logits"], wide_ref.row_rel_err(got, torch.from_numpy(want)).item())
            worst["logits (kernel points)"] = max(worst["logits (kernel points)"], wide_ref.row_rel_err(kern, torch.from_numpy(want)).item())
            for l in range(nl):
                worst["K"] = max(worst["K"], wide_ref.row_rel_err(K[l], torch.from_numpy(fk[l][:, pos])).max().item())
                worst["V"] = max(worst["V"], wide_ref.row_rel_err(V[l], torch.from_numpy(fv[l][:, pos])).max().item())
            pk, pv = [a.astype(np.float16).astype(np.float32) for a in fk], [a.astype(np.float16).astype(np.float32) for a in fv]
    print(f"[wide_ref decode step {geom}] worst row rel err: " + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))
    # as in the prompt-pass pin: fp32 against float64 arithmetic between the same fp16 rounding points moves a few q|k|v and SiLU*up
    # elements by one fp16 ulp (~1e-3 of a row's max).  Measured at most 5.9e-4 (logits), 9.2e-4 (K) and 9.0e-4 (V, one ulp)
    assert worst["logits"] <= 2e-3 and worst["K"] <= 2e-3 and worst["V"] <= 2e-3, worst
    # the kernels' points drop the fp16 rounding of the RMSNorm outputs and round q * alpha: a step apart from the oracle's by that
    # rounding only (measured 1.2e-3), far inside the 1e-2 the decode tests allow against it
    assert worst["logits (kernel points)"] <= 5e-3, worst
