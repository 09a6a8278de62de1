"""A float64 restatement of the W4A16 prompt pass and decode step in torch -- TEST INFRASTRUCTURE ONLY.

The scalar C oracle (oracle/tce_oracle.c) is far too slow at the widths the benchmark times (one Llama-2-13B gate|up GEMM at M = 2048 is
about 145 G multiply-adds), so the kernels are checked there against this module, which runs on any torch device: on the CPU it is pinned
against the oracle's composition (tests/test_wide_ref.py), on the GPU it is the reference of tests/test_gpu_wide.py and
tests/test_gpu_decode_wide.py.

Every product of the projections is exact: fp16 x fp16 products are exact in float64, and a float64 sum of a few thousand of them is
the exact sum to ~1e-16 relative.  The only roundings are the fp16 ones the prompt pass and the decode step themselves make, at the same
points (``prompt_pass``, ``decode_step``).
"""
from __future__ import annotations

import math

import torch

GROUP = 128
_CHUNK_ELEMS = 1 << 26  # float64 weight elements expanded at a time (512 MB): the lm_head of Llama-3-8B alone would take 4.2 GB


def f16(x: torch.Tensor) -> torch.Tensor:
    """fp16 rounding of a float64 value, returned as float64.  Through fp32 as on the device, whose kernels round fp32 values."""
    return x.float().half().double()


def ulp_f16(a: torch.Tensor) -> torch.Tensor:
    """Spacing of the fp16 values at |a| (2^-24 in the subnormal range)."""
    e = torch.floor(torch.log2(a.abs().double().clamp_min(2.0 ** -14)))
    return torch.exp2(e - 10)


def expand_w4(w: torch.Tensor, zeros: torch.Tensor, scales: torch.Tensor, group: int = GROUP, exact: bool = False) -> torch.Tensor:
    """fp16 [OC, IC] = fp16(float(q - z) * float(s)) of QM_CUDA tensors (w int32 [OC, IC/8], zeros int32 [OC, zw], scales fp16 [OC, zw*8]):
    what w4_expand_kernel writes.  Weight 8c + i is nibble i of word c; the product is exact in fp32, so there is one rounding.
    exact=True: the float64 products (q - z) * s without that rounding -- the weights of the W4A16 GEMVs, which multiply the integer
    dot products by the scales."""
    OC, wpr = w.shape
    IC = wpr * 8
    ng = IC // group
    sh = torch.arange(8, device=w.device, dtype=torch.int64) * 4
    q = ((w.to(torch.int64).unsqueeze(-1) >> sh) & 0xF).reshape(OC, IC)
    z = ((zeros.to(torch.int64).unsqueeze(-1) >> sh) & 0xF).reshape(OC, -1)[:, :ng]
    s = scales[:, :ng].float()
    d = (q.reshape(OC, ng, group) - z.unsqueeze(-1)).float() * s.unsqueeze(-1)
    return d.double().reshape(OC, IC) if exact else d.half().reshape(OC, IC)


def w16_linear(x16: torch.Tensor, t, exact: bool = False) -> torch.Tensor:
    """float64 [M, OC] = x16 . expand_w4(t, exact=exact)^T, exact (x16: fp16 values in any float dtype).  The weights are expanded a slice
    of rows at a time, and each slice's float64 copy is freed before the next."""
    w, z, s = t
    x = x16.double()
    OC, IC = w.shape[0], w.shape[1] * 8
    step = max(1, _CHUNK_ELEMS // IC)
    out = torch.empty((x.shape[0], OC), dtype=torch.float64, device=x.device)
    for r0 in range(0, OC, step):
        r1 = min(OC, r0 + step)
        wd = expand_w4(w[r0:r1], z[r0:r1], s[r0:r1], exact=exact).double()
        out[:, r0:r1] = x @ wd.T
        del wd
    return out


def rmsnorm(x: torch.Tensor, gamma: torch.Tensor, eps: float) -> torch.Tensor:
    """x * (mean(x^2) + eps)^-1/2 * gamma over the last dimension, in float64."""
    x = x.double()
    return x * torch.rsqrt((x * x).mean(-1, keepdim=True) + eps) * gamma.double()


def rope(x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor) -> torch.Tensor:
    """Rotate-half RoPE of x [n, heads, hd] with the table rows cos / sin [n, hd] of each row's position (HF convention, both halves of a
    row hold the same angles), in float64."""
    h = x.shape[-1] // 2
    c, s = cos.double()[:, None, :], sin.double()[:, None, :]
    x = x.double()
    x0, x1 = x[..., :h], x[..., h:]
    return torch.cat([x0 * c[..., :h] - x1 * s[..., :h], x1 * c[..., h:] + x0 * s[..., h:]], dim=-1)


def gqa_causal_attention(q, k, v, past_k, past_v, pos0: int, alpha: float) -> torch.Tensor:
    """softmax(alpha q K^T + causal mask) V in float64 for n new rows at positions pos0 .. pos0 + n - 1.  q [n, H, hd] and k / v [n, KVH, hd]
    are the rotated projections; past_k / past_v [KVH, pos0, hd] are the cached rows (fp16 values; None when pos0 = 0).  Query head h reads
    KV head h // (H / KVH).  Returns float64 [n, H * hd]."""
    n, H, hd = q.shape
    KVH = k.shape[1]
    rep = H // KVH
    K, V = k.double().transpose(0, 1), v.double().transpose(0, 1)  # [KVH, n, hd]
    if pos0:
        K = torch.cat([past_k.double(), K], dim=1)
        V = torch.cat([past_v.double(), V], dim=1)
    T = pos0 + n
    hidden = torch.arange(T, device=q.device)[None, :] > (pos0 + torch.arange(n, device=q.device))[:, None]  # key j after query i
    out = torch.empty((n, H, hd), dtype=torch.float64, device=q.device)
    for g in range(KVH):
        qg = q[:, g * rep:(g + 1) * rep].double().transpose(0, 1)  # [rep, n, hd]
        S = (qg @ K[g].T) * alpha
        S.masked_fill_(hidden, -math.inf)
        out[:, g * rep:(g + 1) * rep] = (torch.softmax(S, dim=-1) @ V[g]).transpose(0, 1)
        del S
    return out.reshape(n, H * hd)


def prompt_pass(W, geom, prompts, pos0s, past, cos, sin, *, round_qk: bool = True):
    """Prompt pass of a W4A16 Llama over one or more prompts, each in its own cache: prompt i at positions pos0s[i].. after the rows
    past[i] = per-layer list of (K, V) fp16 [KVH, pos0s[i], hd] (or None).  W: the weight dict of llama.make_random_weights; cos / sin:
    the fp32 tables of oracle.capi.rope_tables.  Returns (logits fp32 [rows, vocab] of every position of every prompt, K, V) with
    K[l][i] / V[l][i] = float64 [KVH, len(prompts[i]), hd], the rows layer l appends for prompt i.

    Rounded to fp16 where the prompt pass of llama_decoder.cu (LlamaDecoder::prefill_rows) holds fp16: the RMSNorm outputs, q|k|v
    (EpiHalf), the rotated q and k and the V rows (rope_kv_append_kernel), the attention output, and SiLU(gate) * up, computed from the
    unrounded gate and up (EpiSiluMul).  The o_proj and down_proj products are added UNROUNDED into the residual (EpiAddF32), which stays
    float64 here (fp32 on the device), and the logits are the product of the fp16 final-norm output with the fp16-expanded lm_head.
    These are not the decode step's rounding points (``decode_step``).
    round_qk=False keeps the rotated q and k unrounded, as oracle.llama_ref.llama_forward does."""
    g = geom
    H, KVH, hd = g.num_heads, g.num_kv_heads, g.head_dim
    dev = W["embed"].device
    lengths = [len(p) for p in prompts]
    N = sum(lengths)
    tok = torch.tensor([int(t) for p in prompts for t in p], dtype=torch.int64, device=dev)
    pos = torch.cat([torch.arange(p0, p0 + n, device=dev) for p0, n in zip(pos0s, lengths)])
    cos_r = torch.as_tensor(cos, device=dev)[pos]
    sin_r = torch.as_tensor(sin, device=dev)[pos]
    alpha = 1.0 / math.sqrt(hd)
    x = W["embed"][tok].double()  # residual stream [N, E]
    K, V = [], []
    for l, L in enumerate(W["layers"]):
        xn = f16(rmsnorm(x, L["input_norm"], g.rms_eps))
        q = f16(w16_linear(xn, L["q"])).reshape(N, H, hd)
        k = f16(w16_linear(xn, L["k"])).reshape(N, KVH, hd)
        v = f16(w16_linear(xn, L["v"])).reshape(N, KVH, hd)
        q, k = rope(q, cos_r, sin_r), rope(k, cos_r, sin_r)
        if round_qk:
            q, k = f16(q), f16(k)
        att = torch.empty((N, H * hd), dtype=torch.float64, device=dev)
        Kl, Vl = [], []
        r = 0
        for i, (n, p0) in enumerate(zip(lengths, pos0s)):
            pk, pv = past[i][l] if past is not None and past[i] is not None else (None, None)
            att[r:r + n] = gqa_causal_attention(q[r:r + n], k[r:r + n], v[r:r + n], pk, pv, p0, alpha)
            Kl.append(k[r:r + n].transpose(0, 1).contiguous())
            Vl.append(v[r:r + n].transpose(0, 1).contiguous())
            r += n
        K.append(Kl)
        V.append(Vl)
        x = x + w16_linear(f16(att), L["o"])
        xn = f16(rmsnorm(x, L["post_norm"], g.rms_eps))
        gate, up = w16_linear(xn, L["gate"]), w16_linear(xn, L["up"])
        x = x + w16_linear(f16(gate / (1.0 + torch.exp(-gate)) * up), L["down"])
        del xn, q, k, v, att, gate, up
    xn = f16(rmsnorm(x, W["final_norm"], g.rms_eps))
    return w16_linear(xn, W["lm_head"]).float(), K, V


def decode_qkv(qkv16: torch.Tensor, H: int, KVH: int, cos_row, sin_row, alpha: float, *, round_q: bool = True):
    """The token's q|k|v words (fp16 values, [(H + 2 KVH) * hd]) -> (q * alpha after RoPE [H, hd], fp16 when round_q; the rotated key
    rounded to fp16 [KVH, hd], as the cache holds it; v [KVH, hd]), all float64.  cos_row / sin_row: the position's table rows [hd]."""
    hd = cos_row.shape[-1]
    x = qkv16.double().reshape(H + 2 * KVH, hd)
    c, s = torch.as_tensor(cos_row, device=x.device)[None], torch.as_tensor(sin_row, device=x.device)[None]
    q = rope(x[None, :H], c, s)[0] * alpha
    k = f16(rope(x[None, H:H + KVH], c, s)[0])
    return (f16(q) if round_q else q), k, x[H + KVH:]


def decode_attention(qa: torch.Tensor, K: torch.Tensor, V: torch.Tensor):
    """softmax(qa K^T) V of one token over every row of K / V [KVH, T, hd] (the cached rows and the token's own, fp16 values), qa [H, hd]
    the scaled query; query head h reads KV head h // (H / KVH).  Returns (out float64 [H, hd], p [H, T] = exp(s - max s), L [H] = sum p)."""
    H, KVH = qa.shape[0], K.shape[0]
    rep = H // KVH
    Kh = K.double().repeat_interleave(rep, dim=0)  # [H, T, hd]
    S = torch.einsum("hd,htd->ht", qa.double(), Kh)
    p = torch.exp(S - S.amax(-1, keepdim=True))
    L = p.sum(-1)
    out = torch.einsum("ht,htd->hd", p, V.double().repeat_interleave(rep, dim=0)) / L[:, None]
    return out, p, L


def silu_mul(gate: torch.Tensor, up: torch.Tensor) -> torch.Tensor:
    return gate / (1.0 + torch.exp(-gate)) * up


def decode_step(W, geom, token: int, pos: int, past, cos, sin, *, round_norm: bool = False, round_q: bool = True):
    """One decode step of a W4A16 Llama after `pos` cached rows: past[l] = (K, V) fp16 values [KVH, pos, hd] of layer l (None when
    pos = 0).  W: the weight dict of llama.make_random_weights; cos / sin: the fp32 tables of oracle.capi.rope_tables.  Returns (logits
    float64 [vocab], K, V) with K[l] / V[l] = float64 [KVH, hd], the row layer l appends.

    The projections take the exact products (q - z) * s as their weights (expand_w4(exact=True)), as the W4A16 GEMVs of both steps
    do: the prompt pass's fp16 expansion is not theirs.  Rounded where both decode steps -- the persistent kernel (decode_persistent.cu) and the kernel-per-op step (w4a16_gemv.cu +
    attention.cu) -- hold fp16, which are the same points in both:
      * q|k|v: the GEMV output is fp16 (PE_HALF_LL / EPI_STORE_HALF);
      * RoPE runs in fp32 on those words; q * alpha is rounded to fp16 for the tensor-core product, the rotated key to fp16 (the
        cache row), v is the GEMV's fp16 word;
      * the attention output is fp16;
      * SiLU(gate) * up is formed from the unrounded gate and up and rounded to fp16 (PE_SILU_LL / EPI_SILU_MUL_HALF).
    NOT rounded: the RMSNorm outputs (both GEMVs take x * gamma as 32-bit block fixed point, exact to ~2^-24 of the group maximum, and
    scale the product by 1 / rms), the o_proj and down_proj outputs (fp32, added to the fp32 residual in the order o, then down:
    PE_DELTA_LL / EPI_ADD_F32), the softmax weights (the kernels round P to fp16 against a running per-block / per-chunk maximum
    while the denominator sums the fp32 weights: below what a per-element reference can restate, so the tests bound it instead)
    and the logits (fp32).
    round_norm=True rounds the RMSNorm outputs to fp16 and round_q=False keeps the scaled query unrounded: the composition of
    helpers.oracle_decode_step (oracle/llama_ref.py::llama_forward with the W4A16 GEMV oracle), which tests/test_wide_ref.py pins."""
    g = geom
    H, KVH = g.num_heads, g.num_kv_heads
    dev = W["embed"].device
    alpha = 1.0 / math.sqrt(g.head_dim)
    cos_r, sin_r = torch.as_tensor(cos[pos], device=dev), torch.as_tensor(sin[pos], device=dev)
    norm = (lambda t: f16(t)) if round_norm else (lambda t: t)
    x = W["embed"][token].double()[None]  # residual stream [1, E]
    Ks, Vs = [], []
    for l, L in enumerate(W["layers"]):
        xn = norm(rmsnorm(x, L["input_norm"], g.rms_eps))
        qkv = f16(torch.cat([w16_linear(xn, L[n], exact=True) for n in ("q", "k", "v")], dim=1))[0]
        qa, k, v = decode_qkv(qkv, H, KVH, cos_r, sin_r, alpha, round_q=round_q)
        K, V = k[:, None], v[:, None]
        if past is not None and past[l] is not None:
            K = torch.cat([past[l][0].double(), K], dim=1)
            V = torch.cat([past[l][1].double(), V], dim=1)
        att, _, _ = decode_attention(qa, K, V)
        Ks.append(k)
        Vs.append(v)
        x = x + w16_linear(f16(att.reshape(1, -1)), L["o"], exact=True)
        xn = norm(rmsnorm(x, L["post_norm"], g.rms_eps))
        gate, up = w16_linear(xn, L["gate"], exact=True), w16_linear(xn, L["up"], exact=True)
        x = x + w16_linear(f16(silu_mul(gate, up)), L["down"], exact=True)
    xn = norm(rmsnorm(x, W["final_norm"], g.rms_eps))
    return w16_linear(xn, W["lm_head"], exact=True)[0], Ks, Vs


def row_rel_err(got: torch.Tensor, ref: torch.Tensor) -> torch.Tensor:
    """Per row: max |got - ref| / max |ref| over the last dimension (rows flattened over the leading ones)."""
    d = (got.double() - ref.double()).abs().reshape(-1, ref.shape[-1]).amax(-1)
    return d / ref.double().abs().reshape(-1, ref.shape[-1]).amax(-1).clamp_min(1e-30)
