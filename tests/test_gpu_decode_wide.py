"""The decode step at the widths the benchmark times, phase by phase, against float64 (tests/wide_ref.py, pinned on the CPU by
tests/test_wide_ref.py).

The logits of a step cannot guard its attention: with random weights the softmax is nearly flat, and a lost flash-decode split moves
the logits of a 2-layer Llama-3-8B step by less than 1e-2.  So the persistent kernel is checked here through its hand-off words
(LlamaModel.handoff_views: after a step of a 1-layer model they hold that layer's q|k|v, attention output, SiLU*up and o_proj /
down_proj outputs), each phase against float64 computed from that phase's own inputs as the kernel saw them.  Errors do not compound,
and every bound sits near fp16 rounding.  The positions follow the attention split plan (attn_split of decode_persistent.cu, restated
by attn_plan) at the device's SM count, and every attention case shows that the bound would see one lost split.  The kernel-per-op
step (the batched and span steps: the stand-alone GEMV and attention kernels) is checked the same way through its step buffers
(LlamaModel.debug_buffer 0..3), at positions that cover the stand-alone attention's split plan and at row counts that cover the GEMV's
K-slice plan, both restated here.  Then whole 2-layer steps on both decode paths, across chunk and split boundaries, each against
wide_ref.decode_step on the cache rows the kernel holds.  Every case prints its worst ratio to its bound."""
import math
import os

import pytest
import torch

import wide_ref
from wide_ref import f16, row_rel_err, ulp_f16

pytestmark = pytest.mark.gpu

HD = 128
CHUNK = 64  # cached rows per attention ring stage (pk::kKvChunk)
DEV = torch.device("cuda", 0)

# fp32 accumulation of the persistent GEMVs, per unit of sum |x_k w_k| (fixed-point activations, exact integer MMA per 128-group, fp32 sum
# of the group partials, 1/rms applied last).  Worst |d| / bound on an H100 SXM (700 W), 1-layer Llama-3-8B and Llama-2-7B at every
# position: o_proj 0.052, down_proj 0.026, logits 0.050 (fp32 outputs: the accumulation alone); q|k|v 0.98 and SiLU*up 0.96, where an
# fp16 output next to a rounding boundary takes up to its whole half ulp (the bound allows half an ulp plus the accumulation, of which
# the fp32 outputs show that about 5 % is used)
C_GEMV = 2.0 ** -21
# attention: the kernels round the softmax weights to fp16 (relative 2^-11, 2^-25 absolute below fp16's normal range) against a running
# maximum; fp32 scores, exponentials, rescaling and split merge add a few 2^-22 per weight.  Worst |d| / bound 0.52 (pos 63), 0.21 at 4095
P_ROUND, P_SUBNORMAL, ATTN_FP32 = 2.0 ** -11, 2.0 ** -25, 2.0 ** -19
# a lost split must move some output element by at least this many bounds: measured >= 125 at every position of both geometries
POWER_MIN = 4.0


# ------------------------------------------------------------------------------------------------ the attention split plan

def attn_plan(ncta: int, KVH: int, pos: int):
    """attn_split of decode_persistent.cu: the visible rows [0, pos] in 64-row chunks; every KV head gets NS = #CTAs / KVH CTAs, each
    taking cps consecutive chunks (the fewest that cover the context, and at most 32 splits).  Returns (NS, cps, chunk ranges of the
    splits that take part)."""
    nch = (pos + 1 + CHUNK - 1) // CHUNK
    NS = max(1, ncta // KVH)
    cps = (nch + NS - 1) // NS
    if cps * 32 < nch:
        cps = (nch + 31) // 32
    nsplit = (nch + cps - 1) // cps
    return NS, cps, [(s * cps, min(nch, s * cps + cps)) for s in range(nsplit)]


def split_classes(ncta: int, KVH: int, pos: int, max_ctx: int) -> set:
    NS, cps, splits = attn_plan(ncta, KVH, pos)
    row = pos % CHUNK
    c = set()
    if len(splits) == 1:
        c.add("one split")
    if len(splits) == 2:
        c.add("two splits")
    if cps == 1 and len(splits) == NS > 1:
        c.add("one chunk per split, every split used")
    if pos and attn_plan(ncta, KVH, pos - 1)[1] != cps:
        c.add("chunks per split change")
    if splits[-1][1] - splits[-1][0] < cps:
        c.add("last split shorter")
    if row in (0, 15, 16, 63):
        c.add(f"token at row {row} of its chunk")
    if pos >= CHUNK and row // 16 < 3:
        c.add("warp without a visible block in the token's chunk")
    if pos == max_ctx - 1:
        c.add("last position")
    return c


REQUIRED_CLASSES = {"one split", "two splits", "one chunk per split, every split used", "chunks per split change", "last split shorter",
                    "token at row 0 of its chunk", "token at row 15 of its chunk", "token at row 16 of its chunk",
                    "token at row 63 of its chunk", "warp without a visible block in the token's chunk", "last position"}


def pick_positions(ncta: int, KVH: int, max_ctx: int) -> list:
    """Positions that meet every class of REQUIRED_CLASSES at this device's split plan."""
    NS = min(max(1, ncta // KVH), 32)
    nch_max = (max_ctx + CHUNK - 1) // CHUNK
    pos = {0, CHUNK - 1, CHUNK, CHUNK * NS - 1, CHUNK * NS, max_ctx - 1}
    for nch in range(NS + 1, nch_max + 1):  # the first context whose last split is shorter than the others
        p = CHUNK * (nch - 1)
        if "last split shorter" in split_classes(ncta, KVH, p, max_ctx):
            pos.add(p)
            break
    mid = nch_max // 3
    pos |= {CHUNK * mid + 15, CHUNK * mid + 16, CHUNK * (nch_max // 2) + 5}
    return sorted(p for p in pos if 0 <= p < max_ctx)


# ------------------------------------------------------------------------------------------------ models and their float64 weights

class Wide:
    """A 1-layer model at a benchmarked geometry: its weights expanded to float64 once, and one LlamaModel per decode path."""

    def __init__(self, ctx, widths: str, max_ctx: int):
        import dataclasses

        from tinychatengine_b200.llama import GEOMETRIES, make_random_weights

        self.ctx = ctx
        self.g = dataclasses.replace(GEOMETRIES[widths], name=f"{widths}-1l", num_layers=1)
        self.max_ctx = max_ctx
        self.W = make_random_weights(self.g, DEV, seed=31, random_zeros=True)
        L = self.W["layers"][0]
        self.w64 = {n: wide_ref.expand_w4(*L[n], exact=True) for n in ("q", "k", "v", "o", "gate", "up", "down")}
        self.w64["qkv"] = torch.cat([self.w64.pop(n) for n in ("q", "k", "v")])
        self.w64["lm_head"] = wide_ref.expand_w4(*self.W["lm_head"], exact=True)
        from oracle import capi

        self.cos, self.sin = (torch.from_numpy(t).to(DEV) for t in capi.rope_tables(max_ctx, HD, self.g.rope_theta))
        self.models = {}

    def _build(self, key, env, weights=None):
        if key not in self.models:
            from tinychatengine_b200.llama import LlamaModel

            saved = {k: os.environ.get(k) for k in env}
            for k, v in env.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
            try:
                self.models[key] = LlamaModel(self.ctx, self.g, max_ctx=self.max_ctx, weights=weights or self.W)
            finally:
                for k, v in saved.items():
                    if v is None:
                        os.environ.pop(k, None)
                    else:
                        os.environ[k] = v
        return self.models[key]

    def model(self):
        """The persistent kernel."""
        m = self._build("persistent", {"TCE_PERSISTENT": "1"})
        assert m.kernels_per_step == 1
        return m

    def step_model(self, deterministic: bool, zero_down: bool = False):
        """The kernel-per-op step (TCE_PERSISTENT=0) with every KV-cache slot, its o_proj / down_proj partials added by RED.ADD or, with
        deterministic (TCE_DETERMINISTIC=1, read when the model is built), by the ordered fix-up.  zero_down: the same weights with
        down_proj's scales set to zero, so that the residual after a step is exactly what o_proj left in it."""
        key = ("step", deterministic, zero_down)
        weights = None
        if zero_down and key not in self.models:
            L = dict(self.W["layers"][0])
            L["down"] = (L["down"][0], L["down"][1], torch.zeros_like(L["down"][2]))
            weights = {**self.W, "layers": [L]}
        m = self._build(key, {"TCE_PERSISTENT": "0", "TCE_DETERMINISTIC": "1" if deterministic else None}, weights)
        m.reserve_slots(m.MAX_BATCH)
        return m

    def close(self):
        for m in self.models.values():
            m.close()


@pytest.fixture(scope="module")
def ctx():
    from tinychatengine_b200.runtime import Context

    c = Context(0)
    yield c
    c.close()


_WIDE = {}


@pytest.fixture(scope="module")
def wide(ctx):
    def get(widths, max_ctx):
        key = (widths, max_ctx)
        if key not in _WIDE:
            for w in list(_WIDE.values()):  # one geometry's float64 weights at a time
                w.close()
            _WIDE.clear()
            torch.cuda.empty_cache()
            _WIDE[key] = Wide(ctx, widths, max_ctx)
        return _WIDE[key]

    yield get
    for w in _WIDE.values():
        w.close()
    _WIDE.clear()


def _linear(x, w):
    """(x . w^T, |x| . |w|^T) in float64, x [E] or [n, E]."""
    x = x.double()
    return x @ w.T, x.abs() @ w.abs().T


def _ratio(got, ref, bound):
    """Elementwise |got - ref| / bound, with inf where got is not finite."""
    return ((got.double() - ref).abs() / bound).nan_to_num(nan=math.inf, posinf=math.inf)


def _first_bad(ratio):
    i = int((ratio > 1.0).flatten().nonzero()[0].item())
    return i, ratio.flatten()[i].item()


def _fill_cache(model, pos, seed, k_std=1.0, v_std=1.0, slot=0):
    """Random fp16 rows below pos and NaN from pos on, in every head of every layer of a slot: a row the step should have written and did
    not, or a row past the token that reaches the output, shows up as NaN."""
    gen = torch.Generator(device=DEV)
    gen.manual_seed(seed)
    for l in range(model.geom.num_layers):
        for which, std in ((0, k_std), (1, v_std)):
            c = model.kv_cache(l, which, slot)
            c.fill_(float("nan"))
            if pos:
                c[:, :pos] = (torch.randn((c.shape[0], pos, HD), device=DEV, generator=gen) * std).to(torch.float16)


def _bits(t):
    return t.view(torch.int16).clone()


# ------------------------------------------------------------------------------------------------ a./b./c./e. every phase of one step

def _units(splits, T: int):
    """The key ranges whose loss the attention check must see, for a row that sees keys 0 .. T - 1 of a plan cut into `splits` (key ranges):
    the splits when there are several, else the 16-row blocks of the one split.  Returns (units, kind)."""
    if len(splits) > 1:
        return [(r0, min(T, r1)) for r0, r1 in splits], "split"
    return [(r, min(T, r + 16)) for r in range(0, T, 16)], "16-row block"


def _attention_check(tag, w, qkv16, positions, kc, vc, got, units, kind, plan, causal=False):
    """The attention words of every row and head against decode_attention on the kernel's own q|k|v words and the cache rows: row i
    (query position positions[i]) sees keys 0 .. positions[i] of kc / vc [KVH, max_ctx, HD] as they are after the step (the appended rows
    are checked elsewhere: K within its bound, V bit for bit).  qkv16 [n, (H + 2 KVH) HD] and got [n, H HD] are the kernel's words.  Then
    the power check: losing any one of `units` (key ranges of the plan) moves some (row, KV head) by `power` bounds; with causal, adding
    row i + 1's key to row i moves some head of row i by `causal power` bounds.  Returns (worst, power, causal power, top) with top[i] =
    (key index, weight share) of the largest softmax weight of every head of row i."""
    g = w.g
    H, KVH = g.num_heads, g.num_kv_heads
    rep = H // KVH
    alpha = 1.0 / math.sqrt(HD)
    T_all = max(positions) + 1 + (1 if causal else 0)
    K = kc[:, :T_all].double()
    V = vc[:, :T_all].double()
    Kh = K.repeat_interleave(rep, dim=0)
    Vh = V.repeat_interleave(rep, dim=0)
    worst, effs, cpow, top = 0.0, {}, math.inf, []
    for i, pos in enumerate(positions):
        T = pos + 1
        q64, _, _ = wide_ref.decode_qkv(qkv16[i], H, KVH, w.cos[pos], w.sin[pos], alpha, round_q=False)
        qa = f16(q64)
        ref, p, L = wide_ref.decode_attention(qa, K[:, :T], V[:, :T])
        y = got[i].double().reshape(H, HD)
        A = torch.einsum("ht,htd->hd", p, Vh[:, :T].abs()) / L[:, None]  # sum_j p_j |v_j| / L
        B = Vh[:, :T].abs().sum(1) / L[:, None]                           # sum_j |v_j| / L
        # score error: the fp32 sum of the MMA, and the elements of q * alpha that lie so close to a rounding boundary of fp16 that the fp32
        # RoPE (error < 2^-21 alpha (|x_d| + |x_d'|)) may round them to the other neighbour (one ulp)
        xq = qkv16[i].double().reshape(-1, HD)[:H].abs()
        xq = xq + torch.cat([xq[:, HD // 2:], xq[:, :HD // 2]], dim=-1)
        near = ((q64 - qa).abs() - 0.5 * ulp_f16(qa)).abs() <= 2.0 ** -21 * alpha * xq
        ds = (torch.einsum("hd,htd->ht", ulp_f16(qa) * near, Kh[:, :T].abs())
              + 2.0 ** -22 * torch.einsum("hd,htd->ht", qa.abs(), Kh[:, :T].abs())).amax(-1)
        bound = 0.5 * ulp_f16(torch.maximum(ref.abs(), y.abs())) + (P_ROUND + 2 * ds[:, None] + ATTN_FP32) * A + P_SUBNORMAL * B
        ratio = _ratio(y, ref, bound)
        worst = max(worst, ratio.max().item())
        share, idx = (p / L[:, None]).max(-1)
        top.append((idx, share))
        N = ref * L[:, None]
        without = {}
        for u, (r0, r1) in enumerate(units):
            r1 = min(r1, T)
            Lu = p[:, r0:r1].sum(-1) if r0 < r1 else None
            if Lu is None or r1 - r0 == T:  # the row sees no key of this unit, or none but its keys
                continue
            Nu = torch.einsum("ht,htd->hd", p[:, r0:r1], Vh[:, r0:r1])
            without[u] = (N - Nu) / (L - Lu)[:, None]
            e = ((without[u] - ref).abs() / bound).reshape(KVH, rep * HD).amax().item()
            effs[u] = max(effs.get(u, 0.0), e)
        if causal and i + 1 < len(positions):
            nxt, _, _ = wide_ref.decode_attention(qa, K[:, :T + 1], V[:, :T + 1])
            cpow = min(cpow, ((nxt - ref).abs() / bound).amax().item())
        if ratio.max().item() > 1.0:
            j, r = _first_bad(ratio)
            h, d = divmod(j, HD)
            if not torch.isfinite(y[h]).all():
                pytest.fail(f"{tag}: row {i} (pos {pos}) attention head {h} (KV head {h // rep}) dim {d} is {y[h, d].item()}: a NaN row of "
                            f"the cache (the token's own before it is appended, or a row past it) reached the P.V product")
            if without:
                near_u = min(without, key=lambda u: (y[h] - without[u][h]).abs().max().item())
                r0, r1 = units[near_u]
                hint = (f"; closest to the reference without {kind} {near_u} (rows {r0}..{r1 - 1}): max |y - that| "
                        f"{(y[h] - without[near_u][h]).abs().max().item():.3g}")
            else:
                hint = ""
            pytest.fail(f"{tag}: row {i} (pos {pos}) attention head {h} (KV head {h // rep}) dim {d}: y {y[h, d].item()} ref {ref[h, d].item()} "
                        f"ratio {r:.3g}{hint}")
    # power: whichever unit is lost, the (row, KV head) where that loss shows most moves by `power` bounds or more (a unit of a single key
    # whose weight is negligible in some head would not move that head's output at all)
    power = min(effs.values()) if len(effs) > 1 else math.inf
    msg = (f"[{tag} attention] worst |y - ref| / bound {worst:.3f} over {len(positions)} x {H} heads; plan {plan}; "
           + (f"losing any one {kind} moves some head by >= {power:.1f} bounds" if len(effs) > 1 else "no partial to lose"))
    if causal:
        msg += f"; the next row's key moves some head by >= {cpow:.1f} bounds"
    print(msg)
    if len(effs) > 1:
        assert power >= POWER_MIN, f"{tag}: the attention bound cannot see a lost {kind} ({power:.2f} bounds)"
    return worst, power, cpow, top


def _phase_case(w, pos, tok=4321, seed=0):
    g = w.g
    H, KVH = g.num_heads, g.num_kv_heads
    model = w.model()
    tag = f"{g.name} max_ctx={w.max_ctx} pos={pos}"
    _fill_cache(model, pos, seed=pos + 1 + seed)
    kc, vc = model.kv_cache(0, 0), model.kv_cache(0, 1)
    before = (_bits(kc), _bits(vc))
    tags_before = {n: t.clone() for n, (_, t) in model.handoff_views().items()}
    lg = torch.empty(g.vocab_size, dtype=torch.float32).pin_memory()
    nxt = model.decode_host(tok, pos, lg)
    torch.cuda.synchronize()
    views = model.handoff_views()
    L0 = w.W["layers"][0]
    worst = {}

    # tags: one per vector and step, every word of the step carries it, none is left over from the previous step
    nphase = 6
    t0 = views["qkv"][1][0].item()
    want_tag = {"qkv": t0, "attn": t0 + 2, "delta0": t0 + 4, "act": t0 + 6, "delta1": t0 + 8}
    for n, t in want_tag.items():
        assert (views[n][1] == t).all(), f"{tag}: {n} words carry tags {views[n][1].unique().tolist()[:6]}, want {t}"
        assert (views[n][1] != tags_before[n]).all(), f"{tag}: a {n} word kept the previous step's tag"
    NS, cps, splits = attn_plan(w.ctx.num_sms, KVH, pos)
    if len(splits) > 1:
        pt = views["part"][1][:, :len(splits)]
        assert (pt == t0 + 3).all() and (pt != tags_before["part"][:, :len(splits)]).all(), f"{tag}: stale split partial"
    if (tags_before["qkv"] != 0).any():
        assert t0 == tags_before["qkv"][0].item() + 2 * nphase + 2

    # q|k|v = RMSNorm(embedding row) -> GEMV, fp16
    x = w.W["embed"][tok].double()
    xn = wide_ref.rmsnorm(x, L0["input_norm"], g.rms_eps)
    ref, mag = _linear(xn, w.w64["qkv"])
    qkv = views["qkv"][0]
    r = _ratio(qkv, ref, 0.5 * ulp_f16(torch.maximum(ref.abs(), qkv.double().abs())) + C_GEMV * mag)
    worst["qkv"] = r.max().item()
    if worst["qkv"] > 1:
        i, rv = _first_bad(r)
        pytest.fail(f"{tag}: q|k|v element {i} (head row {i // HD}): {qkv[i].item()} ref {ref[i].item()} ratio {rv:.3g}")

    # the appended rows: K = RoPE of the kernel's k words rounded to fp16, V = its v words bit for bit; nothing else written
    _, kref, vw = wide_ref.decode_qkv(qkv, H, KVH, w.cos[pos], w.sin[pos], 1.0)
    kin = qkv.double().reshape(H + 2 * KVH, HD)[H:H + KVH].abs()
    pair_mag = kin[:, :HD // 2] + kin[:, HD // 2:]
    kb = 2 * ulp_f16(kref) + 2.0 ** -20 * torch.cat([pair_mag, pair_mag], dim=-1)
    worst["K row (2 ulps + rotation)"] = _ratio(kc[:, pos], kref, kb).max().item()
    assert worst["K row (2 ulps + rotation)"] <= 1.0, tag
    assert torch.equal(vc[:, pos].double(), vw), f"{tag}: the appended V row is not the step's v words"
    after = (_bits(kc), _bits(vc))
    for b, a_, name in ((before[0], after[0], "K"), (before[1], after[1], "V")):
        changed = (b != a_).any(-1)
        changed[:, pos] = False
        assert not changed.any(), f"{tag}: {name} rows other than {pos} changed: {changed.nonzero()[:4].tolist()}"

    # attention: per head, on the kernel's own q / k / v words and the cache
    units, kind = _units([(c0 * CHUNK, c1 * CHUNK) for c0, c1 in splits], pos + 1)
    worst["attention"] = _attention_check(tag, w, qkv[None], [pos], kc, vc, views["attn"][0][None], units, kind,
                                          f"NS={NS} cps={cps} nsplit={len(splits)}")[0]

    # o_proj: the kernel's attention words -> fp32
    attn = views["attn"][0]
    ref, mag = _linear(attn, w.w64["o"])
    d0 = views["delta0"][0]
    r = _ratio(d0, ref, C_GEMV * mag)
    worst["o_proj"] = r.max().item()
    assert worst["o_proj"] <= 1.0, (tag, "o_proj", _first_bad(r))

    # SiLU(gate) * up from RMSNorm(embedding + o_proj), fp16
    x1 = x + d0.double()
    xn = wide_ref.rmsnorm(x1, L0["post_norm"], g.rms_eps)
    gate, mg = _linear(xn, w.w64["gate"])
    up, mu = _linear(xn, w.w64["up"])
    ref = wide_ref.silu_mul(gate, up)
    act = views["act"][0]
    silu = gate / (1.0 + torch.exp(-gate))
    bound = 0.5 * ulp_f16(torch.maximum(ref.abs(), act.double().abs())) + C_GEMV * (1.1 * up.abs() * mg + silu.abs() * mu) + 2.0 ** -21 * ref.abs()
    r = _ratio(act, ref, bound)
    worst["SiLU*up"] = r.max().item()
    assert worst["SiLU*up"] <= 1.0, (tag, "SiLU*up", _first_bad(r))

    # down_proj: the kernel's SiLU*up words -> fp32
    ref, mag = _linear(act, w.w64["down"])
    d1 = views["delta1"][0]
    r = _ratio(d1, ref, C_GEMV * mag)
    worst["down_proj"] = r.max().item()
    assert worst["down_proj"] <= 1.0, (tag, "down_proj", _first_bad(r))

    # logits: final RMSNorm of embedding + o_proj + down_proj -> lm_head, fp32; the greedy token is the first arg-max
    xn = wide_ref.rmsnorm(x1 + d1.double(), w.W["final_norm"], g.rms_eps)
    ref, mag = _linear(xn, w.w64["lm_head"])
    got = lg.to(DEV)
    r = _ratio(got, ref, C_GEMV * mag)
    worst["logits"] = r.max().item()
    assert worst["logits"] <= 1.0, (tag, "logits", _first_bad(r))
    assert nxt == int(torch.argmax(got).item())
    print(f"[{tag}] worst |d| / bound: " + ", ".join(f"{k} {v:.3f}" for k, v in worst.items()))
    return worst


def _phase_cases():
    """(widths, max_ctx, position index or an explicit position): every position of the plan; max_ctx 4000 (not a multiple of 64) at its
    last rows.  "pair" in an id: the kernel runs on clusters of two CTAs."""
    out = [pytest.param("llama3-8b", 4096, i, id=f"llama3-8b-pair-{i}") for i in range(10)]
    out += [pytest.param("llama2-7b", 4096, i, id=f"llama2-7b-pair-{i}") for i in range(10)]
    out += [pytest.param("llama3-8b", 4000, p, id=f"llama3-8b-ctx4000-last{-p}") for p in (-1, -32)]
    return out


@pytest.mark.parametrize("widths,max_ctx,which", _phase_cases())
def test_persistent_step_phases(wide, widths, max_ctx, which):
    """One step of a 1-layer model at Llama-3-8B (GQA 32:8, full vocabulary) or Llama-2-7B (MHA) widths on a cache that is random below
    the token and NaN from it on: every phase against float64 from its own inputs (see the module docstring).  `which` indexes the
    positions of pick_positions at this device's SM count, or (negative) counts back from max_ctx."""
    w = wide(widths, max_ctx)
    if which < 0:
        pos = max_ctx + which
    else:
        positions = pick_positions(w.ctx.num_sms, w.g.num_kv_heads, max_ctx)
        if which >= len(positions):
            pytest.skip(f"{len(positions)} positions at this SM count")
        pos = positions[which]
    _phase_case(w, pos)


@pytest.mark.parametrize("widths", ["llama3-8b", "llama2-7b"])
def test_split_classes_covered(ctx, widths):
    """The positions of test_persistent_step_phases meet every split class at this device's SM count."""
    from tinychatengine_b200.llama import GEOMETRIES

    KVH = GEOMETRIES[widths].num_kv_heads
    positions = pick_positions(ctx.num_sms, KVH, 4096)
    assert len(positions) <= 10, positions  # the test's parameter list
    seen = {}
    for p in positions:
        for c in split_classes(ctx.num_sms, KVH, p, 4096):
            seen.setdefault(c, []).append(p)
    print(f"[split classes {widths}, {ctx.num_sms} SMs, NS={attn_plan(ctx.num_sms, KVH, 0)[0]}] " + "; ".join(f"{c}: {seen[c]}" for c in sorted(seen)))
    assert REQUIRED_CLASSES <= set(seen), REQUIRED_CLASSES - set(seen)


# ------------------------------------------------------------------------------------------------ the kernel-per-op step, phase by phase

# The batched step (LlamaModel.decode_batch_host) and the span step (decode_span) run the stand-alone W4A16 GEMV (w4a16_gemv.cu) at
# M = rows and the stand-alone attention (attention.cu); after a step of a 1-layer model the step's buffers (LlamaModel.debug_buffer 0..3)
# hold every row's final residual, q|k|v, attention output and SiLU*up.  o_proj is never visible on its own (the residual holds
# x + o + d), so a second model on the same weights with down_proj's scales set to zero gives x + o, and SiLU*up is checked there from it.
#
# What the stand-alone kernels add to the persistent kernel's error terms (C_GEMV, P_ROUND, P_SUBNORMAL, ATTN_FP32 carry over: the same
# fixed-point activations, exact integer MMA per group, fp32 group sums and fp16 rounding points):
#   * the RMSNorm prologue scales x by an fp32 rsqrtf (2 ulps) BEFORE quantising, where the persistent kernel applies 1 / rms last: a
#     common relative error of the whole output, NORM_F32 * |y|;
#   * the residual: the fp32 adds into it, each rounding to half an ulp of the running value: two in order (o, then d) with the ordered
#     fix-up; with RED.ADD one per partial tile (<= 3 stream-K pieces of an unsliced tile, one per K-slice of a sliced one), together at
#     most RESID_ADDS of them;
#   * the K-slice fix-up sums the slices' fp32 partials, which is inside the fp32 accumulation of C_GEMV;
#   * q * alpha is rounded to fp16 before the MMA, as in the persistent kernel (the `near` term of _attention_check).
# Worst |d| / bound on an H100 SXM (700 W) over every case of test_kernel_per_op_step_phases, RED.ADD / ordered fix-up: q|k|v 0.986 /
# 0.986, K row 0.500 / 0.500, attention 0.829 / 0.829, o_proj 0.027 / 0.055, SiLU*up 0.961 / 0.961, residual 0.014 / 0.026, logits
# 0.045 / 0.052.  A lost split or 16-row block moves some head by >= 60 bounds, and so does the next span row's key.
NORM_F32 = 2.0 ** -21
RESID_ADDS = {True: 2, False: 12}  # deterministic: o, then d; RED.ADD: o in <= 3 pieces (2 slices at E = 5120), d in <= 7 slices + 2
def chunk_rows(chunk: int) -> int:
    """chunk_rows of attention.cu: cached rows per CTA, attn_chunk <= 0 selecting the default."""
    return chunk if chunk > 0 else 128


ATTN_CHUNK = chunk_rows(int(os.environ.get("TCE_ATTN_CHUNK", "256")))  # the context's attn_chunk (capi.cu reads the same variable and default)
GEMV_CW_OPTION = int(os.environ.get("TCE_GEMV_CONSUMER_WARPS", "8"))  # the context's gemv_consumer_warps (8, 16 or 0 = per shape)
SLOT_ORDER = (5, 0, 7, 2, 6, 1, 3, 4)  # sequence b of a batched step runs in slot SLOT_ORDER[b]


def smem_optin() -> int:
    return torch.cuda.get_device_properties(0).shared_memory_per_block_optin


# ---- the stand-alone attention's plan (attention.cu)

def attn_smem_bytes(nc: int, chunk: int) -> int:
    """smem_bytes of attention.cu: one CTA serving nc query columns over `chunk` cached rows."""
    r16 = (chunk + 15) & ~15
    pitch = HD + 8
    b = 2 * r16 * pitch * 2 + nc * pitch * 2 + nc * max(r16, HD + 8) * 4 + nc * r16 * 2 + 2 * nc * 4
    return (b + 15) & ~15


def attn_span_chunk(H: int, KVH: int, chunk: int, optin: int) -> int:
    """attn_span_chunk of attention.cu: the largest multiple of 16 rows <= chunk whose CTA fits at 8 rows (+ the 16-byte flag word)."""
    nrep = H // KVH
    c = chunk_rows(chunk) & ~15
    while c >= 16:
        if attn_smem_bytes(8 * nrep, c) + 16 <= optin:
            return c
        c -= 16
    return 0


def standalone_splits(chunk: int, pos0: int, n: int = 1):
    """The splits of one sequence of n rows at positions pos0..: one CTA per `chunk` rows of the pos0 + n keys the last row sees; one
    split writes directly, several merge their records in split order."""
    T = pos0 + n
    return [(s * chunk, min(T, s * chunk + chunk)) for s in range(-(-T // chunk))]


def standalone_classes(chunk: int, pos: int, max_ctx: int) -> set:
    T = pos + 1
    ns = len(standalone_splits(chunk, pos))
    row = pos % chunk
    c = set()
    if pos == 0:
        c.add("the token's own key only")
    if T == chunk:
        c.add("one full split")
    if ns > 1 and row == 0:
        c.add("a split holding only the token's row")
    if ns > 1 and row == 1:
        c.add("a split of the token and one cached row")
    if row in (15, 16):
        c.add(f"token at row {row} of its split")
    if ns > 1 and T % 16:
        c.add("last 16-row tile partial")
    if ns == 16:
        c.add("16 splits")
    if pos == max_ctx - 1:
        c.add("last position")
    return c


STANDALONE_REQUIRED = {"the token's own key only", "one full split", "a split holding only the token's row", "a split of the token and one cached row",
                       "token at row 15 of its split", "token at row 16 of its split", "last 16-row tile partial", "16 splits", "last position",
                       "sequences with different split counts in one launch", "peaked softmax, maximum in a later split"}

# batched step: positions of sequences 0..B-1 (sequence b in slot SLOT_ORDER[b]); PEAK: (sequence, cached row) given a key whose score is
# PEAK_SCORE, about 10 above the others: the largest weight of most heads of its row, with about 0.4 of the row's weight
BATCH_CASES = {1: [3000], 2: [256, 4095], 5: [15, 16, 257, 1999, 3840], 8: [0, 255, 256, 271, 272, 600, 2047, 4095]}
PEAK = {2: (1, 3900)}
PEAK_SCORE = 10.0
# span step: (pos0, n) on slot 3, every n from 1 to 8.  Straddling a split boundary (253, 8): rows 0-2 see no key of the second split
# (an m = -inf record)
SPAN_CASES = [(0, 8), (130, 2), (253, 8), (256, 3), (509, 4), (700, 1), (1020, 6), (1500, 5), (2040, 7), (4088, 8)]
SPAN_SLOT = 3


def span_classes(chunk: int, max_ctx: int) -> dict:
    seen = {}
    for p0, n in SPAN_CASES:
        first, last = p0 // chunk, (p0 + n - 1) // chunk
        c = {f"{n} rows"}
        if p0 == 0:
            c.add("row 0 sees only itself")
        if first != last:
            c.add("rows on both sides of a split boundary")
        if p0 and p0 % chunk == 0:
            c.add("span starting on a split boundary")
        if len(standalone_splits(chunk, p0, n)) >= 4:
            c.add("long context (4 splits or more)")
        if p0 + n == max_ctx:
            c.add("span ending at max_ctx")
        for x in c:
            seen.setdefault(x, []).append((p0, n))
    return seen


SPAN_REQUIRED = {f"{n} rows" for n in range(1, 9)} | {"row 0 sees only itself", "rows on both sides of a split boundary",
                                                        "span starting on a split boundary", "long context (4 splits or more)",
                                                        "span ending at max_ctx"}


def batch_classes(chunk: int, max_ctx: int) -> dict:
    seen = {}
    for B, positions in BATCH_CASES.items():
        for p in positions:
            for c in standalone_classes(chunk, p, max_ctx):
                seen.setdefault(c, []).append((B, p))
        if len({len(standalone_splits(chunk, p)) for p in positions}) > 1:
            seen.setdefault("sequences with different split counts in one launch", []).append(B)
    for B, (b, r) in PEAK.items():
        if r >= chunk and r < BATCH_CASES[B][b]:
            seen.setdefault("peaked softmax, maximum in a later split", []).append((B, BATCH_CASES[B][b], r))
    return seen


# ---- the multi-column GEMV's K-slice plan (w4a16_gemv.cu)

def gemv_layout_bytes(IC: int, nst: int, xw: int, ncols: int = 8, cw: int = 8) -> int:
    """Layout<NCOLS, CW>::bytes of w4a16_gemv_impl.cuh: ring, scales / zeros slots, activation planes of xw elements per column, group
    steps and sums, reduction buffers, RMSNorm partials, barriers."""
    NG = IC // 128
    pitch = xw * 4 + (64 if ncols > 1 else 0)
    meta = 320 * ((NG + 7) // 8)
    off_gx = nst * 16384 + (nst + 1) * meta + ncols * pitch
    off_rms = off_gx + 3 * ncols * NG * 4 + 3 * cw * 16 * ncols * 4
    off_bar = (off_rms + ncols * cw * 4 + 15) & ~15
    return off_bar + (2 * nst + 6) * 8 + 16


def gemv_consumer_warps(IC: int, M: int, option: int = GEMV_CW_OPTION) -> int:
    return option if option in (8, 16) else (16 if IC > 8192 and M == 1 else 8)


def gemv_slices(IC: int, M: int, optin: int, option: int = GEMV_CW_OPTION) -> list:
    """The K-slices (in 128-groups) the activation rows are staged in: the whole row at M = 1 (and wherever it fits next to a 4-stage
    ring), else the widest multiple of 16 groups that does (pick_slice / slice_of)."""
    NG = IC // 128
    if M == 1:
        return [NG]
    cw = gemv_consumer_warps(IC, M, option)
    fits = lambda xw: gemv_layout_bytes(IC, 4, xw, 8, cw) <= optin
    if fits(IC):
        return [NG]
    sl = next((s for s in range((NG - 1) // 16 * 16, 15, -16) if fits(s * 128)), 16)
    return [sl] * (NG // sl) + ([NG % sl] if NG % sl else [])


def step_gemvs(g):
    """(name, IC, RMSNorm prologue, epilogue) of every GEMV of a batched step."""
    return [("q|k|v", g.embed_dim, True, "fp16"), ("o_proj", g.num_heads * HD, False, "residual add"), ("gate|up", g.embed_dim, True, "SiLU pair"),
            ("down_proj", g.hidden_dim, False, "residual add"), ("lm_head", g.embed_dim, True, "fp32")]


KPO_WIDTHS = ["llama3-8b", "llama2-7b", "llama2-13b"]


def _kpo_cases():
    """(widths, deterministic, kind, case, consumer-warp option or None for the context's): every batch width and span case in both
    residual modes, and batch 1 with per-shape consumer warps (option 0: 16 at M = 1 on rows longer than 8192)."""
    out = []
    for wd in KPO_WIDTHS:
        for det in (False, True):
            mode = "ordered" if det else "redadd"
            out += [pytest.param(wd, det, "batch", B, None, id=f"{wd}-{mode}-batch{B}") for B in BATCH_CASES]
            out += [pytest.param(wd, det, "span", i, None, id=f"{wd}-{mode}-span{p0}+{n}") for i, (p0, n) in enumerate(SPAN_CASES)]
        out.append(pytest.param(wd, False, "batch", 1, 0, id=f"{wd}-redadd-batch1-cw0"))
    return out


def gemv_classes(optin: int) -> dict:
    """The K-slice classes the cases of test_kernel_per_op_step_phases reach, each with where."""
    from tinychatengine_b200.llama import GEOMETRIES

    seen = {}
    for p in _kpo_cases():
        wd, det, kind, case, cw_opt = p.values
        M = case if kind == "batch" else SPAN_CASES[case][1]
        cw_opt = GEMV_CW_OPTION if cw_opt is None else cw_opt
        for name, IC, norm, epi in step_gemvs(GEOMETRIES[wd]):
            sl = gemv_slices(IC, M, optin, cw_opt)
            cw = gemv_consumer_warps(IC, M, cw_opt)
            where = (wd, name, M)
            if M == 1:
                seen.setdefault(f"M = 1: consume1, {cw} consumer warps" + (" at IC > 8192" if IC > 8192 else ""), []).append(where)
                continue
            if norm:
                seen.setdefault("RMSNorm prologue, unsliced" if len(sl) == 1 else
                                ("RMSNorm prologue, sliced, short last slice" if sl[-1] < sl[0] else "RMSNorm prologue, sliced"), []).append(where)
            if epi == "residual add" and len(sl) > 1:
                seen.setdefault(f"sliced residual add, {'ordered fix-up' if det else 'RED.ADD'}", []).append(where)
            if epi == "SiLU pair":
                seen.setdefault("SiLU pair epilogue at M >= 2" + (", sliced" if len(sl) > 1 else ""), []).append(where)
    return seen


GEMV_REQUIRED = {"M = 1: consume1, 16 consumer warps at IC > 8192", "M = 1: consume1, 8 consumer warps", "RMSNorm prologue, unsliced",
                 "RMSNorm prologue, sliced, short last slice", "sliced residual add, RED.ADD", "sliced residual add, ordered fix-up",
                 "SiLU pair epilogue at M >= 2", "SiLU pair epilogue at M >= 2, sliced"}


def test_standalone_plans_covered():
    """The cases of test_kernel_per_op_step_phases meet every class of the stand-alone attention's split plan and of the multi-column
    GEMV's K-slice plan at this device's shared memory.  Prints the plans."""
    from tinychatengine_b200.llama import GEOMETRIES

    optin = smem_optin()
    for wd in KPO_WIDTHS:
        g = GEOMETRIES[wd]
        print(f"[attention plan {wd}] batched chunk {ATTN_CHUNK}, span chunk {attn_span_chunk(g.num_heads, g.num_kv_heads, ATTN_CHUNK, optin)} "
              f"({g.num_heads // g.num_kv_heads} query heads per KV head, {optin} B of shared memory per block)")
        for name, IC, norm, epi in step_gemvs(g):
            print(f"[K-slices {wd} {name}] IC {IC}: " + ", ".join(f"M={M}: {'+'.join(map(str, gemv_slices(IC, M, optin)))}" for M in (1, 2)))
        assert attn_span_chunk(g.num_heads, g.num_kv_heads, ATTN_CHUNK, optin) > 0
    seen = batch_classes(ATTN_CHUNK, 4096)
    print("[split classes, batched step] " + "; ".join(f"{c}: {seen[c]}" for c in sorted(seen)))
    assert STANDALONE_REQUIRED <= set(seen), STANDALONE_REQUIRED - set(seen)
    for wd in KPO_WIDTHS:
        g = GEOMETRIES[wd]
        span_chunk = attn_span_chunk(g.num_heads, g.num_kv_heads, ATTN_CHUNK, optin)
        seen = span_classes(span_chunk, 4096)
        print(f"[span classes {wd}, chunk {span_chunk}] " + "; ".join(f"{c}: {seen[c]}" for c in sorted(seen)))
        assert SPAN_REQUIRED <= set(seen), (wd, SPAN_REQUIRED - set(seen))
    gs = gemv_classes(optin)
    print("[K-slice classes] " + "; ".join(f"{c}: {gs[c][:3]}" for c in sorted(gs)))
    assert GEMV_REQUIRED <= set(gs), GEMV_REQUIRED - set(gs)


def _run_step(w, model, kind, tokens, positions, slots, seed, peak=None):
    """Caches of every slot random below its sequence's first position and NaN from there on (NaN in unused slots), rows past the step of
    the four step buffers NaN; then the step.  Returns (logits on the device [n, V], greedy ids, every slot's K / V bits before)."""
    g = w.g
    n = len(tokens)
    first = {}
    for s, p in zip(slots, positions):
        first[s] = min(first.get(s, p), p)
    for s in range(model.MAX_BATCH):
        _fill_cache(model, first.get(s, 0), seed=seed + 101 * s, slot=s)
    if peak is not None:  # (sequence b, cached row r): key r of b's slot aligned with b's query
        b, r = peak
        H, KVH = g.num_heads, g.num_kv_heads
        rep = H // KVH
        xn = wide_ref.rmsnorm(w.W["embed"][tokens[b]].double(), w.W["layers"][0]["input_norm"], g.rms_eps)
        q64, _, _ = wide_ref.decode_qkv(f16(xn @ w.w64["qkv"].T), H, KVH, w.cos[positions[b]], w.sin[positions[b]], 1.0 / math.sqrt(HD),
                                        round_q=False)
        qbar = q64.reshape(KVH, rep, HD).mean(1)
        kc = model.kv_cache(0, 0, slots[b])
        kc[:, r] = (qbar * (PEAK_SCORE / (qbar * qbar).sum(-1, keepdim=True))).to(torch.float16)
    before = {s: (_bits(model.kv_cache(0, 0, s)), _bits(model.kv_cache(0, 1, s))) for s in range(model.MAX_BATCH)}
    for i in range(4):
        model.debug_buffer(i)[n:] = float("nan")
    torch.cuda.synchronize()
    lg = torch.empty((n, g.vocab_size), dtype=torch.float32).pin_memory()
    if kind == "batch":
        ids = model.decode_batch_host(tokens, positions, slots, lg)
    else:
        ids = model.decode_span(tokens, positions[0], slots[0], lg)
    torch.cuda.synchronize()
    for i in range(4):
        assert model.debug_buffer(i)[n:].isnan().all(), f"the {n}-row step wrote row >= {n} of step buffer {i}"
    return lg.to(DEV), ids, before


def _gemv_check(tag, name, got, ref, bound, worst):
    r = _ratio(got, ref, bound)
    worst[name] = r.max().item()
    if worst[name] > 1.0:
        i, rv = _first_bad(r)
        row, col = divmod(i, ref.shape[-1])
        pytest.fail(f"{tag}: {name} row {row} element {col}: {got.flatten()[i].item()} ref {ref.flatten()[i].item()} ratio {rv:.3g}")


def _kpo_case(w, kind, det, case, cw_opt):
    g = w.g
    H, KVH = g.num_heads, g.num_kv_heads
    L0 = w.W["layers"][0]
    mode = "ordered" if det else "RED.ADD"
    if kind == "batch":
        positions = BATCH_CASES[case]
        slots = list(SLOT_ORDER[:case])
        peak = PEAK.get(case)
        chunk = ATTN_CHUNK
        tag = f"{g.name} {mode} batch {case} pos {positions}" + (f" cw-option {cw_opt}" if cw_opt is not None else "")
    else:
        p0, n = SPAN_CASES[case]
        positions = list(range(p0, p0 + n))
        slots = [SPAN_SLOT] * n
        peak = None
        chunk = attn_span_chunk(H, KVH, ATTN_CHUNK, smem_optin())
        tag = f"{g.name} {mode} span pos0 {p0} n {n}"
    n = len(positions)
    tokens = [(4321 + 977 * b) % g.vocab_size for b in range(n)]
    seed = 1000 * n + positions[0]
    model, zmodel = w.step_model(det), w.step_model(det, zero_down=True)
    worst = {}

    # the model whose down_proj is zero: o_proj into the residual, and SiLU*up from that residual
    _run_step(w, zmodel, kind, tokens, positions, slots, seed, peak)
    X = w.W["embed"][tokens].double()
    attn_z = zmodel.debug_buffer(2)[:n]
    o, mo = _linear(attn_z, w.w64["o"])
    x1 = zmodel.debug_buffer(0)[:n]
    _gemv_check(tag, "o_proj", x1, X + o, C_GEMV * mo + RESID_ADDS[det] * 2.0 ** -24 * (X.abs() + mo), worst)
    xn = wide_ref.rmsnorm(x1.double(), L0["post_norm"], g.rms_eps)
    gate, mg = _linear(xn, w.w64["gate"])
    up, mu = _linear(xn, w.w64["up"])
    ref = wide_ref.silu_mul(gate, up)
    act = zmodel.debug_buffer(3)[:n]
    silu = gate / (1.0 + torch.exp(-gate))
    bound = (0.5 * ulp_f16(torch.maximum(ref.abs(), act.double().abs())) + C_GEMV * (1.1 * up.abs() * mg + silu.abs() * mu)
             + (2.0 ** -21 + 2 * NORM_F32) * ref.abs())
    _gemv_check(tag, "SiLU*up", act, ref, bound, worst)

    # the model itself
    got_logits, ids, before = _run_step(w, model, kind, tokens, positions, slots, seed, peak)
    qkv = model.debug_buffer(1)[:n]
    xn = wide_ref.rmsnorm(X, L0["input_norm"], g.rms_eps)
    ref, mag = _linear(xn, w.w64["qkv"])
    _gemv_check(tag, "q|k|v", qkv, ref, 0.5 * ulp_f16(torch.maximum(ref.abs(), qkv.double().abs())) + C_GEMV * mag + NORM_F32 * ref.abs(), worst)

    # the appended rows: K = RoPE of the kernel's k words rounded to fp16, V = its v words bit for bit; no other row of any slot changes
    worst["K row (2 ulps + rotation)"] = 0.0
    for b, (s, p) in enumerate(zip(slots, positions)):
        kc, vc = model.kv_cache(0, 0, s), model.kv_cache(0, 1, s)
        _, kref, vw = wide_ref.decode_qkv(qkv[b], H, KVH, w.cos[p], w.sin[p], 1.0)
        kin = qkv[b].double().reshape(H + 2 * KVH, HD)[H:H + KVH].abs()
        pair_mag = kin[:, :HD // 2] + kin[:, HD // 2:]
        kb = 2 * ulp_f16(kref) + 2.0 ** -20 * torch.cat([pair_mag, pair_mag], dim=-1)
        worst["K row (2 ulps + rotation)"] = max(worst["K row (2 ulps + rotation)"], _ratio(kc[:, p], kref, kb).max().item())
        assert torch.equal(vc[:, p].double(), vw), f"{tag}: row {b}: the appended V row of slot {s} pos {p} is not the row's v words"
    assert worst["K row (2 ulps + rotation)"] <= 1.0, (tag, worst)
    for s in range(model.MAX_BATCH):
        for which, name in ((0, "K"), (1, "V")):
            changed = (before[s][which] != _bits(model.kv_cache(0, which, s))).any(-1)
            for s_b, p in zip(slots, positions):
                if s_b == s:
                    changed[:, p] = False
            assert not changed.any(), f"{tag}: {name} rows of slot {s} other than the step's changed: {changed.nonzero()[:4].tolist()}"

    # attention of every row over its slot, at the stand-alone plan
    attn = model.debug_buffer(2)[:n]
    worst["attention"] = 0.0
    if kind == "batch":
        for b, (s, p) in enumerate(zip(slots, positions)):
            splits = standalone_splits(chunk, p)
            units, ukind = _units(splits, p + 1)
            wv, _, _, top = _attention_check(f"{tag} row {b} slot {s} pos {p}", w, qkv[b:b + 1], [p], model.kv_cache(0, 0, s), model.kv_cache(0, 1, s),
                                             attn[b:b + 1], units, ukind, f"chunk={chunk} nsplit={len(splits)}")
            worst["attention"] = max(worst["attention"], wv)
            if peak is not None and peak[0] == b:
                idx, share = top[0]
                hit = (idx == peak[1])
                print(f"[{tag} row {b}] planted key {peak[1]} (split {peak[1] // chunk}) is the largest weight of {int(hit.sum())} of {H} heads, "
                      f"median weight share {share[hit].median().item() if hit.any() else 0.0:.2f}")
                assert hit.sum().item() >= H // 2 and share[hit].median().item() >= 0.25, f"{tag}: the planted key does not dominate"
    else:
        splits = standalone_splits(chunk, positions[0], n)
        units, ukind = _units(splits, positions[-1] + 1)
        wv, _, cpow, _ = _attention_check(f"{tag}", w, qkv, positions, model.kv_cache(0, 0, SPAN_SLOT), model.kv_cache(0, 1, SPAN_SLOT), attn,
                                          units, ukind, f"chunk={chunk} nsplit={len(splits)}", causal=n > 1)
        worst["attention"] = wv
        if n > 1:
            assert cpow >= POWER_MIN, f"{tag}: the attention bound cannot see a key leaked from the next span row ({cpow:.2f} bounds)"

    # residual = embedding + o_proj(attention words) + down_proj(SiLU*up words), fp32
    act = model.debug_buffer(3)[:n]
    o, mo = _linear(attn, w.w64["o"])
    d, md = _linear(act, w.w64["down"])
    resid = model.debug_buffer(0)[:n]
    _gemv_check(tag, "residual (o_proj + down_proj)", resid, X + o + d, C_GEMV * (mo + md) + RESID_ADDS[det] * 2.0 ** -24 * (X.abs() + mo + md), worst)

    # logits: final RMSNorm of the residual -> lm_head, fp32; the greedy ids are the first arg-max of each row
    xn = wide_ref.rmsnorm(resid.double(), w.W["final_norm"], g.rms_eps)
    ref, mag = _linear(xn, w.w64["lm_head"])
    _gemv_check(tag, "logits", got_logits, ref, C_GEMV * mag + NORM_F32 * ref.abs(), worst)
    assert ids == torch.argmax(got_logits, dim=-1).tolist(), tag
    print(f"[{tag}] worst |d| / bound: " + ", ".join(f"{k} {v:.3f}" for k, v in worst.items()))
    return worst


@pytest.fixture(scope="module")
def kpo_worst():
    """Worst ratio per (geometry, residual mode, step kind) and phase over the cases that ran, printed when the module ends."""
    table = {}
    yield table
    for key, v in sorted(table.items()):
        print(f"[kernel-per-op worst {' '.join(key)}] " + ", ".join(f"{k} {x:.3f}" for k, x in v.items()))


@pytest.mark.parametrize("widths,det,kind,case,cw_opt", _kpo_cases())
def test_kernel_per_op_step_phases(wide, kpo_worst, widths, det, kind, case, cw_opt):
    """One batched step of B sequences, each in its own slot (slots in non-identity order), or one span step of n rows of one slot, of a
    1-layer model at Llama-3-8B (GQA 32:8, full vocabulary), Llama-2-7B (MHA, F = 11008: 86 groups) or Llama-2-13B (E = 5120: the
    RMSNorm-prologue GEMVs K-slice) widths, with the residual partials added by RED.ADD or by the ordered fix-up, on caches random below
    each sequence's first position and NaN from it on and step buffers NaN past the step's rows: every phase of every row against float64
    from its own inputs (see above)."""
    w = wide(widths, 4096)
    if cw_opt is not None:
        w.ctx.set_option("gemv_consumer_warps", cw_opt)
    try:
        worst = _kpo_case(w, kind, det, case, cw_opt)
    finally:
        if cw_opt is not None:
            w.ctx.set_option("gemv_consumer_warps", GEMV_CW_OPTION)
    row = kpo_worst.setdefault((w.g.name, "ordered" if det else "RED.ADD", kind), {})
    for k, v in worst.items():
        row[k] = max(row.get(k, 0.0), v)


# ------------------------------------------------------------------------------------------------ d. whole 2-layer steps, both paths

# about twice the worst value of an H100 SXM (700 W) run, given after each bound
E2E_LOGITS = 1.2e-3    # per step: max |d| / max |ref|; 6.1e-4 (7B, per op), 4.7e-4 (8B, persistent)
E2E_KV0_ULPS = 1       # layer-0 K/V rows: max |d| over a row in fp16 ulps of the row's max; 0.5
E2E_KV1 = 2e-3         # layer-1 K/V rows: max |d| / max |ref| per row; 1.01e-3
DEVICE_ENTRY = 2e-4    # decode() against decode_host() of the same step, per-op path (fp32 RED.ADD order): 8.6e-5 (7B), 0 (8B); the
                       # persistent path is bitwise


@pytest.mark.parametrize("mega", ["1", "0"])
@pytest.mark.parametrize("widths", ["llama3-8b", "llama2-7b"])
def test_two_layer_steps_across_boundaries(widths, mega, monkeypatch):
    """2 layers at the benchmarked widths, TCE_PERSISTENT=1 (persistent kernel) and 0 (kernel per op), a cache NaN from the token on:
    the steps 1020 -> 1030 and 4090 -> 4095, each against wide_ref.decode_step on the rows the cache holds before it; the rows of both
    layers, no other row touched, and decode() (device token / position) against decode_host()."""
    import dataclasses

    from oracle import capi
    from tinychatengine_b200.llama import GEOMETRIES, LlamaModel
    from tinychatengine_b200.runtime import Context

    for w in _WIDE.values():  # the 1-layer models and their float64 weights make room
        w.close()
    _WIDE.clear()
    torch.cuda.empty_cache()
    monkeypatch.setenv("TCE_PERSISTENT", mega)
    g = dataclasses.replace(GEOMETRIES[widths], name=f"{widths}-2l", num_layers=2)
    ctx = Context(0)
    model = LlamaModel(ctx, g, max_ctx=4096, seed=23, random_zeros=True)
    assert (model.kernels_per_step == 1) == (mega == "1")
    cosb, sinb = capi.rope_tables(4096, HD, g.rope_theta)
    lg = torch.empty(g.vocab_size, dtype=torch.float32).pin_memory()
    worst = {"logits": 0.0, "kv layer0 ulps": 0.0, "kv layer1": 0.0, "decode vs decode_host": 0.0}
    tok = 777
    for p0, p1 in ((1020, 1030), (4090, 4095)):
        _fill_cache(model, p0, seed=p0)
        for pos in range(p0, p1 + 1):
            caches = [(model.kv_cache(l, 0), model.kv_cache(l, 1)) for l in range(2)]
            before = [(_bits(k), _bits(v)) for k, v in caches]
            past = [(k[:, :pos], v[:, :pos]) for k, v in caches]
            ref, K, V = wide_ref.decode_step(model.W, g, tok, pos, past, cosb, sinb)
            nxt = model.decode_host(tok, pos, lg)
            got = lg.to(DEV)
            assert torch.isfinite(got).all(), (widths, mega, pos)
            e = row_rel_err(got, ref).item()
            worst["logits"] = max(worst["logits"], e)
            assert nxt == int(torch.argmax(got).item())
            for l, (k, v) in enumerate(caches):
                for name, c, R in (("K", k, K[l]), ("V", v, V[l])):
                    d = (c[:, pos].double() - R).abs().amax(-1)
                    mx = R.abs().amax(-1)
                    if l == 0:
                        worst["kv layer0 ulps"] = max(worst["kv layer0 ulps"], (d / ulp_f16(mx)).max().item())
                    else:
                        worst["kv layer1"] = max(worst["kv layer1"], (d / mx).max().item())
                    b = before[l][0 if name == "K" else 1]
                    changed = (b != _bits(c)).any(-1)
                    changed[:, pos] = False
                    assert not changed.any(), (widths, mega, pos, l, name, changed.nonzero()[:4].tolist())
            if e > E2E_LOGITS:
                print(f"[{widths} TCE_PERSISTENT={mega}] pos {pos}: logits rel err {e:.3g}")
            # the device entry point on the same step (it rewrites row pos with the same values)
            model.decode(torch.tensor([tok, pos], dtype=torch.int32, device=DEV))
            torch.cuda.synchronize()
            dev_logits = model.logits()
            if mega == "1":
                assert torch.equal(dev_logits, got), (widths, pos, "decode() != decode_host()")
            else:
                worst["decode vs decode_host"] = max(worst["decode vs decode_host"], row_rel_err(dev_logits, got.double()).item())
            tok = (nxt * 7 + pos) % g.vocab_size
    tagname = f"2-layer steps {widths} TCE_PERSISTENT={mega}, 1020..1030 and 4090..4095"
    print(f"[{tagname}] " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))
    bounds = {"logits": E2E_LOGITS, "kv layer0 ulps": E2E_KV0_ULPS, "kv layer1": E2E_KV1, "decode vs decode_host": DEVICE_ENTRY}
    model.close()
    ctx.close()
    for k, v in worst.items():
        assert v <= bounds[k], (tagname, k, v, bounds[k])
