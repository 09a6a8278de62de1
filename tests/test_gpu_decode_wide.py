"""The decode step at the widths the benchmark times, phase by phase, against float64 (tests/wide_ref.py, pinned on the CPU by
tests/test_wide_ref.py).

The logits of a step cannot guard its attention: with random weights the softmax is nearly flat, and a lost flash-decode split moves
the logits of a 2-layer Llama-3-8B step by less than 1e-2.  So the persistent kernel is checked here through its hand-off words
(LlamaModel.handoff_views: after a step of a 1-layer model they hold that layer's q|k|v, attention output, SiLU*up and o_proj /
down_proj outputs), each phase against float64 computed from that phase's own inputs as the kernel saw them.  Errors do not compound,
and every bound sits near fp16 rounding.  The positions follow the attention split plan (attn_split of decode_persistent.cu, restated
by attn_plan) at the device's SM count, and every attention case shows that the bound would see one lost split.  Then whole 2-layer
steps on both decode paths, across chunk and split boundaries, each against wide_ref.decode_step on the cache rows the kernel holds.
Every case prints its worst ratio to its bound."""
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
    """A 1-layer model at a benchmarked geometry: its weights expanded to float64 once, and one LlamaModel per staging mode."""

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

    def model(self, pair: bool):
        if pair not in self.models:
            from tinychatengine_b200.llama import LlamaModel

            saved = {k: os.environ.get(k) for k in ("TCE_PERSISTENT", "TCE_PK_PAIR")}
            os.environ["TCE_PERSISTENT"] = "1"
            if pair:
                os.environ.pop("TCE_PK_PAIR", None)
            else:
                os.environ["TCE_PK_PAIR"] = "0"
            try:
                self.models[pair] = LlamaModel(self.ctx, self.g, max_ctx=self.max_ctx, weights=self.W)
            finally:
                for k, v in saved.items():
                    if v is None:
                        os.environ.pop(k, None)
                    else:
                        os.environ[k] = v
        return self.models[pair]

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


def _fill_cache(model, pos, seed, k_std=1.0, v_std=1.0):
    """Random fp16 rows below pos and NaN from pos on, in every head of every layer: a row the step should have written and did not, or
    a row past the token that reaches the output, shows up as NaN."""
    gen = torch.Generator(device=DEV)
    gen.manual_seed(seed)
    for l in range(model.geom.num_layers):
        for which, std in ((0, k_std), (1, v_std)):
            c = model.kv_cache(l, which)
            c.fill_(float("nan"))
            if pos:
                c[:, :pos] = (torch.randn((c.shape[0], pos, HD), device=DEV, generator=gen) * std).to(torch.float16)


def _bits(t):
    return t.view(torch.int16).clone()


# ------------------------------------------------------------------------------------------------ a./b./c./e. every phase of one step

def _attention_check(tag, w, model, pos, qkv16, kc, vc):
    """The attention words of every head against decode_attention on the kernel's own q|k|v words and the cache rows; then the power
    check: the smallest change that losing one split (or, with one split, one 16-row block) of one KV head makes, in bounds."""
    g = w.g
    H, KVH = g.num_heads, g.num_kv_heads
    rep = H // KVH
    alpha = 1.0 / math.sqrt(HD)
    q64, k, v = wide_ref.decode_qkv(qkv16, H, KVH, w.cos[pos], w.sin[pos], alpha, round_q=False)
    qa = f16(q64)
    K = kc[:, :pos + 1].double().clone()
    V = vc[:, :pos].double()
    V = torch.cat([V, v[:, None]], dim=1)  # the token's value: its own v word (the appended row is checked bit for bit elsewhere)
    ref, p, L = wide_ref.decode_attention(qa, K, V)
    got = model.handoff_views()["attn"][0].double().reshape(H, HD)
    Vh = V.repeat_interleave(rep, dim=0)
    Kh = K.repeat_interleave(rep, dim=0)
    A = torch.einsum("ht,htd->hd", p, Vh.abs()) / L[:, None]       # sum_j p_j |v_j| / L
    B = Vh.abs().sum(1) / L[:, None]                                 # sum_j |v_j| / L
    # score error: the fp32 sum of the MMA, and the elements of q * alpha that lie so close to a rounding boundary of fp16 that the fp32
    # RoPE (error < 2^-21 alpha (|x_d| + |x_d'|)) may round them to the other neighbour (one ulp)
    xq = qkv16.double().reshape(-1, HD)[:H].abs()
    xq = xq + torch.cat([xq[:, HD // 2:], xq[:, :HD // 2]], dim=-1)
    near = ((q64 - qa).abs() - 0.5 * ulp_f16(qa)).abs() <= 2.0 ** -21 * alpha * xq
    ds = (torch.einsum("hd,htd->ht", ulp_f16(qa) * near, Kh.abs()) + 2.0 ** -22 * torch.einsum("hd,htd->ht", qa.abs(), Kh.abs())).amax(-1)
    bound = 0.5 * ulp_f16(torch.maximum(ref.abs(), got.abs())) + (P_ROUND + 2 * ds[:, None] + ATTN_FP32) * A + P_SUBNORMAL * B
    ratio = _ratio(got, ref, bound)
    worst = ratio.max().item()

    # the units a lost partial would take away: the splits of the plan, or the 16-row blocks of a single split
    NS, cps, splits = attn_plan(w.ctx.num_sms, KVH, pos)
    if len(splits) > 1:
        units = [(c0 * CHUNK, min(pos + 1, c1 * CHUNK)) for c0, c1 in splits]
        kind = "split"
    else:
        units = [(r, min(pos + 1, r + 16)) for r in range(0, pos + 1, 16)]
        kind = "16-row block"
    N = ref * L[:, None]
    without = []
    for r0, r1 in units:
        Nu = torch.einsum("ht,htd->hd", p[:, r0:r1], Vh[:, r0:r1])
        Lu = p[:, r0:r1].sum(-1)
        without.append((N - Nu) / (L - Lu)[:, None])
    # power: whichever unit is lost, the KV head where that loss shows most moves by `power` bounds or more (a unit of a single key
    # whose weight is negligible in some head would not move that head's output at all)
    power = math.inf
    if len(units) > 1:
        eff = torch.stack([((o - ref).abs() / bound).reshape(KVH, rep * HD).amax(-1) for o in without])  # [unit, kvh]
        power = eff.amax(1).min().item()
    msg = (f"[{tag} attention] worst |y - ref| / bound {worst:.3f} over {H} heads; plan NS={NS} cps={cps} nsplit={len(splits)}; "
           + (f"losing any one {kind} moves some head by >= {power:.1f} bounds" if len(units) > 1 else "one key: no partial to lose"))
    print(msg)
    if worst > 1.0:
        i, r = _first_bad(ratio)
        h, d = divmod(i, HD)
        if not torch.isfinite(got[h]).all():
            pytest.fail(f"{tag}: attention head {h} (KV head {h // rep}) dim {d} is {got[h, d].item()}: a NaN row of the cache (the token's "
                        f"own before it is patched into the stage, or a V row past it) reached the P.V product")
        near = min(range(len(units)), key=lambda u: (got[h] - without[u][h]).abs().max().item())
        r0, r1 = units[near]
        pytest.fail(f"{tag}: attention head {h} (KV head {h // rep}) dim {d}: y {got[h, d].item()} ref {ref[h, d].item()} ratio {r:.3g}; "
                    f"closest to the reference without {kind} {near} (rows {r0}..{r1 - 1}): max |y - that| "
                    f"{(got[h] - without[near][h]).abs().max().item():.3g}")
    if len(units) > 1:
        assert power >= POWER_MIN, f"{tag}: the attention bound cannot see a lost {kind} ({power:.2f} bounds)"
    return worst


def _phase_case(w, pos, pair, tok=4321, seed=0):
    g = w.g
    H, KVH = g.num_heads, g.num_kv_heads
    model = w.model(pair)
    tag = f"{g.name} max_ctx={w.max_ctx} pos={pos} {'pair' if pair else 'pair0'}"
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
    worst["attention"] = _attention_check(tag, w, model, pos, qkv, kc, vc)

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
    """(widths, max_ctx, pair, position index or an explicit position): pair staging at every position of the plan, single-CTA staging
    at a subset; max_ctx 4000 (not a multiple of 64) at its last rows."""
    out = [pytest.param("llama3-8b", 4096, True, i, id=f"llama3-8b-pair-{i}") for i in range(10)]
    out += [pytest.param("llama3-8b", 4096, False, i, id=f"llama3-8b-pair0-{i}") for i in (1, 4, 8)]
    out += [pytest.param("llama2-7b", 4096, True, i, id=f"llama2-7b-pair-{i}") for i in range(10)]
    out += [pytest.param("llama3-8b", 4000, True, p, id=f"llama3-8b-ctx4000-last{-p}") for p in (-1, -32)]
    return out


@pytest.mark.parametrize("widths,max_ctx,pair,which", _phase_cases())
def test_persistent_step_phases(wide, widths, max_ctx, pair, which):
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
    _phase_case(w, pos, pair)


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
