"""Speculative decoding: the span step (tce_llama_decode_span_host: n consecutive tokens of one slot in one pass) and the greedy prompt-lookup
loop (tce_llama_generate_lookup) against the oracle, a host replay, the batched step and the plain greedy loop."""
import numpy as np
import pytest
import torch

from helpers import np_w4, rel_err
from oracle import capi
from oracle.sampling import apply_penalties

pytestmark = pytest.mark.gpu

PEN = dict(repeat_penalty=1.3, frequency_penalty=0.1, presence_penalty=0.05, repeat_last_n=16)


def _model(geom, max_ctx, seed=7, n_slots=4, deterministic=True, monkeypatch=None, chunk=None):
    """chunk: cached rows per attention CTA (the context's attn_chunk, read when the model is built); None keeps the default"""
    from tinychatengine_b200.llama import GEOMETRIES, LlamaModel
    from tinychatengine_b200.runtime import Context

    if deterministic and monkeypatch is not None:
        monkeypatch.setenv("TCE_DETERMINISTIC", "1")
    ctx = Context(0)
    if chunk is not None:
        ctx.set_option("attn_chunk", chunk)
    model = LlamaModel(ctx, GEOMETRIES[geom] if isinstance(geom, str) else geom, max_ctx=max_ctx, seed=seed, random_zeros=True)
    model.reserve_slots(n_slots)
    return ctx, model


def _close(model, ctx):
    model.close()
    ctx.close()


def _fill(model, n_slots, seed):
    gen = torch.Generator(device="cuda")
    gen.manual_seed(seed)
    for s in range(n_slots):
        for l in range(model.geom.num_layers):
            for w in (0, 1):
                c = model.kv_cache(l, w, s)
                c.copy_((torch.randn(c.shape, device="cuda", generator=gen) * 0.5).to(torch.float16))


def _snap(model, n_slots):
    return [[[model.kv_cache(l, w, s).cpu().clone() for w in (0, 1)] for l in range(model.geom.num_layers)] for s in range(n_slots)]


def _assert_untouched(before, after, slot=None, lo=0, hi=0):
    """every row of every slot byte-identical, except rows [lo, hi) of `slot`"""
    for s in range(len(before)):
        for l in range(len(before[s])):
            for w in (0, 1):
                a, b = before[s][l][w].clone(), after[s][l][w].clone()
                if s == slot:
                    a[:, lo:hi] = 0
                    b[:, lo:hi] = 0
                assert torch.equal(a, b), (s, l, w, lo, hi)


def _oracle_span(model, tokens, pos0, snap, slot):
    """logits [n, V] and the new K / V rows of n tokens after the pos0 cached rows of `slot` (llama_ref.llama_forward, the fused path's arithmetic)"""
    from oracle import llama_ref

    g = model.geom
    cosb, sinb = capi.rope_tables(model.max_ctx, g.head_dim, g.rope_theta)
    pk = [snap[slot][l][0][:, :pos0].float().numpy() if pos0 else None for l in range(g.num_layers)]
    pv = [snap[slot][l][1][:, :pos0].float().numpy() if pos0 else None for l in range(g.num_layers)]

    def linear(xh, t):
        w, z, s = np_w4(t)
        return capi.w4a16_gemv(np.asarray(xh).astype(np.float16), w, z, s)

    layers = []
    for l in range(g.num_layers):
        lt = model.layer_tensors(l)
        layers.append({**{n: lt[n] for n in llama_ref.LINEARS}, "input_norm": lt["input_norm"].cpu().numpy(), "post_norm": lt["post_norm"].cpu().numpy()})
    return llama_ref.llama_forward(
        list(tokens), pk, pv, embed_row=lambda t: model.embed[t].float().cpu().numpy(), layers=layers, final_norm=model.final_norm.cpu().numpy(),
        lm_head=model.tensors[-1], linear=linear, cosb=cosb, sinb=sinb, H=g.num_heads, KVH=g.num_kv_heads, hd=g.head_dim, eps=g.rms_eps,
        rnd=lambda a: np.asarray(a).astype(np.float16), round_new_k=lambda a: a.astype(np.float16).astype(np.float32))


# ---------------------------------------------------------------------------------------------------------------- span attention alone
def _np_span_attention(qkv, pk, pv, pos0, H, KVH, cosb, sinb):
    """numpy causal GQA attention of n tokens at pos0.. over pos0 cached rows (capi.llama_attention_core, fp32)"""
    n = qkv.shape[0]
    q = qkv[:, :H * 128].astype(np.float32)
    k = qkv[:, H * 128:(H + KVH) * 128].astype(np.float32)
    v = qkv[:, (H + KVH) * 128:].astype(np.float32)
    return capi.llama_attention_core(q, k, v, pk.astype(np.float32) if pos0 else None, pv.astype(np.float32) if pos0 else None,
                                     capi.causal_mask(n, pos0), cosb, sinb, 1.0 / np.sqrt(128), H, KVH, 128)


@pytest.mark.parametrize("chunk", [16, 64, 256])
@pytest.mark.parametrize("H,KVH", [(4, 4), (8, 2), (16, 2)])
def test_span_attention_matches_numpy(H, KVH, chunk):
    """tce_attn_span against numpy for n = 1..8 at contexts 1..4096: spans inside one split, spans whose new rows cross a split boundary
    (two CTAs append parts of the span, and a split holds query rows that see none of its keys), one split and many."""
    from tinychatengine_b200.runtime import Context

    max_ctx = 4096
    c = Context(0)
    c.set_option("attn_chunk", chunk)
    dev = torch.device("cuda", 0)
    cosb, sinb = capi.rope_tables(max_ctx, 128, 500000.0)
    dcos, dsin = torch.from_numpy(cosb).to(dev), torch.from_numpy(sinb).to(dev)
    rng = np.random.default_rng(100 * H + chunk)
    for n in range(1, 9):
        for pos0 in sorted({0, 1, chunk - 1 - n // 2, 3 * chunk - 2, 1000, max_ctx - n}):
            qkv = rng.standard_normal((n, (H + 2 * KVH) * 128)).astype(np.float16)
            pk = (rng.standard_normal((KVH, pos0, 128)) * 0.7).astype(np.float16)
            pv = rng.standard_normal((KVH, pos0, 128)).astype(np.float16)
            want, fk, fv = _np_span_attention(qkv, pk, pv, pos0, H, KVH, cosb, sinb)
            kc = torch.full((KVH, max_ctx, 128), float("nan"), dtype=torch.float16, device=dev)  # unwritten rows must never be read
            vc = torch.full_like(kc, float("nan"))
            kc[:, :pos0] = torch.from_numpy(pk).to(dev)
            vc[:, :pos0] = torch.from_numpy(pv).to(dev)
            out = torch.zeros((n, H * 128), dtype=torch.float16, device=dev)
            c.attn_span(torch.from_numpy(qkv).to(dev), kc, vc, dcos, dsin, out, 1.0 / np.sqrt(128), n, pos0, H, KVH, 128, max_ctx)
            torch.cuda.synchronize()
            got = out.float().cpu().numpy()
            assert np.all(np.isfinite(got)), (n, pos0)
            assert np.abs(got - want).max() / max(np.abs(want).max(), 1e-6) <= 3e-3, (n, pos0)
            assert np.allclose(kc[:, pos0:pos0 + n].float().cpu().numpy(), fk[:, pos0:], atol=2e-3, rtol=1e-3), (n, pos0)
            assert np.array_equal(vc[:, pos0:pos0 + n].cpu().numpy(), fv[:, pos0:].astype(np.float16)), (n, pos0)
            assert torch.equal(kc[:, :pos0].cpu(), torch.from_numpy(pk)) and torch.equal(vc[:, :pos0].cpu(), torch.from_numpy(pv))
            assert torch.isnan(kc[:, pos0 + n:]).all() and torch.isnan(vc[:, pos0 + n:]).all()
    c.close()


# ---------------------------------------------------------------------------------------------------------------- span step
@pytest.mark.parametrize("n", list(range(1, 9)))
@pytest.mark.parametrize("geom", ["tiny-gqa", "tiny-mha"])
def test_span_step_matches_oracle(geom, n, monkeypatch):
    """16-row attention splits (8 over max_ctx 128): pos0 = 13 and 45 put the new rows of n >= 4 across a split boundary."""
    max_ctx = 128
    ctx, model = _model(geom, max_ctx, monkeypatch=monkeypatch, chunk=16)
    g = model.geom
    for slot in (0, 3):
        for pos0 in (0, 13, 45, max_ctx - n):
            _fill(model, 4, 1000 * n + 10 * slot + pos0 % 7)
            before = _snap(model, 4)
            toks = [(97 * i + 13 * n + pos0 + slot) % g.vocab_size for i in range(n)]
            lg = torch.empty((n, g.vocab_size), dtype=torch.float32).pin_memory()
            nxt = model.decode_span(toks, pos0, slot, lg)
            after = _snap(model, 4)
            want, fk, fv = _oracle_span(model, toks, pos0, before, slot)
            got = lg.numpy()
            for i in range(n):
                assert rel_err(got[i], want[i]) <= 1e-2, (slot, pos0, i, rel_err(got[i], want[i]))
                assert nxt[i] == int(np.argmax(got[i]))
            for l in range(g.num_layers):
                k = after[slot][l][0][:, pos0:pos0 + n].float().numpy()
                v = after[slot][l][1][:, pos0:pos0 + n].float().numpy()
                assert np.abs(k - fk[l][:, pos0:pos0 + n]).max() <= 2e-2 * max(1.0, np.abs(fk[l]).max()), (slot, pos0, l)
                assert np.abs(v - fv[l][:, pos0:pos0 + n]).max() <= 5e-3 * max(1.0, np.abs(fv[l][:, pos0:pos0 + n]).max()), (slot, pos0, l)
            _assert_untouched(before, after, slot, pos0, pos0 + n)
            # n consecutive batched steps on a copy of the same cache: the same rows to rounding
            for s in range(4):
                for l in range(g.num_layers):
                    for w in (0, 1):
                        model.kv_cache(l, w, s).copy_(before[s][l][w].cuda())
            seq = np.stack([_one_row(model, t, pos0 + i, slot) for i, t in enumerate(toks)])
            tol = 1e-2 * np.abs(seq).max()
            assert np.abs(seq - got).max() <= tol
            for i in range(n):
                top2 = np.sort(seq[i])[-2:]
                if top2[1] - top2[0] > 2 * tol:
                    assert nxt[i] == int(np.argmax(seq[i]))
    _close(model, ctx)


def _one_row(model, tok, pos, slot):
    lg = torch.empty((1, model.geom.vocab_size), dtype=torch.float32).pin_memory()
    model.decode_batch_host([tok], [pos], [slot], lg)
    return lg.numpy()[0].copy()


def test_span_of_one_row_is_the_batched_step(monkeypatch):
    """TCE_DETERMINISTIC=1, GQA 4:1, 256-row splits (the span runs the same split): the span step of one token and the batched step of one
    sequence give the same logits and K / V cache bits, on slot 0 and another slot, in one split, on a split boundary and over many."""
    ctx, model = _model("tiny-gqa", 1024, monkeypatch=monkeypatch, chunk=256)
    g = model.geom
    for slot in (0, 3):
        for pos in (0, 255, 256, 1000):
            _fill(model, 4, 10 * slot + pos)
            before = _snap(model, 4)
            tok = (31 * pos + 7 * slot + 1) % g.vocab_size
            lg = torch.empty((1, g.vocab_size), dtype=torch.float32).pin_memory()
            model.decode_span([tok], pos, slot, lg)
            span_lg, span_kv = lg.numpy()[0].copy(), _snap(model, 4)
            for s in range(4):
                for l in range(g.num_layers):
                    for w in (0, 1):
                        model.kv_cache(l, w, s).copy_(before[s][l][w].cuda())
            assert np.array_equal(span_lg, _one_row(model, tok, pos, slot)), (slot, pos)
            after = _snap(model, 4)
            for s in range(4):
                for l in range(g.num_layers):
                    for w in (0, 1):
                        assert torch.equal(span_kv[s][l][w], after[s][l][w]), (slot, pos, s, l, w)
    _close(model, ctx)


def test_span_step_long_context(monkeypatch):
    """Contexts up to 4096 with the default 256-row splits (16 of them), GQA 4:1: the span rows against the oracle, also with the new rows
    across a split boundary (pos0 = 253, 510)."""
    ctx, model = _model("tiny-gqa", 4096, n_slots=1, monkeypatch=monkeypatch)
    g = model.geom
    for n, pos0 in ((8, 4096 - 8), (3, 1000), (5, 253), (8, 510)):
        _fill(model, 1, n)
        before = _snap(model, 1)
        toks = [(31 * i + 5) % g.vocab_size for i in range(n)]
        lg = torch.empty((n, g.vocab_size), dtype=torch.float32).pin_memory()
        model.decode_span(toks, pos0, 0, lg)
        want, _, _ = _oracle_span(model, toks, pos0, before, 0)
        for i in range(n):
            assert rel_err(lg.numpy()[i], want[i]) <= 1e-2, (n, pos0, i)
        _assert_untouched(before, _snap(model, 1), 0, pos0, pos0 + n)
    _close(model, ctx)


@pytest.mark.parametrize("n", [7, 8])
def test_span_step_eight_query_heads_per_kv_head(n, monkeypatch):
    """8 query heads per KV head (64 MMA columns at n = 8): the default 256-row split does not fit shared memory, the span attention runs the
    largest one that does; the step and the lookup loop at max_draft 7 run and agree with the oracle."""
    from tinychatengine_b200.llama import LlamaGeometry

    g = LlamaGeometry("tiny-rep8", 2, 16, 2, 1024, 2816, 2048, 1e-5, 500000.0)
    ctx, model = _model(g, 1024, n_slots=1, monkeypatch=monkeypatch)
    _fill(model, 1, n)
    for pos0 in (0, 230, 1024 - n):
        before = _snap(model, 1)
        toks = [(53 * i + 9) % g.vocab_size for i in range(n)]
        lg = torch.empty((n, g.vocab_size), dtype=torch.float32).pin_memory()
        model.decode_span(toks, pos0, 0, lg)
        want, _, _ = _oracle_span(model, toks, pos0, before, 0)
        for i in range(n):
            assert rel_err(lg.numpy()[i], want[i]) <= 1e-2, (pos0, i)
        _assert_untouched(before, _snap(model, 1), 0, pos0, pos0 + n)
    prompt = [(7 * i + 3) % g.vocab_size for i in range(16)]
    ids, st = model.generate_lookup(prompt[-1], 15, 24, history=prompt[:-1], corpus=prompt, max_draft=7)
    assert len(ids) == 24 and st["drafted"] > 0
    _close(model, ctx)


# ---------------------------------------------------------------------------------------------------------------- the lookup loop
def draft(S, max_draft, ngram, d):
    """the drafter rule of include/tce_b200.h, restated"""
    d = min(max_draft, d)
    if d <= 0:
        return []
    for ng in range(ngram[1], ngram[0] - 1, -1):
        if ng + 1 > len(S):
            continue
        suf = S[len(S) - ng:]
        for p in range(len(S) - ng - 1, -1, -1):
            if S[p:p + ng] == suf:
                return S[p + ng:p + ng + d]
    return []


def replay(model, first, pos0, n_predict, history, corpus, max_draft, ngram, eos_id, pen):
    """the loop on the host, each step through the same entry point at the same M"""
    V = model.geom.vocab_size
    n_predict = min(n_predict, model.max_ctx - pos0)
    S = list(corpus) + list(history) + [first]
    seq = list(history)  # the penalty window's sequence
    ids, pos, last = [], pos0, first
    st = {"steps": 0, "drafted": 0, "accepted": 0}
    rl = pen["repeat_last_n"]
    while len(ids) < n_predict:
        left = n_predict - len(ids)
        dr = draft(S, max_draft, ngram, min(left - 1, model.max_ctx - pos - 1))
        d = len(dr)
        lg = torch.empty((d + 1, V), dtype=torch.float32).pin_memory()
        if d == 0:
            model.decode_host(last, pos, lg[0])
        else:
            model.decode_span([last] + dr, pos, 0, lg)
        greedy = []
        for j in range(d + 1):
            win = (seq + dr[:j])
            win = win[-rl:] if rl >= 0 else win
            win = [0] * max(0, (rl if rl >= 0 else 0) - len(win)) + win
            pl = apply_penalties(lg.numpy()[j], win, pen["repeat_penalty"], pen["frequency_penalty"], pen["presence_penalty"])
            greedy.append(int(np.argmax(pl)))
        k = 0
        while k < d and greedy[k] == dr[k]:
            k += 1
        out = []
        for i in range(k + 1):
            if len(out) >= left:
                break
            t = dr[i] if i < k else greedy[k]
            out.append(t)
            if t == eos_id:
                break
        st["steps"] += 1
        st["drafted"] += d
        st["accepted"] += min(k, len(out))
        ids += out
        S += out
        seq += out
        pos += len(out)
        last = out[-1]
        if out[-1] == eos_id:
            break
    return ids, st


@pytest.mark.parametrize("geom", ["tiny-gqa", "tiny-mha"])
def test_lookup_loop_matches_host_replay(geom, monkeypatch):
    ctx, model = _model(geom, 256, n_slots=1, monkeypatch=monkeypatch)
    V = model.geom.vocab_size
    prompt = [(7 * i + 3) % V for i in range(20)]
    prompt = prompt + prompt[:12]  # repeats, so the drafter has something to propose
    model.prefill(prompt[:-1], 0)
    first, pos0, hist = prompt[-1], len(prompt) - 1, prompt[:-1]
    G, _ = model.generate_lookup(first, pos0, 40, history=hist, max_draft=0, **PEN)
    corpus = [first] + G[:25]
    for max_draft, ngram in ((7, (1, 3)), (3, (2, 2)), (7, (1, 1))):
        ids, st = model.generate_lookup(first, pos0, 40, history=hist, corpus=corpus, max_draft=max_draft, ngram=ngram, **PEN)
        r_ids, r_st = replay(model, first, pos0, 40, hist, corpus, max_draft, ngram, -1, PEN)
        assert ids == r_ids, (max_draft, ngram)
        assert st == r_st, (st, r_st)
        assert st["accepted"] > 0
    # every budget from 1 to 40: ids and counts agree at each, so a difference in any one step's draft, acceptance or emitted ids would
    # show at the budgets that end inside or right after that step, not only in the sums of a whole run
    for budget in range(1, 41):
        ids, st = model.generate_lookup(first, pos0, budget, history=hist, corpus=corpus, **PEN)
        assert (ids, st) == replay(model, first, pos0, budget, hist, corpus, 7, (1, 3), -1, PEN), budget
    _close(model, ctx)


def _top2_gap(model, first, pos0, hist, prefix, pen):
    """penalised top-2 gap of the one-token path at the step after `prefix`"""
    V = model.geom.vocab_size
    lg = torch.empty(V, dtype=torch.float32).pin_memory()
    last, seq = first, list(hist)
    for i, t in enumerate(prefix):
        model.decode_host(last, pos0 + i, lg)
        seq.append(t)
        last = t
    model.decode_host(last, pos0 + len(prefix), lg)
    rl = pen["repeat_last_n"]
    pl = apply_penalties(lg.numpy(), seq[-rl:], pen["repeat_penalty"], pen["frequency_penalty"], pen["presence_penalty"])
    top2 = np.sort(pl)[-2:]
    return float(top2[1] - top2[0]), 1e-2 * float(np.abs(pl).max())


@pytest.mark.parametrize("geom", ["tiny-gqa", "tiny-mha"])
def test_acceptance_happens(geom, monkeypatch):
    ctx, model = _model(geom, 256, n_slots=1, monkeypatch=monkeypatch)
    V = model.geom.vocab_size
    prompt = [(11 * i + 1) % V for i in range(16)]
    model.prefill(prompt[:-1], 0)
    first, pos0, hist = prompt[-1], len(prompt) - 1, prompt[:-1]
    G, st0 = model.generate_lookup(first, pos0, 48, history=hist, max_draft=0, **PEN)
    # max_draft = 0 is the plain greedy loop: the same step and the same sampler
    assert G == model.generate(first, pos0, 48, history=hist, temp=0.0, **PEN)
    assert st0 == {"steps": len(G), "drafted": 0, "accepted": 0}
    ids, st = model.generate_lookup(first, pos0, 48, history=hist, corpus=[first] + G, **PEN)
    n = len(ids)
    assert st["steps"] <= n / 2, st
    assert n == st["accepted"] + st["steps"], st
    if ids != G:
        k = next(i for i in range(min(n, len(G))) if ids[i] != G[i])
        gap, tol = _top2_gap(model, first, pos0, hist, G[:k], PEN)
        assert gap <= tol, ("ids differ at", k, gap, tol)
    _close(model, ctx)


def test_stopping_and_row_contract(monkeypatch):
    ctx, model = _model("tiny-gqa", 128, n_slots=2, monkeypatch=monkeypatch)
    V = model.geom.vocab_size
    prompt = [(5 * i + 2) % V for i in range(12)]
    model.prefill(prompt[:-1], 0)
    first, pos0, hist = prompt[-1], len(prompt) - 1, prompt[:-1]
    G, _ = model.generate_lookup(first, pos0, 40, history=hist, max_draft=0, **PEN)
    corpus = [first] + G
    # eos inside an accepted draft ends the output at it
    e = 9
    eos = G[e]
    ids, st = model.generate_lookup(first, pos0, 40, history=hist, corpus=corpus, eos_id=eos, **PEN)
    assert ids == G[:G.index(eos) + 1]
    assert len(ids) <= st["accepted"] + st["steps"]
    # the budget cuts an accepted run
    ids, st = model.generate_lookup(first, pos0, 10, history=hist, corpus=corpus, **PEN)
    assert ids == G[:10] and st["accepted"] + st["steps"] == 10
    # rows: [pos0, pos0 + n_out) hold the sequence, nothing at or past pos0 + n_out + max_draft and no other slot changes
    _fill(model, 2, 3)
    model.prefill(prompt[:-1], 0)
    before = _snap(model, 2)
    ids, _ = model.generate_lookup(first, pos0, 17, history=hist, corpus=corpus, max_draft=5, **PEN)
    after = _snap(model, 2)
    n = len(ids)
    _assert_untouched(before, after, 0, pos0, pos0 + n + 5)
    lg = torch.empty(V, dtype=torch.float32).pin_memory()
    for i, t in enumerate([first] + ids[:-1]):
        model.decode_host(t, pos0 + i, lg)
    for l in range(model.geom.num_layers):
        for w in (0, 1):
            a = after[0][l][w][:, pos0:pos0 + n].float()
            b = model.kv_cache(l, w, 0)[:, pos0:pos0 + n].float().cpu()
            assert (a - b).abs().max() <= 2e-2 * max(1.0, b.abs().max()), (l, w)
    # a start three rows before max_ctx stops there: exactly 3 ids, rows 125..127 of slot 0 written and nothing else
    before = _snap(model, 2)
    ids, st = model.generate_lookup(first, 125, 40, history=hist, corpus=corpus, **PEN)
    assert len(ids) == 3 and ids == replay(model, first, 125, 40, hist, corpus, 7, (1, 3), -1, PEN)[0]
    after = _snap(model, 2)
    _assert_untouched(before, after, 0, 125, 128)
    # n_predict = 0 writes nothing
    before = _snap(model, 2)
    ids, st = model.generate_lookup(first, pos0, 0, history=hist, corpus=corpus, **PEN)
    assert ids == [] and st == {"steps": 0, "drafted": 0, "accepted": 0}
    _assert_untouched(before, _snap(model, 2))
    _close(model, ctx)


def test_refusals(monkeypatch):
    import ctypes as C

    from tinychatengine_b200 import _lib

    ctx, model = _model("tiny-gqa", 64, n_slots=2, monkeypatch=monkeypatch)
    V = model.geom.vocab_size
    _fill(model, 2, 5)
    before = _snap(model, 2)
    L = ctx.L

    def span(slot, pos0, toks):
        arr = (C.c_int * max(1, len(toks)))(*toks)
        return L.tce_llama_decode_span_host(model.h, slot, pos0, len(toks), arr, None, None)

    assert span(0, 0, []) == -1
    assert span(0, 0, [1] * 9) == -1
    assert span(0, 60, [1] * 5) == -1
    assert span(0, -1, [1]) == -1
    assert span(2, 0, [1]) == -1
    assert span(0, 0, [1, V]) == -1
    assert span(0, 0, [-1]) == -1
    assert L.tce_llama_decode_span_host(model.h, 0, 0, 1, None, None, None) == -1

    def look(first=1, pos0=0, n_predict=4, hist=(), corpus=(), md=3, ng=(1, 2), temp=0.0, n_out=True, out=True, nh=None, nc=None):
        cfg = _lib.Sampling(40, 0.95, temp, 1.1, 0.0, 0.0, 64, 0)
        lk = _lib.Lookup(md, ng[0], ng[1])
        h = (C.c_int * max(1, len(hist)))(*hist)
        c = (C.c_int * max(1, len(corpus)))(*corpus)
        o = (C.c_int * 8)()
        n = C.c_int(0)
        st = _lib.LookupStats()
        return L.tce_llama_generate_lookup(model.h, first, pos0, n_predict, C.byref(cfg), h, len(hist) if nh is None else nh, c,
                                           len(corpus) if nc is None else nc, C.byref(lk), -1, o if out else None, C.byref(n) if n_out else None,
                                           C.byref(st))

    assert look(md=-1) == -1 and look(md=8) == -1
    assert look(ng=(0, 2)) == -1 and look(ng=(3, 2)) == -1
    assert look(n_predict=-1) == -1 and look(nh=-1) == -1 and look(nc=-1) == -1
    assert look(n_out=False) == -1 and look(out=False) == -1
    assert look(first=V) == -1 and look(pos0=64) == -1
    assert look(temp=0.8) == -2
    _assert_untouched(before, _snap(model, 2))
    _close(model, ctx)
