"""Speculative decoding at temp > 0: the acceptance rule on the device (tce_spec_accept) against its numpy statement (tests/spec_rule.py),
and the sampled prompt-lookup loop (tce_llama_sample_lookup, LlamaModel.generate_lookup(temp > 0)) against generate, a host replay and the
sampled distribution."""
import ctypes as C

import numpy as np
import pytest
import torch
from scipy.stats import chisquare

from spec_rule import accept_from_chains, window
from test_gpu_spec_decode import PEN, _assert_untouched, _close, _fill, _model, _snap, draft

pytestmark = pytest.mark.gpu

SEEDS = 200


def _chain(ctx, row_dev, win, cfg):
    """the device chain's (ids, probs) of one logits row under a penalty window (tce_sample's candidate output)"""
    _, ids, probs = ctx.sample(row_dev.clone(), win, candidates=True, **cfg)
    return ids, probs


# ---------------------------------------------------------------------------------------------------------------- the rule alone
@pytest.mark.parametrize("V", [64, 2048, 128256])
def test_spec_accept_matches_rule(V):
    """ids, count, accepted, stop and q bit for bit against the numpy rule over the device chain's own probabilities, for every top_k, top_p
    and temp, penalties on and off, drafts that are the top candidate, a lower one, a repeat or no candidate, eos among the drafts and
    budgets below the row count"""
    from tinychatengine_b200.runtime import Context

    ctx = Context(0)
    dev = torch.device("cuda", 0)
    case = 0
    for top_k in (1, 40, 1024):
        for top_p in (0.9, 1.0):
            for temp in (0.0, 0.2, 0.7, 1.5):
                case += 1
                rng = np.random.default_rng(1000 * case + V)
                rows = 1 + case % 8
                d = rows - 1
                pen = PEN if case % 2 else dict(repeat_penalty=1.0, frequency_penalty=0.0, presence_penalty=0.0, repeat_last_n=16)
                cfg = dict(top_k=top_k, top_p=top_p, temp=temp, **pen)
                lg = rng.standard_normal((rows, V)).astype(np.float32)
                peak = rng.integers(0, V, rows)
                lg[np.arange(rows), peak] += rng.uniform(1.0, 6.0, rows).astype(np.float32)  # a leader of varying weight in every row
                base = torch.from_numpy(lg).to(dev)
                seq = [int(t) for t in rng.integers(0, min(V, 50), 10)]
                drafts, chains = [], []
                for j in range(rows):
                    chains.append(_chain(ctx, base[j], window(seq, drafts, j, pen["repeat_last_n"]), cfg))
                    if j == d:
                        break
                    ids = chains[j][0]
                    kind = rng.integers(0, 5)
                    if kind <= 1:
                        drafts.append(int(ids[0]))
                    elif kind == 2:
                        drafts.append(int(ids[min(1, ids.size - 1)]))
                    elif kind == 3:
                        drafts.append(drafts[-1] if drafts else int(ids[-1]))
                    else:
                        drafts.append(next((t for t in range(V) if t not in set(ids.tolist())), int(ids[-1])))
                eos = drafts[1] if case % 4 == 1 and d > 1 else -1
                budget = 2 if case % 3 == 2 else rows
                for seed in range(SEEDS):
                    s = int(rng.integers(0, 2**63)) if seed else 0
                    h = len(seq) + seed
                    got = ctx.spec_accept(base.clone(), drafts, seq, seed=s, draw_index=h, eos_id=eos, budget=budget, **cfg)
                    want = accept_from_chains(chains, drafts, s, h, eos, budget)
                    assert got[:3] == want[:3], (V, cfg, drafts, seed, got, want)
                    assert np.array_equal(got[3].view(np.uint32), want[3].view(np.uint32)), (V, cfg, seed, got[3], want[3])
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- the sampled loop
def _prompt_model(geom, monkeypatch, max_ctx=256, n_slots=1, n=16):
    ctx, model = _model(geom, max_ctx, n_slots=n_slots, monkeypatch=monkeypatch)
    V = model.geom.vocab_size
    prompt = [(11 * i + 1) % V for i in range(n)]
    model.prefill(prompt[:-1], 0)
    return ctx, model, prompt[-1], len(prompt) - 1, prompt[:-1]


@pytest.mark.parametrize("geom", ["tiny-gqa", "tiny-mha"])
def test_max_draft_zero_is_generate(geom, monkeypatch):
    ctx, model, first, pos0, hist = _prompt_model(geom, monkeypatch)
    for temp, top_k, top_p in ((0.2, 40, 0.95), (0.7, 40, 0.9), (1.5, 100, 1.0)):
        for seed in (0, 1, 987654321):
            kw = dict(temp=temp, top_k=top_k, top_p=top_p, seed=seed, **PEN)
            G = model.generate(first, pos0, 40, history=hist, **kw)
            ids, st = model.generate_lookup(first, pos0, 40, history=hist, max_draft=0, **kw)
            assert ids == G, (temp, seed)
            assert st == {"steps": len(G), "drafted": 0, "accepted": 0}
    _close(model, ctx)


def replay(model, first, pos0, n_predict, history, corpus, max_draft, ngram, cfg, seed):
    """the sampled loop on the host: each step's logits through decode_host / decode_span, the device chain of every row, then the rule"""
    V = model.geom.vocab_size
    n_predict = min(n_predict, model.max_ctx - pos0)
    S = list(corpus) + list(history) + [first]
    seq = list(history)
    ids, pos, last = [], pos0, first
    st = {"steps": 0, "drafted": 0, "accepted": 0}
    while len(ids) < n_predict:
        left = n_predict - len(ids)
        dr = draft(S, max_draft, ngram, min(left - 1, model.max_ctx - pos - 1))
        d = len(dr)
        lg = torch.empty((d + 1, V), dtype=torch.float32).pin_memory()
        if d == 0:
            model.decode_host(last, pos, lg[0])
        else:
            model.decode_span([last] + dr, pos, 0, lg)
        lgd = lg.cuda()
        chains = [_chain(model.ctx, lgd[j], window(seq, dr, j, cfg["repeat_last_n"]), cfg) for j in range(d + 1)]
        out, acc, stop, _ = accept_from_chains(chains, dr, seed, len(seq), -1, left)
        st["steps"] += 1
        st["drafted"] += d
        st["accepted"] += acc
        ids += out
        S += out
        seq += out
        pos += len(out)
        last = out[-1]
    return ids, st


@pytest.mark.parametrize("geom", ["tiny-gqa", "tiny-mha"])
def test_sampled_loop_matches_host_replay(geom, monkeypatch):
    ctx, model = _model(geom, 256, n_slots=1, monkeypatch=monkeypatch)
    V = model.geom.vocab_size
    prompt = [(7 * i + 3) % V for i in range(20)]
    prompt = prompt + prompt[:12]
    model.prefill(prompt[:-1], 0)
    first, pos0, hist = prompt[-1], len(prompt) - 1, prompt[:-1]
    seed = 4242
    # the random weights give flat distributions, where drafts are seldom accepted: lower the temperature until some are, so that the
    # replay also covers steps that emit several ids
    for temp in (0.2, 0.05, 0.01):
        cfg = dict(temp=temp, top_k=40, top_p=0.9, **PEN)
        G = model.generate(first, pos0, 40, history=hist, seed=seed, **cfg)
        corpus = [first] + G[:25]
        accepted = 0
        for max_draft, ngram in ((7, (1, 3)), (3, (2, 2)), (7, (1, 1))):
            ids, st = model.generate_lookup(first, pos0, 40, history=hist, corpus=corpus, max_draft=max_draft, ngram=ngram, seed=seed, **cfg)
            assert (ids, st) == replay(model, first, pos0, 40, hist, corpus, max_draft, ngram, cfg, seed), (temp, max_draft, ngram)
            accepted += st["accepted"]
        if accepted > 0:
            break
    assert accepted > 0
    for budget in range(1, 41):
        got = model.generate_lookup(first, pos0, budget, history=hist, corpus=corpus, seed=seed, **cfg)
        assert got == replay(model, first, pos0, budget, hist, corpus, 7, (1, 3), cfg, seed), budget
    _close(model, ctx)


def test_sample_lookup_at_temp_zero_is_the_greedy_loop(monkeypatch):
    from tinychatengine_b200 import _lib

    ctx, model, first, pos0, hist = _prompt_model("tiny-gqa", monkeypatch)
    G, _ = model.generate_lookup(first, pos0, 48, history=hist, max_draft=0, **PEN)
    for corpus in ([], [first] + G):
        want = model.generate_lookup(first, pos0, 48, history=hist, corpus=corpus, **PEN)
        cfg = _lib.Sampling(40, 0.95, 0.0, PEN["repeat_penalty"], PEN["frequency_penalty"], PEN["presence_penalty"], PEN["repeat_last_n"], 99)
        lk = _lib.Lookup(7, 1, 3)
        h = (C.c_int * len(hist))(*hist)
        c = (C.c_int * max(1, len(corpus)))(*corpus)
        o = (C.c_int * 48)()
        n = C.c_int(0)
        st = _lib.LookupStats()
        assert ctx.L.tce_llama_sample_lookup(model.h, first, pos0, 48, C.byref(cfg), h, len(hist), c, len(corpus), C.byref(lk), -1, o, C.byref(n),
                                             C.byref(st)) == 0
        assert (list(o[:n.value]), {"steps": st.steps, "drafted": st.drafted, "accepted": st.accepted}) == want
    _close(model, ctx)


def test_first_id_has_the_sampled_distribution(monkeypatch):
    """a first-step draft with q near 0.5: over 2000 seeds the first emitted id follows p_0 (chi-square), whether the draft was accepted or
    replaced"""
    ctx, model = _model("tiny-gqa", 64, n_slots=1, monkeypatch=monkeypatch)
    V = model.geom.vocab_size
    first = 5
    lg = torch.empty(V, dtype=torch.float32).pin_memory()
    model.decode_host(first, 0, lg)
    best = None
    for temp in (0.02, 0.05, 0.1, 0.2, 0.3, 0.5, 0.7, 1.0, 1.5):
        cfg = dict(temp=temp, top_k=40, top_p=1.0, **PEN)
        ids, probs = _chain(ctx, lg.cuda(), window([], [], 0, PEN["repeat_last_n"]), cfg)
        if best is None or abs(probs[0] - 0.5) < abs(best[1][1][0] - 0.5):
            best = (cfg, (ids, probs))
    cfg, (ids, probs) = best
    assert 0.2 < probs[0] < 0.8, probs[:4]
    X = int(ids[0])
    counts = {}
    n_seeds = 2000
    accepted = 0
    for seed in range(n_seeds):
        out, st = model.generate_lookup(first, 0, 2, corpus=[first, X], max_draft=1, seed=seed, **cfg)
        assert st["drafted"] >= 1
        accepted += st["accepted"] > 0
        counts[out[0]] = counts.get(out[0], 0) + 1
    p = {int(t): float(q) for t, q in zip(ids, probs)}
    assert set(counts) <= set(p)
    keys = [t for t in p if p[t] * n_seeds >= 5]
    obs = [counts.get(t, 0) for t in keys] + [n_seeds - sum(counts.get(t, 0) for t in keys)]
    exp = [p[t] * n_seeds for t in keys] + [n_seeds * (1 - sum(p[t] for t in keys))]
    if exp[-1] < 1e-9:
        obs, exp = obs[:-1], exp[:-1]
    exp = np.array(exp) * (n_seeds / sum(exp))
    assert chisquare(obs, exp).pvalue > 1e-3, (obs, exp)
    assert 0 < accepted < n_seeds
    _close(model, ctx)


@pytest.mark.parametrize("geom", ["tiny-gqa", "tiny-mha"])
def test_acceptance_happens(geom, monkeypatch):
    ctx, model, first, pos0, hist = _prompt_model(geom, monkeypatch)
    cfg = dict(temp=0.2, top_k=40, top_p=0.9, seed=31, **PEN)
    G = model.generate(first, pos0, 48, history=hist, **cfg)
    ids, st = model.generate_lookup(first, pos0, 48, history=hist, corpus=[first] + G, **cfg)
    assert len(ids) == 48
    assert st["accepted"] > 0 and st["steps"] < len(ids), st
    assert len(ids) == st["accepted"] + st["steps"]
    _close(model, ctx)


def test_row_contract_and_refusals(monkeypatch):
    from tinychatengine_b200 import _lib

    ctx, model = _model("tiny-gqa", 128, n_slots=2, monkeypatch=monkeypatch)
    V = model.geom.vocab_size
    prompt = [(5 * i + 2) % V for i in range(12)]
    first, pos0, hist = prompt[-1], len(prompt) - 1, prompt[:-1]
    cfg = dict(temp=0.7, top_k=40, top_p=0.9, seed=3, **PEN)
    _fill(model, 2, 3)
    model.prefill(prompt[:-1], 0)
    G = model.generate(first, pos0, 40, history=hist, **cfg)
    model.prefill(prompt[:-1], 0)
    before = _snap(model, 2)
    ids, st = model.generate_lookup(first, pos0, 17, history=hist, corpus=[first] + G, max_draft=5, **cfg)
    after = _snap(model, 2)
    assert len(ids) == 17 and st["drafted"] > 0
    _assert_untouched(before, after, 0, pos0, pos0 + len(ids) + 5)
    # a start three rows before max_ctx stops there, having written rows 125..127 of slot 0 only
    before = after
    ids, st = model.generate_lookup(first, 125, 40, history=hist, corpus=[first] + G, **cfg)
    assert len(ids) == 3
    _assert_untouched(before, _snap(model, 2), 0, 125, 128)

    before = _snap(model, 2)

    def look(top_k=40, temp=0.7, md=3, ng=(1, 2), n_predict=4, first=1, pos0=0, n_out=True):
        c = _lib.Sampling(top_k, 0.95, temp, 1.1, 0.0, 0.0, 64, 0)
        lk = _lib.Lookup(md, ng[0], ng[1])
        o = (C.c_int * 8)()
        n = C.c_int(0)
        st = _lib.LookupStats()
        return ctx.L.tce_llama_sample_lookup(model.h, first, pos0, n_predict, C.byref(c), None, 0, None, 0, C.byref(lk), -1, o,
                                             C.byref(n) if n_out else None, C.byref(st))

    assert look(top_k=0) == -2 and look(top_k=1025) == -2
    assert look(md=8) == -1 and look(ng=(0, 2)) == -1 and look(n_predict=-1) == -1 and look(first=V) == -1 and look(pos0=128) == -1
    assert look(n_out=False) == -1
    _assert_untouched(before, _snap(model, 2))
    # tce_spec_accept: the chain's limits and bad arguments
    lg = torch.zeros((2, 2048), dtype=torch.float32, device="cuda")
    with pytest.raises(_lib.TceError, match=r"\(-2\)"):
        ctx.spec_accept(lg, [1], top_k=0, temp=0.7)
    with pytest.raises(_lib.TceError, match=r"\(-1\)"):
        ctx.spec_accept(lg, [1], budget=0)
    _close(model, ctx)
