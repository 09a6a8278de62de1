"""Batched generation: the ragged prompt pass (tce_llama_prefill_batch: several prompts, one pass over the weights) and the batched device
generate loop (tce_llama_generate_batch: one batched step + one sampler launch per token), against the oracle, against one prompt per call,
and against a host replay of the batched step through the oracle sampler."""
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import oracle_decode_step, rel_err
from oracle import sampling

pytestmark = pytest.mark.gpu


def _model(geom, max_ctx, n_slots, seed=7):
    from tinychatengine_b200.llama import GEOMETRIES, LlamaModel
    from tinychatengine_b200.runtime import Context

    ctx = Context(0)
    model = LlamaModel(ctx, GEOMETRIES[geom] if isinstance(geom, str) else geom, max_ctx=max_ctx, seed=seed, random_zeros=True)
    model.reserve_slots(n_slots)
    return ctx, model


def _fill_caches(model, n_slots, seed):
    gen = torch.Generator(device="cuda")
    gen.manual_seed(seed)
    for s in range(n_slots):
        for l in range(model.geom.num_layers):
            for w in (0, 1):
                c = model.kv_cache(l, w, s)
                c.copy_((torch.randn(c.shape, device="cuda", generator=gen) * 0.5).to(torch.float16))


def _snapshot(model, n_slots):
    return [[[model.kv_cache(l, w, s).cpu().clone() for w in (0, 1)] for l in range(model.geom.num_layers)] for s in range(n_slots)]


def _restore(model, snap):
    for s, layers in enumerate(snap):
        for l, kv in enumerate(layers):
            for w in (0, 1):
                model.kv_cache(l, w, s).copy_(kv[w].cuda())


def _check_rows(before, after, written):
    """written: slot -> (first row, count).  Those rows changed, every other row of every slot is byte-identical."""
    for s in range(len(before)):
        for l in range(len(before[s])):
            for w in (0, 1):
                a, b = before[s][l][w].clone(), after[s][l][w].clone()
                if s in written:
                    r0, n = written[s]
                    if n:
                        assert not torch.equal(a[:, r0:r0 + n], b[:, r0:r0 + n]), (s, l, w)
                    a[:, r0:r0 + n] = 0
                    b[:, r0:r0 + n] = 0
                assert torch.equal(a, b), (s, l, w)


def _tokens(n, vocab, seed):
    return [int(t) for t in np.random.default_rng(seed).integers(0, vocab, n)]


# ------------------------------------------------------------------------------------------------ ragged prompt pass

@pytest.mark.parametrize("geom", ["tiny-gqa", "tiny-mha"])
def test_ragged_prefill_matches_oracle(geom):
    """Prompts of 70, 1, 33, 64 and 65 tokens into out-of-order slots, plus one that continues slot 3 at position 40, in one pass: each
    prompt's logits against its oracle chain, its K/V rows against the oracle, and every other cache row untouched."""
    ctx, model = _model(geom, 256, 8)
    g = model.geom
    _fill_caches(model, 8, 21)
    before = _snapshot(model, 8)
    lengths, pos0s, slots = [70, 1, 33, 64, 65, 20], [0, 0, 0, 0, 0, 40], [5, 0, 7, 2, 1, 3]
    prompts = [_tokens(n, g.vocab_size, 100 + i) for i, n in enumerate(lengths)]
    lg = torch.empty((len(prompts), g.vocab_size), dtype=torch.float32).pin_memory()
    nxt = model.prefill_batch(prompts, slots, pos0s, lg)
    after = _snapshot(model, 8)
    for b, (prompt, p0, slot) in enumerate(zip(prompts, pos0s, slots)):
        if p0 == 0:
            pk, pv = [None] * g.num_layers, [None] * g.num_layers
        else:
            pk = [before[slot][l][0][:, :p0].float().numpy() for l in range(g.num_layers)]
            pv = [before[slot][l][1][:, :p0].float().numpy() for l in range(g.num_layers)]
        for i, tok in enumerate(prompt):
            want, pk, pv = oracle_decode_step(model, tok, p0 + i, pk, pv)
        got = lg[b].numpy()
        assert np.all(np.isfinite(got))
        assert rel_err(got, want) <= 1e-2, (b, rel_err(got, want))
        assert nxt[b] == int(np.argmax(got))
        rows = slice(p0, p0 + len(prompt))
        for l in range(g.num_layers):
            kc = after[slot][l][0][:, rows].float().numpy()
            vc = after[slot][l][1][:, rows].float().numpy()
            assert np.abs(kc - pk[l][:, rows]).max() <= 2e-2 * max(1.0, np.abs(pk[l]).max()), (b, l)
            assert np.abs(vc - pv[l][:, rows]).max() <= 2e-2 * max(1.0, np.abs(pv[l]).max()), (b, l)
    _check_rows(before, after, {s: (p0, len(p)) for p, p0, s in zip(prompts, pos0s, slots)})
    model.close()
    ctx.close()


def test_ragged_prefill_equals_one_prompt_per_call():
    """Llama-3-8B widths (2 layers, max_ctx 4096), 8 prompts: the ragged pass writes the same K/V bits as one prefill_slot call per prompt
    (GEMM rows are independent, attention is per row and its query blocks never straddle two prompts); the logits come from the
    multi-column lm_head GEMV instead of the M = 1 one, so they agree to rounding."""
    from tinychatengine_b200.llama import GEOMETRIES, LlamaGeometry

    b = GEOMETRIES["llama3-8b"]
    g = LlamaGeometry("llama3-8b-2l", 2, b.num_heads, b.num_kv_heads, b.embed_dim, b.hidden_dim, b.vocab_size, b.rms_eps, b.rope_theta, b.head_dim)
    ctx, model = _model(g, 4096, 16, seed=5)
    lengths = [300, 17, 129, 64, 1, 250, 96, 200]
    pos0s = [0, 100, 0, 3000, 4095, 0, 512, 3896]
    prompts = [_tokens(n, g.vocab_size, 7 + i) for i, n in enumerate(lengths)]
    lg = torch.empty((8, g.vocab_size), dtype=torch.float32).pin_memory()
    nxt = model.prefill_batch(prompts, list(range(8)), pos0s, lg)
    one = torch.empty(g.vocab_size, dtype=torch.float32).pin_memory()
    for i in range(8):
        model.prefill(prompts[i], pos0s[i], one, slot=8 + i)
        assert rel_err(lg[i].numpy(), one.numpy()) <= 2e-3, (i, rel_err(lg[i].numpy(), one.numpy()))
        assert nxt[i] == int(np.argmax(lg[i].numpy()))
        for l in range(g.num_layers):
            for w in (0, 1):
                assert torch.equal(model.kv_cache(l, w, i), model.kv_cache(l, w, 8 + i)), (i, l, w)
    model.close()
    ctx.close()


def test_prefill_batch_refusals():
    """Every host-side refusal raises TCE_ERR_INVALID before anything is enqueued: all caches stay byte-identical."""
    ctx, model = _model("tiny-gqa", 128, 3)
    g = model.geom
    _fill_caches(model, 3, 4)
    before = _snapshot(model, 3)
    L = ctx.L

    def call(prompts, slots, pos0s):
        arr = lambda v: (C.c_int * max(1, len(v)))(*[int(x) for x in v])
        flat = [t for p in prompts for t in p]
        return L.tce_llama_prefill_batch(model.h, len(prompts), arr(flat), arr([len(p) for p in prompts]), arr(pos0s), arr(slots), None, None)

    bad = [
        ([], [], []),                                      # no prompt
        ([[1]] * 9, list(range(9)), [0] * 9),              # 9 prompts
        ([[1, 2], []], [0, 1], [0, 0]),                    # an empty prompt
        ([[1, 2], [3] * 10], [0, 1], [0, 120]),            # past the end of the cache
        ([[1, 2], [3]], [0, 1], [0, -1]),                  # pos0 < 0
        ([[1, 2], [3]], [0, 3], [0, 0]),                   # slot not reserved
        ([[1, 2], [3]], [1, 1], [0, 0]),                   # the same slot twice
        ([[1, 2], [3]], [0, -1], [0, 0]),                  # slot < 0
        ([[1, 2], [g.vocab_size]], [0, 1], [0, 0]),        # token >= vocab
        ([[1, -2], [3]], [0, 1], [0, 0]),                  # token < 0
    ]
    for prompts, slots, pos0s in bad:
        assert call(prompts, slots, pos0s) == -1, (prompts, slots, pos0s)
        torch.cuda.synchronize()
        after = _snapshot(model, 3)
        _check_rows(before, after, {})
    assert L.tce_llama_prefill_batch(model.h, 1, None, None, None, None, None, None) == -1
    model.close()
    ctx.close()


# ------------------------------------------------------------------------------------------------ batched generate loop

ROWS = [  # mixed positions, budgets, seeds and chains
    dict(first_token=5, pos0=0, slot=3, n_predict=20, temp=0.0, repeat_penalty=1.0),
    dict(first_token=77, pos0=10, slot=0, n_predict=24, history=[77], top_k=40, top_p=0.9, temp=0.9, repeat_penalty=1.2, frequency_penalty=0.1,
         presence_penalty=0.05, repeat_last_n=16, seed=77),
    dict(first_token=1000, pos0=50, slot=6, n_predict=17, history=[3, 9, 1000, 9], top_k=5, top_p=1.0, temp=1.3, repeat_penalty=1.0,
         repeat_last_n=-1, seed=5),
    dict(first_token=2, pos0=100, slot=1, n_predict=28, top_k=100, top_p=0.5, temp=0.7, seed=123),
    dict(first_token=2047, pos0=3, slot=7, n_predict=9, history=[2047, 2047], top_k=1, temp=0.5, repeat_penalty=1.5, repeat_last_n=4, seed=9),
]
DEFAULTS = dict(history=(), eos_id=-1, top_k=40, top_p=0.95, temp=0.8, repeat_penalty=1.1, frequency_penalty=0.0, presence_penalty=0.0,
                repeat_last_n=64, seed=0)


def _replay(model, reqs, outs, max_ctx):
    """Host replay of the generate loop: decode_batch_host logits of every row (batch size kept, finished rows ride along) through the oracle
    sampler, with the history window of the device ring and the draw index = history head.  Follows the device at a bin edge."""
    V = model.geom.vocab_size
    rq = [{**DEFAULTS, **r} for r in reqs]
    hist = [list(r["history"]) for r in rq]
    tok = [r["first_token"] for r in rq]
    replay = [[] for _ in rq]
    steps = max(len(o) for o in outs)
    lg = torch.empty((len(rq), V), dtype=torch.float32).pin_memory()
    for i in range(steps):
        live = [i < len(outs[b]) for b in range(len(rq))]
        pos = [min(r["pos0"] + i, max_ctx - 1) for r in rq]
        model.decode_batch_host([t if lv else 1 for t, lv in zip(tok, live)], pos, [r["slot"] for r in rq], lg)
        for b, r in enumerate(rq):
            if not live[b]:
                continue
            W = max_ctx if r["repeat_last_n"] < 0 else min(r["repeat_last_n"], max_ctx)
            window = ([0] * W + hist[b])[-W:] if W else []
            ids, probs = sampling.candidates(lg[b].numpy(), window, top_k=r["top_k"], top_p=r["top_p"], temp=r["temp"],
                                             repeat_penalty=r["repeat_penalty"], frequency_penalty=r["frequency_penalty"],
                                             presence_penalty=r["presence_penalty"])
            u = sampling.uniform01(r["seed"], len(hist[b]))
            t = sampling.draw(ids, probs, u)
            cdf = np.cumsum(probs.astype(np.float64))
            if r["temp"] > 0 and np.min(np.abs(cdf - u)) < 1e-4 and outs[b][i] != t:
                t = outs[b][i]  # bin edge: follow the device so that the rest of the sequence stays comparable
            replay[b].append(t)
            hist[b].append(t)
            tok[b] = t
    return replay


def test_generate_batch_matches_host_replay(monkeypatch):
    monkeypatch.setenv("TCE_DETERMINISTIC", "1")
    ctx, model = _model("tiny-gqa", 128, 8, seed=3)
    _fill_caches(model, 8, 12)
    before = _snapshot(model, 8)
    outs = model.generate_batch(ROWS)
    after = _snapshot(model, 8)
    assert [len(o) for o in outs] == [r["n_predict"] for r in ROWS]
    _check_rows(before, after, {r["slot"]: (r["pos0"], len(o)) for r, o in zip(ROWS, outs)})
    _restore(model, before)
    replay = _replay(model, ROWS, outs, 128)
    for b in range(len(ROWS)):
        assert outs[b] == replay[b], (b, outs[b], replay[b])
    model.close()
    ctx.close()


def test_generate_batch_stopping(monkeypatch):
    """EOS ends its own row only; a row near the end of the cache stops there; a row with no budget writes nothing.  Slot s gains exactly
    n_out rows at pos0 .. pos0 + n_out - 1."""
    monkeypatch.setenv("TCE_DETERMINISTIC", "1")
    ctx, model = _model("tiny-gqa", 128, 5, seed=4)
    _fill_caches(model, 5, 13)
    orig = _snapshot(model, 5)
    base = [dict(first_token=11, pos0=5, slot=2, n_predict=30, seed=1, top_k=20),
            dict(first_token=12, pos0=0, slot=0, n_predict=25, seed=2, top_k=20),
            dict(first_token=13, pos0=60, slot=4, n_predict=18, seed=3, top_k=20)]
    ref = model.generate_batch(base)
    assert [len(o) for o in ref] == [30, 25, 18]
    eos = ref[1][6]
    cut = ref[1].index(eos) + 1
    reqs = [dict(base[0]), dict(base[1], eos_id=eos), dict(base[2])]
    _restore(model, orig)
    out = model.generate_batch(reqs)
    after = _snapshot(model, 5)
    assert out[1] == ref[1][:cut]
    assert out[0] == ref[0] and out[2] == ref[2]
    _check_rows(orig, after, {2: (5, 30), 0: (0, cut), 4: (60, 18)})
    # near the end of the cache: the budget is clamped to max_ctx - pos0, and the row stops there; n_predict = 0 generates nothing
    reqs = [dict(first_token=3, pos0=125, slot=1, n_predict=10, seed=4), dict(first_token=4, pos0=20, slot=3, n_predict=0),
            dict(first_token=5, pos0=127, slot=0, n_predict=1, temp=0.0)]
    before = _snapshot(model, 5)
    out = model.generate_batch(reqs)
    after = _snapshot(model, 5)
    assert [len(o) for o in out] == [3, 0, 1]
    _check_rows(before, after, {1: (125, 3), 3: (20, 0), 0: (127, 1)})
    model.close()
    ctx.close()


def test_generate_batch_rows_are_independent(monkeypatch):
    monkeypatch.setenv("TCE_DETERMINISTIC", "1")
    ctx, model = _model("tiny-gqa", 128, 8, seed=6)
    _fill_caches(model, 8, 14)
    ref = model.generate_batch(ROWS)
    perm = [3, 0, 4, 2, 1]
    got = model.generate_batch([ROWS[i] for i in perm])
    assert got == [ref[i] for i in perm]
    # row 1 next to other requests (other slots, positions, chains, budgets)
    other = [dict(first_token=9, pos0=7, slot=2, n_predict=40, seed=8, top_k=3), ROWS[1], dict(first_token=8, pos0=90, slot=4, n_predict=2),
             dict(ROWS[0], slot=5, pos0=30), dict(first_token=4, pos0=0, slot=6, n_predict=30, temp=0.0)]
    assert model.generate_batch(other)[1] == ref[1]
    model.close()
    ctx.close()


def test_generate_batch_greedy_equals_step_chain():
    """temp = 0, no penalties: the ids are the chain of the batched step's own arg-max (default, non-deterministic residual adds)."""
    ctx, model = _model("tiny-mha", 128, 4, seed=8)
    _fill_caches(model, 4, 15)
    before = _snapshot(model, 4)
    reqs = [dict(first_token=t, pos0=p, slot=s, n_predict=12, temp=0.0, repeat_penalty=1.0) for t, p, s in [(1, 0, 2), (500, 40, 0), (77, 9, 3)]]
    outs = model.generate_batch(reqs)
    _restore(model, before)
    tok, chain = [r["first_token"] for r in reqs], [[], [], []]
    for i in range(12):
        tok = model.decode_batch_host(tok, [r["pos0"] + i for r in reqs], [r["slot"] for r in reqs])
        for b in range(3):
            chain[b].append(tok[b])
    assert outs == chain
    model.close()
    ctx.close()


def test_generate_batch_refusals():
    """Every host-side refusal returns before anything is enqueued (caches byte-identical): TCE_ERR_INVALID for bad requests, TCE_ERR_UNSUPPORTED
    for temp > 0 without 1 <= top_k <= 1024."""
    from tinychatengine_b200 import _lib

    ctx, model = _model("tiny-gqa", 128, 3)
    g = model.geom
    _fill_caches(model, 3, 16)
    model.generate_batch([dict(first_token=1, pos0=0, slot=0, n_predict=2)])  # allocate + capture once
    before = _snapshot(model, 3)
    L = ctx.L

    def call(reqs, stride=8, out_ok=True, n_out_ok=True):
        arr = (_lib.GenRequest * max(1, len(reqs)))()
        for i, r in enumerate(reqs):
            q = {**DEFAULTS, "n_history": 0, **r}
            arr[i] = _lib.GenRequest(q["first_token"], q["pos0"], q["slot"], q["n_predict"], q["eos_id"], None, q["n_history"],
                                     _lib.Sampling(q["top_k"], q["top_p"], q["temp"], q["repeat_penalty"], 0.0, 0.0, 64, 0))
        out = (C.c_int * (8 * max(1, stride)))()
        n_out = (C.c_int * 8)()
        return L.tce_llama_generate_batch(model.h, len(reqs), arr, out if out_ok else None, stride, n_out if n_out_ok else None)

    ok = dict(first_token=1, pos0=0, slot=0, n_predict=4)
    bad = [
        [],                                                          # batch 0
        [dict(ok, slot=i % 3) for i in range(9)],                    # batch 9
        [ok, dict(ok, slot=3)],                                      # slot not reserved
        [ok, dict(ok, slot=-1)],                                     # slot < 0
        [ok, dict(ok)],                                              # the same slot twice
        [dict(ok, first_token=-1)],                                  # token < 0
        [dict(ok, first_token=g.vocab_size)],                        # token >= vocab
        [dict(ok, pos0=-1)],                                         # pos0 < 0
        [dict(ok, pos0=128)],                                        # pos0 >= max_ctx
        [dict(ok, n_predict=-1)],                                    # n_predict < 0
        [dict(ok, n_history=129)],                                   # n_history > max_ctx (and no history pointer)
        [dict(ok, n_history=2)],                                     # history pointer NULL
    ]
    for reqs in bad:
        assert call(reqs) == -1, reqs
    assert call([dict(ok, n_predict=9)], stride=8) == -1             # out_stride below n_predict
    assert call([dict(ok, pos0=124, n_predict=9)], stride=4) == 0    # ... after clamping to max_ctx - pos0 it fits
    before = _snapshot(model, 3)
    assert call([ok], out_ok=False) == -1                            # NULL output
    assert call([ok], n_out_ok=False) == -1
    assert L.tce_llama_generate_batch(model.h, 1, None, None, 8, None) == -1
    assert call([ok, dict(ok, slot=1, top_k=0)]) == -2                # whole-vocabulary sampling at temp > 0
    assert call([ok, dict(ok, slot=1, top_k=1025)]) == -2
    assert b"top_k" in L.tce_last_error()
    torch.cuda.synchronize()
    _check_rows(before, _snapshot(model, 3), {})
    with pytest.raises(_lib.TceError):
        model.generate_batch([dict(ok, slot=5)])
    model.close()
    ctx.close()


def test_tensor_parallel_model_is_unsupported():
    from tinychatengine_b200._lib import GenRequest, TceError
    from tinychatengine_b200.llama import GEOMETRIES, LlamaModel, make_random_weights, shard_weights
    from tinychatengine_b200.runtime import Context

    ctx = Context(0)
    g = GEOMETRIES["tiny-gqa"]
    W = make_random_weights(g, torch.device("cuda", 0), 3)
    Wl, gl = shard_weights(W, g, 0, 2)
    model = LlamaModel(ctx, gl, max_ctx=128, weights=Wl, tp_rank=0, tp_size=2)
    L = ctx.L
    one = (C.c_int * 1)(0)
    assert L.tce_llama_prefill_batch(model.h, 1, one, (C.c_int * 1)(1), one, one, None, None) == -2
    req = (GenRequest * 1)()
    req[0].n_predict = 1
    out = (C.c_int * 1)()
    n_out = (C.c_int * 1)()
    assert L.tce_llama_generate_batch(model.h, 1, req, out, 1, n_out) == -2
    with pytest.raises(TceError, match="tp_size"):
        model.prefill_batch([[1, 2]], [0])
    with pytest.raises(TceError, match="tp_size"):
        model.generate_batch([dict(first_token=1, pos0=0, slot=0, n_predict=1)])
    model.close()
    ctx.close()
