"""Prompt processing (tce_llama_prefill: wgmma GEMMs + causal flash attention) vs the oracle-composed decode steps, vs the
decode path on the same weights, and chunked against one-shot."""
import numpy as np
import pytest
import torch

from helpers import oracle_decode_step, rel_err

pytestmark = pytest.mark.gpu


def _tokens(n, vocab, seed):
    return [int(t) for t in np.random.default_rng(seed).integers(0, vocab, n)]


@pytest.mark.parametrize("geom,n", [("tiny-gqa", 70), ("tiny-mha", 33)])
def test_prefill_matches_oracle(geom, n, monkeypatch):
    from tinychatengine_b200.llama import GEOMETRIES, LlamaModel
    from tinychatengine_b200.runtime import Context

    ctx = Context(0)
    g = GEOMETRIES[geom]
    model = LlamaModel(ctx, g, max_ctx=128, seed=11, random_zeros=True)
    toks = _tokens(n, g.vocab_size, 5)
    lg = torch.empty(g.vocab_size, dtype=torch.float32).pin_memory()
    nxt = model.prefill(toks, 0, lg)
    got = lg.numpy().copy()
    past_k, past_v = [None] * g.num_layers, [None] * g.num_layers
    for pos, tok in enumerate(toks):
        want, past_k, past_v = oracle_decode_step(model, tok, pos, past_k, past_v)
    assert np.all(np.isfinite(got))
    assert rel_err(got, want) <= 1e-2, rel_err(got, want)
    assert nxt == int(np.argmax(got))
    for l in range(g.num_layers):
        kc = model.kv_cache(l, 0)[:, :n].float().cpu().numpy()
        vc = model.kv_cache(l, 1)[:, :n].float().cpu().numpy()
        assert np.abs(kc - past_k[l]).max() <= 2e-2 * max(1.0, np.abs(past_k[l]).max())
        assert np.abs(vc - past_v[l]).max() <= 2e-2 * max(1.0, np.abs(past_v[l]).max())
    model.close()
    ctx.close()


def test_prefill_then_decode_agrees_with_decode_only(monkeypatch):
    from tinychatengine_b200.llama import GEOMETRIES, LlamaModel
    from tinychatengine_b200.runtime import Context

    g = GEOMETRIES["tiny-gqa"]
    toks = _tokens(45, g.vocab_size, 9)
    outs = []
    for use_prefill in (True, False):
        ctx = Context(0)
        model = LlamaModel(ctx, g, max_ctx=128, seed=4, random_zeros=True)
        lg = torch.empty(g.vocab_size, dtype=torch.float32).pin_memory()
        seq = []
        if use_prefill:
            model.prefill(toks[:40], 0, lg)
            seq.append(lg.clone())
            start = 40
        else:
            for pos in range(40):
                model.decode_host(toks[pos], pos, lg)
            seq.append(lg.clone())
            start = 40
        for pos in range(start, 45):
            model.decode_host(toks[pos], pos, lg)
            seq.append(lg.clone())
        outs.append(torch.stack(seq).numpy())
        model.close()
        ctx.close()
    for a, b in zip(outs[0], outs[1]):
        assert rel_err(a, b) <= 1e-2, rel_err(a, b)


def test_chunked_prefill_equals_one_shot(monkeypatch):
    from tinychatengine_b200.llama import GEOMETRIES, LlamaModel
    from tinychatengine_b200.runtime import Context

    g = GEOMETRIES["tiny-gqa"]
    toks = _tokens(100, g.vocab_size, 2)
    ctx = Context(0)
    model = LlamaModel(ctx, g, max_ctx=128, seed=6)
    lg1 = torch.empty(g.vocab_size, dtype=torch.float32).pin_memory()
    lg2 = torch.empty_like(lg1).pin_memory()
    n1 = model.prefill(toks, 0, lg1)
    k1 = model.kv_cache(1, 0)[:, :100].clone()
    model.prefill(toks[:37], 0, None)
    n2 = model.prefill(toks[37:], 37, lg2)
    k2 = model.kv_cache(1, 0)[:, :100].clone()
    assert rel_err(lg2.numpy(), lg1.numpy()) <= 1e-3
    assert n1 == n2
    assert (k1.float() - k2.float()).abs().max().item() <= 1e-2
    # argument checking: past the end of the cache, bad token id
    from tinychatengine_b200 import _lib

    with pytest.raises(_lib.TceError):
        model.prefill(toks, 60, None)
    with pytest.raises(_lib.TceError):
        model.prefill([g.vocab_size], 0, None)
    model.close()
    ctx.close()
