"""Attention inside the persistent decode kernel at single positions on a random-filled cache: with one attention split per KV head
(every visible key in one CTA) and with several (flash-decode partials merged across CTAs), the token's key and value landing at
the start, inside and at the end of a 64-key chunk."""
import numpy as np
import pytest
import torch

from helpers import oracle_decode_step, rel_err

pytestmark = pytest.mark.gpu

# tiny-gqa (2 KV heads) and tiny-mha (4 KV heads) on an H100 give every KV head 66 / 33 CTAs: positions below 64 take one split,
# the others one split per 64-key chunk (pos 1000: 16 splits; pos 2047: 32, the most the split merge takes)
POSITIONS = [0, 37, 63, 64, 130, 1000, 2047]


@pytest.mark.parametrize("pos", POSITIONS, ids=lambda pos: f"{pos}-pair")  # "pair": the kernel runs on clusters of two CTAs
@pytest.mark.parametrize("geom", ["tiny-gqa", "tiny-mha"])
def test_persistent_attention_step_matches_oracle(geom, pos, monkeypatch):
    monkeypatch.setenv("TCE_PERSISTENT", "1")
    from tinychatengine_b200.llama import GEOMETRIES, LlamaModel
    from tinychatengine_b200.runtime import Context

    g = GEOMETRIES[geom]
    ctx = Context(0)
    model = LlamaModel(ctx, g, max_ctx=2048, seed=13, random_zeros=True)
    assert model.kernels_per_step == 1
    gen = torch.Generator(device="cuda")
    gen.manual_seed(pos + 7)
    past_k, past_v = [], []
    for l in range(g.num_layers):
        for which, store in ((0, past_k), (1, past_v)):
            c = model.kv_cache(l, which)
            c.copy_((torch.randn(c.shape, device="cuda", generator=gen) * 0.5).to(torch.float16))
            store.append(c[:, :pos].float().cpu().numpy() if pos else None)
    lg = torch.empty(g.vocab_size, dtype=torch.float32).pin_memory()
    nxt = model.decode_host(321, pos, lg)
    want, fk, fv = oracle_decode_step(model, 321, pos, past_k, past_v)
    got = lg.numpy()
    assert np.all(np.isfinite(got))
    e = rel_err(got, want)
    assert e <= 1e-2, (pos, e)
    assert nxt == int(np.argmax(got))
    for l in range(g.num_layers):
        assert np.abs(model.kv_cache(l, 0)[:, pos].float().cpu().numpy() - fk[l][:, pos]).max() <= 2e-2 * max(1.0, np.abs(fk[l]).max())
        assert np.abs(model.kv_cache(l, 1)[:, pos].float().cpu().numpy() - fv[l][:, pos]).max() <= 5e-3 * max(1.0, np.abs(fv[l][:, pos]).max())
        # rows before the token are read, never written
        if pos:
            assert np.array_equal(model.kv_cache(l, 0)[:, :pos].float().cpu().numpy(), past_k[l])
    model.close()
    ctx.close()
