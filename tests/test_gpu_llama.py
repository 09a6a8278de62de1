"""Fused decode step (tce_llama_*: one persistent kernel per token, or one kernel per op inside a CUDA graph) vs the oracle-composed step."""
import dataclasses

import numpy as np
import pytest
import torch

from helpers import oracle_decode_step, rel_err

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("mega", ["1", "0"])
@pytest.mark.parametrize("geom", ["tiny-gqa", "tiny-mha", "e128"])
def test_decode_steps_match_oracle(geom, mega, monkeypatch):
    """mega=1: one persistent kernel per token (the default); mega=0: one kernel per op inside a CUDA graph.  e128 (embed_dim 128,
    one layer) has a single 128-group in q|k|v, gate|up and lm_head, nothing to split across the two CTAs of a cluster: it is outside
    the persistent kernel's envelope and runs one kernel per op either way."""
    monkeypatch.setenv("TCE_PERSISTENT", mega)
    from tinychatengine_b200.llama import GEOMETRIES, LlamaModel
    from tinychatengine_b200.runtime import Context

    ctx = Context(0)
    if geom == "e128":
        g = dataclasses.replace(GEOMETRIES["tiny-gqa"], name="e128", num_layers=1, num_heads=1, num_kv_heads=1, embed_dim=128, hidden_dim=384)
    else:
        g = GEOMETRIES[geom]
    model = LlamaModel(ctx, g, max_ctx=256, seed=7, random_zeros=True)
    assert (model.kernels_per_step == 1) == (mega == "1" and geom != "e128")
    past_k = [None] * g.num_layers
    past_v = [None] * g.num_layers
    tokens = [3, 77, 1000, 5, 900, 17, 256, 999]
    logits_host = torch.empty(g.vocab_size, dtype=torch.float32).pin_memory()
    for pos, tok in enumerate(tokens):
        nxt = model.decode_host(tok, pos, logits_host)
        want, past_k, past_v = oracle_decode_step(model, tok, pos, past_k, past_v)
        got = logits_host.numpy().copy()
        assert np.all(np.isfinite(got))
        assert rel_err(got, want) <= 1e-2, (geom, pos, rel_err(got, want))
        assert nxt == int(np.argmax(got))
        # device-resident entry point gives the same logits as the host entry point
        tp = torch.tensor([tok, pos], dtype=torch.int32, device="cuda")
        model.decode(tp)
        torch.cuda.synchronize()
        # (o_proj / down_proj split tiles accumulate with RED.ADD by default: last-bit differences are expected)
        assert rel_err(model.logits().cpu().numpy(), got) <= 2e-3
        for l in range(g.num_layers):
            kc = model.kv_cache(l, 0)[:, : pos + 1].float().cpu().numpy()
            assert np.abs(kc - past_k[l]).max() <= 2e-2 * max(1.0, np.abs(past_k[l]).max())
    model.close()
    ctx.close()


def test_graph_and_eager_paths_agree(monkeypatch):
    import os

    monkeypatch.setenv("TCE_DETERMINISTIC", "1")  # ordered stream-K fix-up instead of RED.ADD: bit-reproducible
    monkeypatch.setenv("TCE_PERSISTENT", "0")

    from tinychatengine_b200.llama import GEOMETRIES, LlamaModel
    from tinychatengine_b200.runtime import Context

    outs = []
    for pdl in (1, 0):
        ctx = Context(0)
        ctx.set_option("use_pdl", pdl)
        model = LlamaModel(ctx, GEOMETRIES["tiny-gqa"], max_ctx=128, seed=3)
        lg = torch.empty(model.geom.vocab_size, dtype=torch.float32)
        seq = []
        for pos, tok in enumerate([1, 2, 3, 4]):
            model.decode_host(tok, pos, lg)
            seq.append(lg.clone())
        outs.append(torch.stack(seq))
        model.close()
        ctx.close()
    assert torch.equal(outs[0], outs[1])


def test_persistent_kernel_long_context_matches_graph_path(monkeypatch):
    """many steps through both decode paths on the same weights: the KV caches and logits must stay together (covers
    several attention splits per KV head inside the persistent kernel: chunk 64, ctx up to 200)."""
    from tinychatengine_b200.llama import GEOMETRIES, LlamaModel
    from tinychatengine_b200.runtime import Context

    g = GEOMETRIES["tiny-gqa"]
    outs = {}
    for mega in ("1", "0"):
        monkeypatch.setenv("TCE_PERSISTENT", mega)
        ctx = Context(0)
        model = LlamaModel(ctx, g, max_ctx=256, seed=11)
        assert (model.kernels_per_step == 1) == (mega == "1")
        lg = torch.empty(g.vocab_size, dtype=torch.float32)
        seq = []
        tok = 5
        for pos in range(200):
            tok = model.decode_host(tok % g.vocab_size, pos, lg)
            if pos % 25 == 24 or pos >= 196:
                seq.append(lg.clone())
            tok = (tok * 7 + pos) % g.vocab_size  # data-dependent but identical in both runs unless the paths diverge
        outs[mega] = (torch.stack(seq), model.kv_cache(1, 0)[:, :200].float().cpu().clone())
        model.close()
        ctx.close()
    assert rel_err(outs["1"][0].numpy(), outs["0"][0].numpy()) <= 5e-3
    assert rel_err(outs["1"][1].numpy(), outs["0"][1].numpy()) <= 5e-3


def test_persistent_kernel_is_deterministic_when_asked(monkeypatch):
    """TCE_DETERMINISTIC=1: o_proj / down_proj are cut at tile boundaries (one writer per residual element): same bits every run."""
    monkeypatch.setenv("TCE_DETERMINISTIC", "1")
    monkeypatch.setenv("TCE_PERSISTENT", "1")
    from tinychatengine_b200.llama import GEOMETRIES, LlamaModel
    from tinychatengine_b200.runtime import Context

    outs = []
    for _ in range(2):
        ctx = Context(0)
        model = LlamaModel(ctx, GEOMETRIES["tiny-gqa"], max_ctx=128, seed=3)
        assert model.kernels_per_step == 1
        lg = torch.empty(model.geom.vocab_size, dtype=torch.float32)
        seq = []
        for pos, tok in enumerate([1, 2, 3, 4, 5, 6]):
            model.decode_host(tok, pos, lg)
            seq.append(lg.clone())
        outs.append(torch.stack(seq))
        model.close()
        ctx.close()
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize(
    "widths,pos,mega",
    [pytest.param(w, pos, mega, id=f"{pos}-{mega}" if w == "llama3-8b" else f"{pos}-{mega}-{w}")
     for w in ("llama3-8b", "llama2-7b") for mega in ("1", "0") for pos in (0, 2048, 4095)],
)
def test_benchmarked_geometry_step_matches_oracle(widths, pos, mega, monkeypatch):
    """The configuration bench.py times -- Llama-3-8B widths (E 4096, F 14336, 32:8 heads, vocab 128256), max_ctx 4096 -- with two
    layers, at the start, the middle and the end of the context window, against the oracle-composed step on a random-filled cache.
    Llama-2-7B widths (F 11008: 86 groups per down_proj row) add weight stages that are only partly filled (22 of 32 groups)."""
    monkeypatch.setenv("TCE_PERSISTENT", mega)
    import dataclasses

    from tinychatengine_b200.llama import GEOMETRIES, LlamaModel
    from tinychatengine_b200.runtime import Context

    g = dataclasses.replace(GEOMETRIES[widths], name=f"{widths}-2l", num_layers=2)
    ctx = Context(0)
    model = LlamaModel(ctx, g, max_ctx=4096, seed=21, random_zeros=True)
    assert (model.kernels_per_step == 1) == (mega == "1")
    gen = torch.Generator(device="cuda")
    gen.manual_seed(pos + 1)
    past_k, past_v = [], []
    for l in range(g.num_layers):
        for which, store in ((0, past_k), (1, past_v)):
            c = model.kv_cache(l, which)
            c.copy_((torch.randn(c.shape, device="cuda", generator=gen) * 0.5).to(torch.float16))
            store.append(c[:, :pos].float().cpu().numpy() if pos else None)
    lg = torch.empty(g.vocab_size, dtype=torch.float32).pin_memory()
    nxt = model.decode_host(4321, pos, lg)
    want, fk, fv = oracle_decode_step(model, 4321, pos, past_k, past_v)
    got = lg.numpy()
    assert np.all(np.isfinite(got))
    e = rel_err(got, want)
    assert e <= 1e-2, (pos, e)
    assert nxt == int(np.argmax(got))
    for l in range(g.num_layers):
        assert np.abs(model.kv_cache(l, 0)[:, pos].float().cpu().numpy() - fk[l][:, pos]).max() <= 2e-2 * max(1.0, np.abs(fk[l]).max())
        # (the appended V row is the GEMV's fp16 output: equal to the oracle's up to the GEMV tolerance, not bit for bit)
        assert np.abs(model.kv_cache(l, 1)[:, pos].float().cpu().numpy() - fv[l][:, pos]).max() <= 5e-3 * max(1.0, np.abs(fv[l][:, pos]).max())
    model.close()
    ctx.close()


def test_load_dir_reference_tree(tmp_path):
    """The C++ loader (tce_llama_load_dir) on a parameter tree in the reference's on-disk layout (decoder/layer<i>/self_attn/qkv_proj/...,
    QM_CUDA op files): the loaded model decodes bit-identically to the model built from the same tensors in memory."""
    import numpy as np

    from tinychatengine_b200.llama import GEOMETRIES, LlamaModel
    from tinychatengine_b200.runtime import Context
    from tinychatengine_b200._lib import TceError

    ctx = Context(0)
    g = GEOMETRIES["tiny-gqa"]
    a = LlamaModel(ctx, g, max_ctx=64, seed=5, random_zeros=True)
    a.save_dir(tmp_path / "model", rotary=False)
    b = LlamaModel.load_dir(ctx, tmp_path / "model", g, max_ctx=64)
    la, lb = torch.empty(g.vocab_size), torch.empty(g.vocab_size)
    tok = 3
    for pos in range(5):
        na = a.decode_host(tok, pos, la)
        nb = b.decode_host(tok, pos, lb)
        assert na == nb and torch.equal(la, lb), pos
        tok = na
    # rotary tables / alpha files, when present, are used (fp16 tables of the same angles: close, not identical)
    hd = g.head_dim
    inv = 1.0 / (g.rope_theta ** (np.arange(0, hd, 2, dtype=np.float64) / hd))
    ang = np.arange(64)[:, None] * inv[None, :]
    emb = np.concatenate([ang, ang], axis=1)
    sa = tmp_path / "model" / "decoder" / "layer0" / "self_attn"
    (sa / "rotary_emb").mkdir()
    (sa / "qk_bmm").mkdir()
    np.cos(emb).astype(np.float16).tofile(sa / "rotary_emb" / "cos_cached_half.bin")
    np.sin(emb).astype(np.float16).tofile(sa / "rotary_emb" / "sin_cached_half.bin")
    np.array([1.0 / np.sqrt(hd)], dtype=np.float16).tofile(sa / "qk_bmm" / "alpha_half.bin")
    c = LlamaModel.load_dir(ctx, tmp_path / "model", g, max_ctx=64)
    lc = torch.empty(g.vocab_size)
    a.decode_host(3, 0, la)
    c.decode_host(3, 0, lc)
    a.decode_host(7, 1, la)
    c.decode_host(7, 1, lc)
    assert float((la - lc).abs().max() / la.abs().max()) < 2e-2
    # a truncated file is reported, not read past
    f = tmp_path / "model" / "lm_head" / "weight_int4.bin"
    f.write_bytes(f.read_bytes()[:-4])
    with pytest.raises(TceError, match="bytes on disk"):
        LlamaModel.load_dir(ctx, tmp_path / "model", g, max_ctx=64)
    for m in (a, b, c):
        m.close()
    ctx.close()


@pytest.mark.parametrize("mega", ["1", "0"])
def test_device_resident_token_and_position_are_range_checked(mega, monkeypatch):
    """tce_llama_decode takes {token, position} from device memory, so the host cannot validate them: the kernels must.  A position beyond the
    cache / a token beyond the table neither crashes nor writes any KV row (the next valid step still matches a fresh model), on the
    persistent kernel and on the kernel-per-op path."""
    monkeypatch.setenv("TCE_PERSISTENT", mega)
    from tinychatengine_b200.llama import GEOMETRIES, LlamaModel
    from tinychatengine_b200.runtime import Context

    ctx = Context(0)
    g = GEOMETRIES["tiny-gqa"]
    a = LlamaModel(ctx, g, max_ctx=32, seed=4)
    b = LlamaModel(ctx, g, max_ctx=32, seed=4)
    assert (a.kernels_per_step == 1) == (mega == "1")
    la, lb = torch.empty(g.vocab_size), torch.empty(g.vocab_size)
    assert a.decode_host(5, 0, la) == b.decode_host(5, 0, lb)
    kv_before = [a.kv_cache(l, w).clone() for l in range(g.num_layers) for w in (0, 1)]
    for bad in ([5, 32], [5, 10**6], [5, -1], [g.vocab_size, 31], [-3, 31]):
        a.decode(torch.tensor(bad, dtype=torch.int32, device="cuda"))
    torch.cuda.synchronize()
    kv_after = [a.kv_cache(l, w) for l in range(g.num_layers) for w in (0, 1)]
    # both steps refuse a bad entry: every row of every layer is as the valid step left it
    for x, y in zip(kv_before, kv_after):
        assert torch.equal(x, y)
    na, nb = a.decode_host(7, 1, la), b.decode_host(7, 1, lb)
    assert na == nb
    if mega == "1":
        assert torch.equal(la, lb)
    else:  # the kernel-per-op path finishes split tiles with fp32 atomics: equal up to summation order
        assert float((la - lb).abs().max() / lb.abs().max()) < 1e-4
    a.close()
    b.close()
    ctx.close()
