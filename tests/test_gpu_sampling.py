"""Device sampler and generate loop (csrc/sampling.cu, tce_sample / tce_llama_generate) against the CPU restatement of the reference's
sampling chain (oracle/sampling.py, pinned to llm/src/Generate.cc by tests/test_oracle_golden.py)."""
import numpy as np
import pytest
import torch

from oracle import sampling

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from tinychatengine_b200.runtime import Context

    c = Context(0)
    yield c
    c.close()


def _check(ctx, logits, window, cfg, seed=11, draw_index=3):
    dev = torch.from_numpy(logits.copy()).cuda()
    tok, ids, probs = ctx.sample(dev, window, seed=seed, draw_index=draw_index, candidates=True, repeat_last_n=-1, **cfg)
    oi, op = sampling.candidates(logits, window, **cfg)
    assert np.array_equal(ids, oi), (cfg, ids[:8], oi[:8])
    np.testing.assert_allclose(probs, op, rtol=0, atol=2e-6)
    # penalties were applied in place, exactly
    np.testing.assert_array_equal(dev.cpu().numpy(), sampling.apply_penalties(logits, window, cfg["repeat_penalty"], cfg["frequency_penalty"], cfg["presence_penalty"]))
    u = sampling.uniform01(seed, draw_index)
    cdf = np.cumsum(op.astype(np.float64))
    if cfg["temp"] > 0 and np.min(np.abs(cdf - u)) < 1e-5:
        return  # the uniform sits on a bin edge: either neighbour is right
    assert tok == sampling.draw(oi, op, u), (cfg, tok)


def test_golden_cases(ctx, golden_dir):
    g = np.load(golden_dir / "sampling.npz")
    for i in range(int(g["n_cases"])):
        c = g[f"cfg{i}"]
        cfg = dict(top_k=int(c[0]), top_p=float(c[1]), temp=float(c[2]), repeat_penalty=float(c[3]), frequency_penalty=float(c[4]), presence_penalty=float(c[5]))
        dev = torch.from_numpy(g["logits"].copy()).cuda()
        tok, ids, probs = ctx.sample(dev, g["window"], seed=1, candidates=True, repeat_last_n=-1, **cfg)
        assert np.array_equal(ids, g[f"ids{i}"]), cfg  # the reference's own output
        np.testing.assert_allclose(probs, g[f"probs{i}"], rtol=0, atol=2e-6)
        assert tok in ids


@pytest.mark.parametrize("V", [37, 1000, 32000, 128256])
def test_random_configs(ctx, V):
    rng = np.random.default_rng(V)
    for trial in range(4):
        logits = (rng.standard_normal(V) * rng.uniform(0.5, 6)).astype(np.float32)
        window = rng.integers(0, V, int(rng.integers(0, 130))).astype(np.int32)
        cfg = dict(top_k=int(rng.integers(1, min(V, 300))), top_p=float(rng.uniform(0.3, 1.0)), temp=float(rng.uniform(0.2, 1.5)),
                   repeat_penalty=float(rng.uniform(1.0, 1.5)), frequency_penalty=float(rng.uniform(0, 0.3)), presence_penalty=float(rng.uniform(0, 0.3)))
        _check(ctx, logits, window, cfg, seed=trial, draw_index=trial * 7)


def test_edge_cases(ctx):
    rng = np.random.default_rng(5)
    V = 5000
    logits = (rng.standard_normal(V) * 2).astype(np.float32)
    base = dict(top_k=40, top_p=0.95, temp=0.8, repeat_penalty=1.1, frequency_penalty=0.0, presence_penalty=0.0)
    _check(ctx, logits, (), base)                                    # no history
    _check(ctx, logits, (), dict(base, top_k=1))                     # k = 1
    _check(ctx, logits, (), dict(base, top_k=1024, top_p=1.0))       # the largest supported k, no nucleus cut
    _check(ctx, logits, [int(np.argmax(logits))] * 7, dict(base, temp=0.0, repeat_penalty=1.9))  # greedy after the penalty moved the maximum
    # ties: equal logits are ordered by ascending id, and the lowest ids at the top-k threshold survive
    tied = np.full(V, -1.0, dtype=np.float32)
    tied[[9, 100, 4000]] = 2.0
    tied[[5, 50, 500, 4999]] = 1.0
    tok, ids, probs = ctx.sample(torch.from_numpy(tied.copy()).cuda(), (), candidates=True, **dict(base, top_k=5, top_p=1.0))
    assert ids.tolist() == [9, 100, 4000, 5, 50]
    oi, op = sampling.candidates(tied, (), **dict(base, top_k=5, top_p=1.0))
    np.testing.assert_allclose(probs, op, atol=2e-6)
    # unsupported: sampling from the whole vocabulary
    from tinychatengine_b200._lib import TceError

    with pytest.raises(TceError):
        ctx.sample(torch.from_numpy(logits.copy()).cuda(), (), **dict(base, top_k=0))
    # the empirical distribution of many draws follows the candidate probabilities
    dev_logits = torch.from_numpy(logits.copy()).cuda()
    oi, op = sampling.candidates(logits, (), **dict(base, repeat_penalty=1.0))
    counts = {}
    n = 600
    for i in range(n):
        t = ctx.sample(dev_logits, (), seed=99, draw_index=i, **dict(base, repeat_penalty=1.0))
        counts[t] = counts.get(t, 0) + 1
    assert set(counts) <= set(oi.tolist())
    top = int(oi[0])
    assert abs(counts.get(top, 0) / n - float(op[0])) < 4 * np.sqrt(float(op[0]) * (1 - float(op[0])) / n) + 0.01


def test_generate_loop_matches_stepwise(ctx):
    """tce_llama_generate (decode + sample enqueued back to back, only ids come back) against the same loop driven from the host:
    decode_host -> logits -> oracle sampling with the history window the reference keeps (zeros before the first token)."""
    from tinychatengine_b200.llama import GEOMETRIES, LlamaModel

    g = GEOMETRIES["tiny-gqa"]
    model = LlamaModel(ctx, g, max_ctx=128, seed=3)
    cfg = dict(top_k=40, top_p=0.9, temp=0.9, repeat_penalty=1.2, frequency_penalty=0.1, presence_penalty=0.05)
    seed, first, n = 77, 5, 24
    out = model.generate(first, 0, n, history=[first], eos_id=-1, repeat_last_n=16, seed=seed, **cfg)
    assert len(out) == n
    # host-driven replay on a second model with the same weights
    model2 = LlamaModel(ctx, g, max_ctx=128, seed=3)
    lg = torch.empty(g.vocab_size, dtype=torch.float32)
    hist, tok, replay = [first], first, []
    for i in range(n):
        model2.decode_host(tok, i, lg)
        window = ([0] * 16 + hist)[-16:]
        ids, probs = sampling.candidates(lg.numpy(), window, **cfg)
        u = sampling.uniform01(seed, len(hist))
        cdf = np.cumsum(probs.astype(np.float64))
        tok = sampling.draw(ids, probs, u)
        if np.min(np.abs(cdf - u)) < 1e-4 and out[i] != tok:
            tok = out[i]  # bin edge: follow the device so that the rest of the sequence stays comparable
        assert out[i] == tok, (i, out[:i + 1], replay)
        replay.append(tok)
        hist.append(tok)
    # EOS stops the sequence: generation ends at the first occurrence of the eos id
    eos = out[3]
    out2 = model.generate(first, 0, n, history=[first], eos_id=eos, repeat_last_n=16, seed=seed, **cfg)
    assert out2 == out[:out.index(eos) + 1]
    # greedy generation equals the decode kernel's own arg-max chain
    model3 = LlamaModel(ctx, g, max_ctx=128, seed=3)
    greedy = model3.generate(first, 0, 8, temp=0.0, repeat_penalty=1.0)
    tok, chain = first, []
    for i in range(8):
        tok = model2.decode_host(tok, i, None)
        chain.append(tok)
    assert greedy == chain
    for m in (model, model2, model3):
        m.close()


@pytest.mark.parametrize("persistent", ["1", "0"])
def test_generate_kv_rows(ctx, monkeypatch, persistent):
    """After a budget stop, an eos_id stop and a max_ctx stop, slot 0 holds exactly rows pos0 .. pos0 + n_out - 1 new and every other row
    is byte-identical; a call refused for a NULL history writes nothing."""
    import ctypes as C

    from tinychatengine_b200 import _lib
    from tinychatengine_b200.llama import GEOMETRIES, LlamaModel

    monkeypatch.setenv("TCE_PERSISTENT", persistent)
    monkeypatch.setenv("TCE_DETERMINISTIC", "1")
    g = GEOMETRIES["tiny-gqa"]
    model = LlamaModel(ctx, g, max_ctx=128, seed=3)
    assert (model.kernels_per_step == 1) == (persistent == "1")
    gen = torch.Generator(device="cuda")
    gen.manual_seed(5)
    caches = [model.kv_cache(l, w) for l in range(g.num_layers) for w in (0, 1)]
    for c in caches:
        c.copy_((torch.randn(c.shape, device="cuda", generator=gen) * 0.5).to(torch.float16))
    orig = [c.cpu().clone() for c in caches]

    def run(pos0, n_predict, **kw):
        for c, o in zip(caches, orig):
            c.copy_(o.cuda())
        out = model.generate(7, pos0, n_predict, **kw)
        for c, o in zip(caches, orig):
            a, b = o.clone(), c.cpu().clone()
            assert not torch.equal(a[:, pos0:pos0 + len(out)], b[:, pos0:pos0 + len(out)])
            a[:, pos0:pos0 + len(out)] = 0
            b[:, pos0:pos0 + len(out)] = 0
            assert torch.equal(a, b)
        return out

    ref = run(10, 30, seed=9, top_k=20)  # budget stop
    assert len(ref) == 30
    eos = ref[4]
    assert run(10, 30, seed=9, top_k=20, eos_id=eos) == ref[:ref.index(eos) + 1]  # eos stop, with steps queued behind it
    assert len(run(120, 30, seed=9, top_k=20)) == 8  # max_ctx stop
    for c, o in zip(caches, orig):
        c.copy_(o.cuda())
    cfg = _lib.Sampling(40, 0.95, 0.8, 1.1, 0.0, 0.0, 64, 0)
    out, n = (C.c_int * 8)(*[-7] * 8), C.c_int(-1)
    assert ctx.L.tce_llama_generate(model.h, 7, 0, 8, C.byref(cfg), None, 2, -1, out, C.byref(n)) == -1  # n_history > 0, history NULL
    torch.cuda.synchronize()
    assert n.value == -1 and list(out) == [-7] * 8
    for c, o in zip(caches, orig):
        assert torch.equal(c.cpu(), o)
    model.close()
