"""Prompt scoring (tce_llama_score_batch): per-position log-probabilities of up to 8 prompts from one prompt pass, with the lm_head over every
row and the log-softmax reduced in its GEMM epilogue.  Checked against the oracle, against float64 log_softmax of the logits the same call
stores, against prefill_batch (logits of prefixes, K/V bits), for independence of rows, for its refusals and through tools/perplexity.py."""
import ctypes as C
import importlib.util
from pathlib import Path

import numpy as np
import pytest
import torch

from helpers import oracle_decode_step, rel_err

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]


def _geom(name):
    from tinychatengine_b200.llama import GEOMETRIES, LlamaGeometry

    if name == "chunks":  # lm_head of 2000 rows over a scratch half of 1536 rows of E: two chunks, the second of 464 rows (not a multiple of 128)
        return LlamaGeometry("chunks", 1, 4, 4, 512, 256, 2000, 1e-5, 10000.0)
    if name == "llama3-8b-2l":
        b = GEOMETRIES["llama3-8b"]
        return LlamaGeometry(name, 2, b.num_heads, b.num_kv_heads, b.embed_dim, b.hidden_dim, b.vocab_size, b.rms_eps, b.rope_theta, b.head_dim)
    return GEOMETRIES[name]


def _model(name, max_ctx, n_slots, seed=7):
    from tinychatengine_b200.llama import LlamaModel
    from tinychatengine_b200.runtime import Context

    ctx = Context(0)
    model = LlamaModel(ctx, _geom(name), max_ctx=max_ctx, seed=seed, random_zeros=True)
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
    torch.cuda.synchronize()
    return [[[model.kv_cache(l, w, s).clone() for w in (0, 1)] for l in range(model.geom.num_layers)] for s in range(n_slots)]


def _restore(model, snap):
    for s, layers in enumerate(snap):
        for l, kv in enumerate(layers):
            for w in (0, 1):
                model.kv_cache(l, w, s).copy_(kv[w])
    torch.cuda.synchronize()


def _check_rows(before, after, written):
    """written: slot -> (first row, count).  Every row outside those is byte-identical."""
    for s in range(len(before)):
        for l in range(len(before[s])):
            for w in (0, 1):
                a, b = before[s][l][w].clone(), after[s][l][w].clone()
                if s in written:
                    r0, n = written[s]
                    a[:, r0:r0 + n] = 0
                    b[:, r0:r0 + n] = 0
                assert torch.equal(a, b), (s, l, w)


def _tokens(n, vocab, seed):
    return [int(t) for t in np.random.default_rng(seed).integers(0, vocab, n)]


def _targets(lengths, vocab, seed):
    rng = np.random.default_rng(seed)
    out = []
    for n in lengths:
        t = rng.integers(0, vocab, n)
        t[rng.random(n) < 0.2] = -1
        out.append([int(x) for x in t])
    return out


def _check_stats(res, logits, targets):
    """Fused outputs against float64 log_softmax of the logits the same call stored.  Returns the largest |logprob - ref|."""
    lsm = torch.log_softmax(logits.double(), dim=1).cpu().numpy()
    worst, r = 0.0, 0
    for (lp, gr, glp), tg in zip(res, targets):
        for i, t in enumerate(tg):
            ref = lsm[r + i]
            want_g = int(np.argmax(ref))  # lowest id among equal maxima
            assert gr[i] == want_g, (r + i, gr[i], want_g)
            assert abs(glp[i] - ref[want_g]) <= 1e-5, (r + i, glp[i], ref[want_g])
            if t < 0:
                assert np.isnan(lp[i]), (r + i, lp[i])
            else:
                assert abs(lp[i] - ref[t]) <= 1e-5, (r + i, lp[i], ref[t])
                worst = max(worst, abs(float(lp[i]) - float(ref[t])))
        r += len(tg)
    return worst


def _same(a, b):
    for (x0, x1, x2), (y0, y1, y2) in zip(a, b):
        assert np.array_equal(x0.view(np.uint32), y0.view(np.uint32))
        assert np.array_equal(x1, y1)
        assert np.array_equal(x2.view(np.uint32), y2.view(np.uint32))


# ------------------------------------------------------------------------------------------------ against the oracle

@pytest.mark.parametrize("geom", ["tiny-gqa", "tiny-mha", "chunks"])
def test_score_matches_oracle(geom):
    """Prompts of 70, 1, 33 and 65 tokens in out-of-order slots plus one that continues slot 3 at position 40, random targets with -1s: every
    row of logits_dev against the oracle, the fused statistics against float64 log_softmax of those logits, the same outputs without
    logits_dev, and no KV row outside the prompts' rows touched."""
    ctx, model = _model(geom, 256, 8)
    g = model.geom
    _fill_caches(model, 8, 21)
    before = _snapshot(model, 8)
    lengths, pos0s, slots = [70, 1, 33, 65, 20], [0, 0, 0, 0, 40], [5, 0, 7, 2, 3]
    prompts = [_tokens(n, g.vocab_size, 100 + i) for i, n in enumerate(lengths)]
    targets = _targets(lengths, g.vocab_size, 5)
    n = sum(lengths)
    logits = torch.full((n, g.vocab_size), float("nan"), dtype=torch.float32, device="cuda")
    res = model.score_batch(prompts, slots, pos0s, targets, logits)
    after = _snapshot(model, 8)
    _check_rows(before, after, {s: (p0, len(p)) for p, p0, s in zip(prompts, pos0s, slots)})
    lg = logits.cpu().numpy()
    assert np.all(np.isfinite(lg))
    worst, r = 0.0, 0
    for prompt, p0, slot in zip(prompts, pos0s, slots):
        if p0 == 0:
            pk, pv = [None] * g.num_layers, [None] * g.num_layers
        else:
            pk = [before[slot][l][0][:, :p0].float().cpu().numpy() for l in range(g.num_layers)]
            pv = [before[slot][l][1][:, :p0].float().cpu().numpy() for l in range(g.num_layers)]
        for i, tok in enumerate(prompt):
            want, pk, pv = oracle_decode_step(model, tok, p0 + i, pk, pv)
            e = rel_err(lg[r + i], want)
            assert e <= 1e-2, (r + i, e)
            worst = max(worst, e)
        r += len(prompt)
    lp_worst = _check_stats(res, logits, targets)
    print(f"[{geom}] logits rel err vs oracle <= {worst:.3e}; |logprob - float64 log_softmax| <= {lp_worst:.2e}")
    _same(res, model.score_batch(prompts, slots, pos0s, targets))  # without logits_dev: bit-identical outputs
    model.close()
    ctx.close()


def test_default_targets_are_next_tokens():
    """targets = None scores each position against the next token of its prompt, NaN on each prompt's last position."""
    ctx, model = _model("chunks", 128, 3)
    g = model.geom
    lengths = [40, 1, 17]
    prompts = [_tokens(n, g.vocab_size, 30 + i) for i, n in enumerate(lengths)]
    nxt = [p[1:] + [-1] for p in prompts]
    _same(model.score_batch(prompts, [2, 0, 1]), model.score_batch(prompts, [2, 0, 1], targets=nxt))
    for lp, _, _ in model.score_batch(prompts, [2, 0, 1]):
        assert np.isnan(lp[-1]) and np.all(np.isfinite(lp[:-1]))
    model.close()
    ctx.close()


# ------------------------------------------------------------------------------------------------ Llama-3-8B widths: 5 lm_head chunks

def test_llama3_widths_against_prefill_batch():
    """Llama-3-8B widths (2 layers, max_ctx 4096), 8 prompts up to position 4095, 5 lm_head chunks: score rows against the last-row logits of
    a prefill_batch of the same prefix in a spare slot, the fused statistics against the stored logits, and the K/V caches bit-identical to
    those prefill_batch leaves with the same arguments."""
    ctx, model = _model("llama3-8b-2l", 4096, 9, seed=5)
    g = model.geom
    _fill_caches(model, 9, 3)
    before = _snapshot(model, 9)
    lengths = [300, 17, 129, 64, 1, 250, 96, 200]
    pos0s = [0, 100, 0, 3000, 4095, 0, 512, 3896]
    slots = list(range(8))
    prompts = [_tokens(n, g.vocab_size, 7 + i) for i, n in enumerate(lengths)]
    targets = _targets(lengths, g.vocab_size, 9)
    n = sum(lengths)
    logits = torch.empty((n, g.vocab_size), dtype=torch.float32, device="cuda")
    res = model.score_batch(prompts, slots, pos0s, targets, logits)
    scored = _snapshot(model, 9)
    _check_rows(before, scored, {s: (p0, len(p)) for p, p0, s in zip(prompts, pos0s, slots)})
    lp_worst = _check_stats(res, logits, targets)
    # the same arguments through prefill_batch write the same K/V bits
    _restore(model, before)
    model.prefill_batch(prompts, slots, pos0s)
    pre = _snapshot(model, 9)
    for s in range(9):
        for l in range(g.num_layers):
            for w in (0, 1):
                assert torch.equal(scored[s][l][w], pre[s][l][w]), (s, l, w)
    # rows of logits_dev against prefill_batch of the prefix into the spare slot 8, which first gets the prompt's slot history
    lg = logits.cpu().numpy()
    one = torch.empty((1, g.vocab_size), dtype=torch.float32).pin_memory()
    worst, r = 0.0, 0
    for b, (prompt, p0) in enumerate(zip(prompts, pos0s)):
        for i in sorted({0, len(prompt) // 5, len(prompt) // 3, len(prompt) // 2, (3 * len(prompt)) // 4, len(prompt) - 1}):
            for l in range(g.num_layers):
                for w in (0, 1):
                    model.kv_cache(l, w, 8).copy_(before[b][l][w])
            model.prefill_batch([prompt[:i + 1]], [8], [p0], one)
            e = rel_err(lg[r + i], one[0].numpy())
            assert e <= 1e-2, (b, i, e)
            worst = max(worst, e)
        r += len(prompt)
    print(f"[llama3-8b widths] score rows vs prefill_batch last rows: rel err <= {worst:.3e}; |logprob - ref| <= {lp_worst:.2e}")
    model.close()
    ctx.close()


# ------------------------------------------------------------------------------------------------ independence of rows

@pytest.mark.parametrize("geom", ["tiny-gqa", "chunks"])
def test_rows_are_independent(geom):
    """A prompt's outputs and logits are bit-identical alone, inside a batch of 8, with the batch permuted, and over two repeated calls."""
    ctx, model = _model(geom, 512, 8)
    g = model.geom
    lengths = [5, 300, 1, 129, 64, 257, 33, 128]
    prompts = [_tokens(n, g.vocab_size, 50 + i) for i, n in enumerate(lengths)]
    targets = _targets(lengths, g.vocab_size, 11)
    n = sum(lengths)

    def run(idx):
        lg = torch.empty((sum(lengths[i] for i in idx), g.vocab_size), dtype=torch.float32, device="cuda")
        res = model.score_batch([prompts[i] for i in idx], list(idx), None, [targets[i] for i in idx], lg)
        out, r = {}, 0
        for k, i in enumerate(idx):
            out[i] = (res[k], lg[r:r + lengths[i]].cpu())
            r += lengths[i]
        return out

    full = run(list(range(8)))
    assert len(full) == 8 and n == sum(lengths)
    for other in (run([3, 7, 0, 5, 1, 6, 2, 4]), run(list(range(8))), {i: run([i])[i] for i in range(8)}):
        for i in range(8):
            _same([full[i][0]], [other[i][0]])
            assert torch.equal(full[i][1], other[i][1]), i
    model.close()
    ctx.close()


# ------------------------------------------------------------------------------------------------ refusals

def test_score_batch_refusals():
    """Every refusal returns TCE_ERR_INVALID before anything is enqueued: all caches stay byte-identical."""
    ctx, model = _model("tiny-gqa", 128, 3)
    g = model.geom
    _fill_caches(model, 3, 4)
    before = _snapshot(model, 3)
    L = ctx.L
    arr = lambda v: (C.c_int * max(1, len(v)))(*[int(x) for x in v])

    def call(prompts, slots, pos0s, targets=None):
        flat = [t for p in prompts for t in p]
        return L.tce_llama_score_batch(model.h, len(prompts), arr(flat), arr([len(p) for p in prompts]), arr(pos0s), arr(slots),
                                       None if targets is None else arr(targets), None, None, None, None)

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
        _check_rows(before, _snapshot(model, 3), {})
    for tg in ([5, -2, 1], [5, g.vocab_size, 1], [-1, -1, -7]):  # targets outside [-1, vocab)
        assert call([[1, 2], [3]], [0, 1], [0, 0], tg) == -1, tg
        _check_rows(before, _snapshot(model, 3), {})
    assert L.tce_llama_score_batch(model.h, 1, None, None, None, None, None, None, None, None, None) == -1
    model.close()
    ctx.close()


def test_tensor_parallel_model_is_unsupported():
    from tinychatengine_b200._lib import TceError
    from tinychatengine_b200.llama import GEOMETRIES, LlamaModel, make_random_weights, shard_weights
    from tinychatengine_b200.runtime import Context

    ctx = Context(0)
    g = GEOMETRIES["tiny-gqa"]
    Wl, gl = shard_weights(make_random_weights(g, torch.device("cuda", 0), 3), g, 0, 2)
    model = LlamaModel(ctx, gl, max_ctx=128, weights=Wl, tp_rank=0, tp_size=2)
    one = (C.c_int * 1)(0)
    assert ctx.L.tce_llama_score_batch(model.h, 1, one, (C.c_int * 1)(1), one, one, None, None, None, None, None) == -2
    with pytest.raises(TceError, match="tp_size"):
        model.score_batch([[1, 2]], [0])
    model.close()
    ctx.close()


# ------------------------------------------------------------------------------------------------ tools/perplexity.py

def test_perplexity_tool_equals_direct_calls(tmp_path):
    """The tool's strided windows (C = 128, S = 64) over 300 tokens of a saved tiny model, loaded back with load_dir: its NLL sum equals the
    sum over one direct score_batch call per window."""
    from tinychatengine_b200.llama import LlamaModel

    spec = importlib.util.spec_from_file_location("perplexity_tool", ROOT / "tools" / "perplexity.py")
    pp = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(pp)
    ctx, model = _model("tiny-gqa", 128, 1, seed=9)
    model.save_dir(tmp_path)
    g = model.geom
    model.close()
    loaded = LlamaModel.load_dir(ctx, tmp_path, g, max_ctx=128)
    tokens = np.random.default_rng(4).integers(0, g.vocab_size, 300)
    nll, count = pp.score_tokens(loaded, tokens, 128, 64)
    assert count == 299
    direct, seen = 0.0, 0
    for start, length, first in pp.window_plan(len(tokens), 128, 64):
        tg = pp.window_targets(tokens, start, length, first)
        (lp, _, _), = loaded.score_batch([tokens[start:start + length].tolist()], [0], targets=[tg])
        m = tg >= 0
        assert np.all(np.isfinite(lp[m]))
        direct -= float(np.sum(lp[m].astype(np.float64)))
        seen += int(m.sum())
    assert seen == count
    assert nll == direct, (nll, direct)
    print(f"[perplexity] 300 tokens, C=128, S=64: ppl {np.exp(nll / count):.3f}")
    loaded.close()
    ctx.close()
