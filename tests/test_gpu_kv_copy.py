"""KV-cache row copies (tce_llama_kv_copy): forks of a prompt's rows into other slots and context shifts inside a slot.  Checked bit for bit
against a numpy restatement of the kernel's rounding, against prompt passes at the new positions, against prompt passes of the whole
prompts, and inside the generate loops (n_keep) against host step chains."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HD = 128


def _model(geom, max_ctx, n_slots, seed=7, tables=None):
    """A synthetic model with n_slots KV-cache slots; tables = (cos, sin) CUDA float32 [max_ctx][128] makes it use the caller's RoPE tables."""
    from tinychatengine_b200 import _lib
    from tinychatengine_b200.llama import GEOMETRIES, LlamaModel
    from tinychatengine_b200.runtime import Context

    ctx = Context(0)
    model = LlamaModel(ctx, GEOMETRIES[geom], max_ctx=max_ctx, seed=seed, random_zeros=True)
    if tables is not None:
        w = _lib.LlamaWeights()
        w.embed_f16, w.layers, w.final_norm, w.lm_head = model.weights.embed_f16, model.weights.layers, model.weights.final_norm, model.weights.lm_head
        w.rope_cos, w.rope_sin = tables[0].data_ptr(), tables[1].data_ptr()
        h = C.c_void_p()
        _lib.check(ctx.L.tce_llama_create(ctx.h, C.byref(model.cfg), C.byref(w), C.byref(h)), "tce_llama_create")
        ctx.L.tce_llama_destroy(model.h)
        model.h, model._caller_tables = h, (w, tables)
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
    return [[[model.kv_cache(l, w, s).cpu().numpy().copy() for w in (0, 1)] for l in range(model.geom.num_layers)] for s in range(n_slots)]


def _restore(model, snap):
    for s, layers in enumerate(snap):
        for l, kv in enumerate(layers):
            for w in (0, 1):
                model.kv_cache(l, w, s).copy_(torch.from_numpy(kv[w]).cuda())


def _same_bits(a, b):
    return np.array_equal(a.view(np.uint16), b.view(np.uint16))


def _tokens(n, vocab, seed):
    return [int(t) for t in np.random.default_rng(seed).integers(0, vocab, n)]


def _theta_tables(theta, max_ctx):
    """The tables LlamaDecoder::create generates from rope_theta, computed the same way (double precision libm, then rounded to float)."""
    c = np.empty((max_ctx, HD), np.float32)
    s = np.empty((max_ctx, HD), np.float32)
    for i in range(HD // 2):
        inv = 1.0 / math.pow(float(theta), (2.0 * i) / HD)
        for p in range(max_ctx):
            ang = p * inv
            c[p, i] = c[p, i + HD // 2] = math.cos(ang)
            s[p, i] = s[p, i + HD // 2] = math.sin(ang)
    return c, s


def _rotate(x16, delta, cos, sin):
    """numpy restatement of kv_copy_kernel for K rows x16 (float16 [..., 128]) moved by delta: fp32 products and sums, each rounded on its
    own (numpy float32 arithmetic has no contraction), then round to fp16."""
    if delta == 0:
        return x16.copy()
    c = cos[abs(delta)]
    s = sin[abs(delta)] * np.float32(1.0 if delta > 0 else -1.0)
    x = x16.astype(np.float32)
    xj, xk = x[..., :HD // 2], x[..., HD // 2:]
    lo = xj * c[:HD // 2] - xk * s[:HD // 2]
    hi = xk * c[HD // 2:] + xj * s[HD // 2:]
    return np.concatenate([lo, hi], axis=-1).astype(np.float16)


# ------------------------------------------------------------------------------------------------ the kernel, bit for bit

MAX_CTX = 256
CASES = [  # (src_slot, src_pos, n, [(dst_slot, dst_pos), ...])
    (0, 10, 50, [(1, 10)]),                                 # d = 0 into another slot
    (2, 5, 100, [(3, 77)]),                                 # d > 0
    (4, 150, 60, [(5, 3)]),                                 # d < 0
    (6, 9, 200, [(6, 8)]),                                  # shift by -1, over two 128-row tiles
    (1, 50, 180, [(1, 13)]),                                # shift by -37, less than a tile
    (2, 130, 100, [(2, 4)]),                                # shift with |d| >= n
    (3, 20, 190, [(3, 61)]),                                # overlapping d > 0 inside one slot
    (7, 0, 255, [(7, 1)]),                                  # d = +1 over the whole slot but one row
    (0, 30, 40, [(1, 30), (2, 0), (3, 100), (4, 216), (5, 31), (6, 150), (7, 70)]),  # 7-way fork, different positions
    (5, 0, MAX_CTX, [(6, 0), (7, 0)]),                      # n = max_ctx
    (1, 0, 0, [(2, 5)]),                                    # n = 0
]


@pytest.mark.parametrize("tables", ["rope_theta", "caller"])
@pytest.mark.parametrize("geom", ["tiny-gqa", "tiny-mha"])
def test_kv_copy_matches_numpy(geom, tables):
    """Every case: every layer's K and V rows of every destination equal the numpy restatement on the model's tables (memmove semantics:
    computed from the cache before the call), and every other row of every slot is byte-identical."""
    from tinychatengine_b200.llama import GEOMETRIES

    g = GEOMETRIES[geom]
    if tables == "caller":
        gen = torch.Generator(device="cuda")
        gen.manual_seed(5)
        cos_t, sin_t = ((torch.rand((MAX_CTX, HD), device="cuda", generator=gen) * 2 - 1).float() for _ in range(2))
        ctx, model = _model(geom, MAX_CTX, 8, tables=(cos_t, sin_t))
        cos, sin = cos_t.cpu().numpy(), sin_t.cpu().numpy()
    else:
        ctx, model = _model(geom, MAX_CTX, 8)
        cos, sin = _theta_tables(np.float32(g.rope_theta), MAX_CTX)
    for k, (src, sp, n, dsts) in enumerate(CASES):
        _fill_caches(model, 8, 40 + k)
        before = _snapshot(model, 8)
        model.kv_copy(src, sp, n, [d for d, _ in dsts], [p for _, p in dsts])
        after = _snapshot(model, 8)
        want = [[[kv.copy() for kv in layer] for layer in slot] for slot in before]
        for d, dp in dsts:
            for l in range(g.num_layers):
                want[d][l][0][:, dp:dp + n] = _rotate(before[src][l][0][:, sp:sp + n], dp - sp, cos, sin)
                want[d][l][1][:, dp:dp + n] = before[src][l][1][:, sp:sp + n]
        for s in range(8):
            for l in range(g.num_layers):
                for w in (0, 1):
                    assert _same_bits(after[s][l][w], want[s][l][w]), (CASES[k], s, l, w)
    model.close()
    ctx.close()


# ------------------------------------------------------------------------------------------------ the rotation is RoPE

def test_shifted_keys_equal_a_prompt_pass_at_the_new_positions():
    """Prefill 200 tokens into slot 1, shift rows [78, 200) down to 8, and prefill tokens 78.. at position 8 into slot 2.  Layer 0's pre-RoPE
    keys are the same in both passes (they depend on the token only), so its K rows agree within fp16 rounding: the stored row carries one
    half-ulp error per element, which the rotation mixes over the pair (j, j + 64), and both results are rounded once more, so
    |got - want| <= 2^-11 (|x_j| + |x_{j+64}| + |got| + |want|) plus fp32 and table rounding (1e-6 of the pair).  V rows are bit-identical.
    Deeper layers are not compared: their rows depend on the context the shift removed."""
    ctx, model = _model("tiny-gqa", MAX_CTX, 3, seed=12)
    g = model.geom
    toks = _tokens(200, g.vocab_size, 3)
    model.prefill(toks, 0, slot=1)
    x = model.kv_cache(0, 0, 1)[:, 78:200].cpu().numpy().astype(np.float32)
    assert model.kv_shift(1, 200, 8, 70) == 130
    model.prefill(toks[78:], 8, slot=2)
    torch.cuda.synchronize()
    got = model.kv_cache(0, 0, 1)[:, 8:130].cpu().numpy().astype(np.float32)
    want = model.kv_cache(0, 0, 2)[:, 8:130].cpu().numpy().astype(np.float32)
    pair = np.abs(x) + np.abs(np.roll(x, HD // 2, axis=-1))
    tol = 2.0 ** -11 * (pair + np.abs(got) + np.abs(want)) + 1e-6 * pair + 2.0 ** -24
    assert np.all(np.abs(got - want) <= tol), float(np.max(np.abs(got - want) - tol))
    assert torch.equal(model.kv_cache(0, 1, 1)[:, 8:130], model.kv_cache(0, 1, 2)[:, 8:130])
    model.close()
    ctx.close()


# ------------------------------------------------------------------------------------------------ forks end to end

def test_fork_equals_prompt_pass_per_slot(monkeypatch):
    """One prompt pass into slot 3 forked into 7 slots holds the same K/V bits as the ragged prompt pass of 8 copies, and the batched
    generate loop with 8 seeds returns the same ids on both."""
    monkeypatch.setenv("TCE_DETERMINISTIC", "1")
    ctx, model = _model("tiny-gqa", MAX_CTX, 16, seed=9)
    g = model.geom
    prompt = _tokens(100, g.vocab_size, 5)
    nxt = model.prefill(prompt, 0, slot=3)
    model.fork(3, 100, [0, 1, 2, 4, 5, 6, 7])
    model.prefill_batch([prompt] * 8, list(range(8, 16)))
    torch.cuda.synchronize()
    for i in range(8):
        for l in range(g.num_layers):
            for w in (0, 1):
                assert torch.equal(model.kv_cache(l, w, i), model.kv_cache(l, w, 8 + i)), (i, l, w)
    reqs = lambda base: [dict(first_token=nxt, pos0=100, slot=base + i, n_predict=24, seed=100 + i) for i in range(8)]
    forked = model.generate_batch(reqs(0))
    assert forked == model.generate_batch(reqs(8))
    assert len({tuple(o) for o in forked}) > 1  # the seeds do give different continuations
    model.close()
    ctx.close()


def test_multiple_choice_scores_through_a_fork():
    """A context prefilled once and forked to 4 slots, then the 4 endings scored at pos0 = len(context): the endings' log-probabilities and
    greedy ids are bit-identical to scoring the 4 full prompts (every GEMM row is independent of the others, and a row's attention visits
    the same key tiles in the same order, wherever its query block starts)."""
    ctx, model = _model("tiny-gqa", MAX_CTX, 8, seed=11)
    g = model.geom
    context = _tokens(60, g.vocab_size, 21)
    endings = [_tokens(n, g.vocab_size, 30 + i) for i, n in enumerate([5, 9, 2, 12])]
    model.prefill(context, 0, slot=0)
    model.fork(0, 60, [1, 2, 3])
    forked = model.score_batch(endings, [0, 1, 2, 3], pos0s=[60] * 4)
    full = model.score_batch([context + e for e in endings], [4, 5, 6, 7])
    for f, w in zip(forked, full):
        assert np.array_equal(f[0], w[0][60:], equal_nan=True)
        assert np.array_equal(f[1], w[1][60:])
        assert np.array_equal(f[2], w[2][60:])
    model.close()
    ctx.close()


# ------------------------------------------------------------------------------------------------ context shift in the generate loops

N_KEEP, N_PREDICT, POS0 = 8, 400, 100


def _host_chain(model, first, slots, step):
    """Greedy host chain from POS0 with the shift of every slot at each full context: step(tokens, positions) -> next tokens."""
    tok, pos, out = list(first), POS0, [[] for _ in slots]
    for _ in range(N_PREDICT):
        if pos == model.max_ctx:
            pos = [model.kv_shift(s, model.max_ctx, N_KEEP) for s in slots][0]
        tok = step(tok, [pos] * len(slots))
        for b, t in enumerate(tok):
            out[b].append(t)
        pos += 1
    return out


def test_generate_batch_context_shift(monkeypatch):
    """max_ctx 128, greedy: generate_batch with n_keep = 8 and a budget of 400 ids from position 100 (7 shifts) returns the ids of a host
    chain of batched steps that shifts at the same points; without n_keep the loop stops at max_ctx as before."""
    monkeypatch.setenv("TCE_DETERMINISTIC", "1")
    ctx, model = _model("tiny-gqa", 128, 4, seed=13)
    _fill_caches(model, 4, 50)
    before = _snapshot(model, 4)
    slots, first = [2, 0, 3], [5, 700, 1999]
    reqs = [dict(first_token=t, pos0=POS0, slot=s, n_predict=N_PREDICT, temp=0.0, repeat_penalty=1.0) for t, s in zip(first, slots)]
    outs = model.generate_batch(reqs, n_keep=N_KEEP)
    assert [len(o) for o in outs] == [N_PREDICT] * 3
    _restore(model, before)
    chain = _host_chain(model, first, slots, lambda tok, pos: model.decode_batch_host(tok, pos, slots))
    assert outs == chain
    _restore(model, before)
    plain = model.generate_batch(reqs)
    assert plain == [o[:128 - POS0] for o in outs]
    model.close()
    ctx.close()


def test_generate_context_shift_persistent(monkeypatch):
    """The same on the single-sequence loop (slot 0, the persistent decode kernel): generate(..., n_keep = 8) against a chain of decode_host
    steps with kv_shift at each full context."""
    monkeypatch.setenv("TCE_DETERMINISTIC", "1")
    ctx, model = _model("tiny-gqa", 128, 1, seed=14)
    assert model.kernels_per_step == 1  # the persistent kernel
    _fill_caches(model, 1, 51)
    before = _snapshot(model, 1)
    out = model.generate(77, POS0, N_PREDICT, temp=0.0, repeat_penalty=1.0, n_keep=N_KEEP)
    assert len(out) == N_PREDICT
    _restore(model, before)
    chain = _host_chain(model, [77], [0], lambda tok, pos: [model.decode_host(tok[0], pos[0])])
    assert out == chain[0]
    _restore(model, before)
    assert model.generate(77, POS0, N_PREDICT, temp=0.0, repeat_penalty=1.0) == out[:128 - POS0]
    model.close()
    ctx.close()


# ------------------------------------------------------------------------------------------------ refusals

def test_kv_copy_refusals():
    """Every refusal returns TCE_ERR_INVALID before anything is enqueued: all caches stay byte-identical."""
    from tinychatengine_b200 import _lib

    ctx, model = _model("tiny-gqa", 128, 3)
    _fill_caches(model, 3, 60)
    before = _snapshot(model, 3)
    L = ctx.L

    def call(src, sp, n, dsts):
        arr = lambda v: (C.c_int * max(1, len(v)))(*v)
        return L.tce_llama_kv_copy(model.h, src, sp, n, len(dsts), arr([d for d, _ in dsts]), arr([p for _, p in dsts]))

    bad = [
        (0, 0, 4, []),                                  # no destination
        (0, 0, 4, [(1, 10 * i) for i in range(9)]),     # 9 destinations
        (3, 0, 4, [(1, 0)]),                            # source slot not reserved
        (-1, 0, 4, [(1, 0)]),                           # source slot < 0
        (0, 0, 4, [(3, 0)]),                            # destination slot not reserved
        (0, 0, 4, [(1, 0), (-1, 0)]),                   # destination slot < 0
        (0, -1, 4, [(1, 0)]),                           # source before row 0
        (0, 120, 10, [(1, 0)]),                         # source past max_ctx
        (0, 0, 10, [(1, 125)]),                         # destination past max_ctx
        (0, 0, 10, [(1, -1)]),                          # destination before row 0
        (0, 0, 129, [(1, 0)]),                          # n > max_ctx
        (0, 0, -1, [(1, 0)]),                           # n < 0
        (0, 0, 10, [(1, 0), (1, 9)]),                   # two destinations overlap in one slot
        (0, 0, 10, [(2, 50), (1, 0), (2, 45)]),
        (0, 0, 10, [(0, 5), (1, 0)]),                   # a destination overlaps the source with n_dst > 1
        (1, 20, 10, [(2, 0), (1, 29)]),
    ]
    for case in bad:
        assert call(*case) == -1, case
    assert L.tce_llama_kv_copy(model.h, 0, 0, 4, 1, None, None) == -1
    assert L.tce_llama_kv_copy(None, 0, 0, 4, 1, (C.c_int * 1)(1), (C.c_int * 1)(0)) == -1
    with pytest.raises(ValueError):
        model.kv_shift(1, 100, 99)                      # n_discard = 0
    with pytest.raises(ValueError):
        model.generate_batch([dict(first_token=1, pos0=0, slot=0, n_predict=1)], n_keep=127)
    _check = _snapshot(model, 3)
    for s in range(3):
        for l in range(model.geom.num_layers):
            for w in (0, 1):
                assert _same_bits(before[s][l][w], _check[s][l][w]), (s, l, w)
    # the boundaries that are allowed: the last row, a destination adjacent to the source, n = 0 at max_ctx
    assert call(0, 127, 1, [(1, 0)]) == 0
    assert call(0, 0, 10, [(0, 10)]) == 0 and call(0, 0, 10, [(1, 10), (0, 10)]) == 0
    assert call(0, 128, 0, [(1, 128)]) == 0
    with pytest.raises(_lib.TceError):
        model.kv_copy(0, 0, 4, [5])
    model.close()
    ctx.close()


def test_tensor_parallel_model_is_unsupported():
    from tinychatengine_b200._lib import TceError
    from tinychatengine_b200.llama import GEOMETRIES, LlamaModel, make_random_weights, shard_weights
    from tinychatengine_b200.runtime import Context

    ctx = Context(0)
    g = GEOMETRIES["tiny-gqa"]
    W = make_random_weights(g, torch.device("cuda", 0), 3)
    Wl, gl = shard_weights(W, g, 0, 2)
    model = LlamaModel(ctx, gl, max_ctx=128, weights=Wl, tp_rank=0, tp_size=2)
    one = (C.c_int * 1)(0)
    assert ctx.L.tce_llama_kv_copy(model.h, 0, 0, 4, 1, one, one) == -2
    with pytest.raises(TceError, match="tp_size"):
        model.fork(0, 4, [0])
    model.close()
    ctx.close()
