"""Batched decode (tce_llama_decode_batch*): up to 8 sequences per step, each in its own KV-cache slot, against the oracle-composed step of
each sequence; the multi-column W4A16 GEMV that streams each weight byte once at any IC; request validation and determinism."""
import numpy as np
import pytest
import torch

from helpers import assert_w4_close, oracle_decode_step, rel_err

pytestmark = pytest.mark.gpu

MIXED_POS = [0, 1, 37, 63, 64, 130, 200, 255]


def _model(geom, max_ctx, seed=7, n_slots=8):
    from tinychatengine_b200.llama import GEOMETRIES, LlamaGeometry, LlamaModel
    from tinychatengine_b200.runtime import Context

    g = GEOMETRIES[geom] if isinstance(geom, str) else geom
    assert isinstance(g, LlamaGeometry)
    ctx = Context(0)
    model = LlamaModel(ctx, g, max_ctx=max_ctx, seed=seed, random_zeros=True)
    model.reserve_slots(n_slots)
    return ctx, model


def _fill_caches(model, n_slots, seed):
    gen = torch.Generator(device="cuda")
    gen.manual_seed(seed)
    for s in range(n_slots):
        for l in range(model.geom.num_layers):
            for which in (0, 1):
                c = model.kv_cache(l, which, s)
                c.copy_((torch.randn(c.shape, device="cuda", generator=gen) * 0.5).to(torch.float16))


def _snapshot(model, n_slots):
    return [[[model.kv_cache(l, w, s).cpu().clone() for w in (0, 1)] for l in range(model.geom.num_layers)] for s in range(n_slots)]


def _past(snap, slot, pos):
    if pos == 0:
        return [None] * len(snap[slot]), [None] * len(snap[slot])
    return ([snap[slot][l][0][:, :pos].float().numpy() for l in range(len(snap[slot]))],
            [snap[slot][l][1][:, :pos].float().numpy() for l in range(len(snap[slot]))])


def _check_step(model, before, after, entries, got_logits, got_next, n_slots):
    """entries: (token, pos, slot) that must have run; every other cache row of every slot must be byte-identical"""
    touched = {}
    for b, (tok, pos, slot) in enumerate(entries):
        pk, pv = _past(before, slot, pos)
        want, fk, fv = oracle_decode_step(model, tok, pos, pk, pv)
        got = got_logits[b]
        assert np.all(np.isfinite(got))
        e = rel_err(got, want)
        assert e <= 1e-2, (b, tok, pos, slot, e)
        if got_next is not None:
            assert got_next[b] == int(np.argmax(got)), (b, got_next[b])
        for l in range(model.geom.num_layers):
            k = after[slot][l][0][:, pos].float().numpy()
            v = after[slot][l][1][:, pos].float().numpy()
            assert np.abs(k - fk[l][:, pos]).max() <= 2e-2 * max(1.0, np.abs(fk[l]).max()), (b, l)
            assert np.abs(v - fv[l][:, pos]).max() <= 5e-3 * max(1.0, np.abs(fv[l][:, pos]).max()), (b, l)
        touched[slot] = pos
    for s in range(n_slots):
        for l in range(model.geom.num_layers):
            for w in (0, 1):
                a, b_ = before[s][l][w].clone(), after[s][l][w].clone()
                if s in touched:
                    a[:, touched[s]] = 0
                    b_[:, touched[s]] = 0
                assert torch.equal(a, b_), (s, l, w)


@pytest.mark.parametrize("batch", [1, 3, 8])
@pytest.mark.parametrize("geom", ["tiny-gqa", "tiny-mha"])
def test_batched_step_matches_oracle(geom, batch):
    ctx, model = _model(geom, 256)
    g = model.geom
    _fill_caches(model, 8, 100 + batch)
    before = _snapshot(model, 8)
    # mixed positions, slots out of order; the batch uses a subset of the 8 slots
    slots = [5, 0, 7, 2, 1, 6, 3, 4][:batch]
    pos = MIXED_POS[:batch] if batch < 8 else MIXED_POS
    toks = [(17 * i + 3) % g.vocab_size for i in range(batch)]
    lg = torch.empty((batch, g.vocab_size), dtype=torch.float32).pin_memory()
    nxt = model.decode_batch_host(toks, pos, slots, lg)
    after = _snapshot(model, 8)
    _check_step(model, before, after, list(zip(toks, pos, slots)), lg.numpy(), nxt, 8)
    # the device-resident entry point computes the same step (RED.ADD residual: last-bit differences)
    req = torch.tensor(list(zip(toks, pos, slots)), dtype=torch.int32, device="cuda")
    model.decode_batch(req)
    torch.cuda.synchronize()
    assert rel_err(model.batch_logits()[:batch].cpu().numpy(), lg.numpy()) <= 2e-3
    model.close()
    ctx.close()


def _wide_geom(name, base, layers):
    from tinychatengine_b200.llama import GEOMETRIES, LlamaGeometry

    b = GEOMETRIES[base]
    return LlamaGeometry(name, layers, b.num_heads, b.num_kv_heads, b.embed_dim, b.hidden_dim, b.vocab_size, b.rms_eps, b.rope_theta, b.head_dim)


@pytest.mark.parametrize("case", ["llama3-8b-2l", "llama2-13b-1l"])
def test_batched_step_full_widths(case):
    """Llama-3-8B widths (down_proj IC = 14336 runs K-sliced) at 8 sequences up to the last cache row; Llama-2-13B widths (IC = 5120 with the
    RMSNorm prologue and the SiLU pair epilogue, IC = 13824 down_proj) at 4."""
    if case == "llama3-8b-2l":
        g, max_ctx, pos = _wide_geom(case, "llama3-8b", 2), 4096, [0, 1, 511, 1024, 2047, 2048, 3000, 4095]
    else:
        g, max_ctx, pos = _wide_geom(case, "llama2-13b", 1), 1024, [0, 77, 512, 1023]
    batch = len(pos)
    ctx, model = _model(g, max_ctx, seed=5, n_slots=batch)
    _fill_caches(model, batch, 31)
    before = _snapshot(model, batch)
    slots = list(range(batch))[::-1]
    toks = [(1009 * i + 11) % g.vocab_size for i in range(batch)]
    lg = torch.empty((batch, g.vocab_size), dtype=torch.float32).pin_memory()
    nxt = model.decode_batch_host(toks, pos, slots, lg)
    after = _snapshot(model, batch)
    _check_step(model, before, after, list(zip(toks, pos, slots)), lg.numpy(), nxt, batch)
    model.close()
    ctx.close()


def test_interleaved_with_single_sequence_and_prefill():
    """Six steps of 3 sequences in slots 1..3, with single-sequence steps on slot 0 and prompt passes into slots 1..3 in between, each
    against its own oracle chain.  A prompt pass touches only its own slot."""
    ctx, model = _model("tiny-gqa", 256, seed=9, n_slots=4)
    g = model.geom
    L = g.num_layers

    def state_of(slot, n):
        snap = _snapshot(model, 4)
        return _past(snap, slot, n)

    seqs = {}  # slot -> [next token, position, past_k, past_v]

    def prefill(slot, prompt):
        before = _snapshot(model, 4)
        nxt = model.prefill(prompt, 0, slot=slot)
        after = _snapshot(model, 4)
        for s in range(4):
            for l in range(L):
                for w in (0, 1):
                    if s != slot:
                        assert torch.equal(before[s][l][w], after[s][l][w]), ("prefill touched slot", s)
                    else:
                        assert torch.equal(before[s][l][w][:, len(prompt):], after[s][l][w][:, len(prompt):])
        pk, pv = state_of(slot, len(prompt))
        seqs[slot] = [nxt, len(prompt), pk, pv]

    prefill(1, [5, 6, 7, 8, 9])
    prefill(2, [100, 200, 300, 400, 500, 600, 700, 800, 900])
    prefill(3, [42, 43, 44])
    s0 = [11, 0, [None] * L, [None] * L]
    lg0 = torch.empty(g.vocab_size, dtype=torch.float32).pin_memory()
    for step in range(6):
        if step == 3:
            prefill(2, [1, 2, 3, 4])  # a new conversation in slot 2
        order = [1, 2, 3] if step % 2 == 0 else [3, 1, 2]
        toks = [seqs[s][0] for s in order]
        pos = [seqs[s][1] for s in order]
        lg = torch.empty((3, g.vocab_size), dtype=torch.float32).pin_memory()
        nxt = model.decode_batch_host(toks, pos, order, lg)
        for b, s in enumerate(order):
            tok, p, pk, pv = seqs[s]
            want, fk, fv = oracle_decode_step(model, tok, p, pk, pv)
            got = lg[b].numpy()
            assert rel_err(got, want) <= 1e-2, (step, s, rel_err(got, want))
            assert nxt[b] == int(np.argmax(got))
            for l in range(L):
                k = model.kv_cache(l, 0, s)[:, p].float().cpu().numpy()
                assert np.abs(k - fk[l][:, p]).max() <= 2e-2 * max(1.0, np.abs(fk[l]).max())
            seqs[s] = [nxt[b], p + 1, fk, fv]
        # the single-sequence path on slot 0 in between
        tok, p, pk, pv = s0
        n0 = model.decode_host(tok, p, lg0)
        want, fk, fv = oracle_decode_step(model, tok, p, pk, pv)
        assert rel_err(lg0.numpy(), want) <= 1e-2
        s0 = [n0, p + 1, fk, fv]
    model.close()
    ctx.close()


def test_host_entry_rejects_bad_requests():
    from tinychatengine_b200._lib import TceError

    ctx, model = _model("tiny-gqa", 128, n_slots=3)
    g = model.geom
    _fill_caches(model, 3, 3)
    model.decode_batch_host([1, 2], [4, 5], [0, 1])  # allocate + capture once
    before = _snapshot(model, 3)
    logits_before = model.batch_logits().cpu().clone()
    bad = [
        ([], [], []),                                    # batch 0
        ([1] * 9, [0] * 9, list(range(9))),              # batch 9
        ([1, 2], [3, 4], [0, 3]),                        # slot >= n_slots
        ([1, 2], [3, 4], [1, 1]),                        # the same slot twice
        ([1, 2], [3, -1], [0, 1]),                       # position < 0
        ([1, 2], [3, 128], [0, 1]),                      # position >= max_ctx
        ([-1, 2], [3, 4], [0, 1]),                       # token < 0
        ([1, g.vocab_size], [3, 4], [0, 1]),             # token >= vocab
        ([1, 2], [3, 4], [0, -1]),                       # slot < 0
    ]
    for toks, pos, slots in bad:
        with pytest.raises(TceError):
            model.decode_batch_host(toks, pos, slots)
        torch.cuda.synchronize()
        after = _snapshot(model, 3)
        for s in range(3):
            for l in range(g.num_layers):
                for w in (0, 1):
                    assert torch.equal(before[s][l][w], after[s][l][w])
        assert torch.equal(model.batch_logits().cpu(), logits_before)
    with pytest.raises(TceError):
        model.reserve_slots(0)
    assert model.ctx.L.tce_llama_kv_cache_slot(model.h, 3, 0, 0) is None
    model.close()
    ctx.close()


def test_device_entry_skips_bad_entries():
    """Entries with a token, position or slot out of range write no KV row anywhere; the valid entries of the same batch still match."""
    ctx, model = _model("tiny-mha", 256, n_slots=4)
    g = model.geom
    _fill_caches(model, 4, 77)
    before = _snapshot(model, 4)
    req = [(5, 10, 0), (g.vocab_size, 20, 1), (7, 256, 2), (9, 30, 4), (-3, 40, 3), (11, 64, 3), (13, 5, -1)]
    model.decode_batch(torch.tensor(req, dtype=torch.int32, device="cuda"))
    torch.cuda.synchronize()
    after = _snapshot(model, 4)
    lg = model.batch_logits()[: len(req)].cpu().numpy()
    valid = [0, 5]
    _check_step(model, before, after, [req[i] for i in valid], lg[valid], None, 4)
    model.close()
    ctx.close()


def test_deterministic_rows_do_not_depend_on_the_batch(monkeypatch):
    """TCE_DETERMINISTIC=1: permuting a batch permutes the logits rows bit for bit, and a row does not change when the other sequences do."""
    monkeypatch.setenv("TCE_DETERMINISTIC", "1")
    ctx, model = _model("tiny-gqa", 256, n_slots=8)
    g = model.geom
    _fill_caches(model, 8, 5)
    toks, pos, slots = [3, 99, 1000, 5, 42], [0, 37, 130, 200, 255], [0, 1, 2, 3, 4]

    def run(t, p, s):
        lg = torch.empty((len(t), g.vocab_size), dtype=torch.float32)
        model.decode_batch_host(t, p, s, lg)
        return lg

    ref = run(toks, pos, slots)
    perm = [3, 0, 4, 2, 1]
    got = run([toks[i] for i in perm], [pos[i] for i in perm], [slots[i] for i in perm])
    assert torch.equal(got, ref[perm])
    # sequence 0 next to other sequences (other slots, positions, tokens)
    other = run([toks[0], 7, 8, 9, 10], [pos[0], 3, 250, 64, 1], [slots[0], 5, 6, 7, 2])
    assert torch.equal(other[0], ref[0])
    model.close()
    ctx.close()


def _per_element_err(y, ref):
    y, ref = np.asarray(y, np.float64), np.asarray(ref, np.float64)
    m = np.abs(ref) > 1e-3 * np.abs(ref).max()
    return float(np.max(np.abs(y - ref)[m] / np.abs(ref)[m]))


@pytest.mark.parametrize("outlier", [False, True])
@pytest.mark.parametrize("oc,ic", [(256, 5120), (256, 13824), (128, 14336)])
@pytest.mark.parametrize("m", [2, 8])
def test_multicolumn_gemv_long_rows(m, oc, ic, outlier):
    """M = 2..8 rows at IC where the activation rows do not fit next to the weight ring whole (K-sliced), against the oracle; with one x1000
    outlier channel per 128-group, also per element."""
    from oracle import capi
    from tinychatengine_b200.runtime import Context, random_w4

    ctx = Context(0)
    dev = torch.device("cuda", 0)
    w, z, s = random_w4(oc, ic, dev, oc + ic + m, random_zeros=True)
    gen = torch.Generator(device=dev)
    gen.manual_seed(ic + m)
    x = torch.randn((m, ic), device=dev, generator=gen)
    if outlier:
        cg = torch.Generator(device="cpu")
        cg.manual_seed(3)
        ch = torch.randint(0, 128, (ic // 128,), generator=cg) + torch.arange(ic // 128) * 128
        x = x * 0.05
        x[:, ch.to(dev)] *= 1000.0
    x = x.to(torch.float16)
    y = ctx.w4a16_gemv(x, w, z, s)
    torch.cuda.synchronize()
    ref = capi.w4a16_gemv(x.cpu().numpy(), w.cpu().numpy().view(np.uint32), z.cpu().numpy().view(np.uint32), s.cpu().numpy())
    got = y.float().cpu().numpy()
    assert_w4_close(got, ref, f"M={m} {oc}x{ic} outlier={outlier}")
    if outlier:
        assert _per_element_err(got, ref) <= 1e-2
    # same bits when called again (ordered fix-up of the slice partials)
    y2 = ctx.w4a16_gemv(x, w, z, s)
    torch.cuda.synchronize()
    assert torch.equal(y, y2)
    ctx.close()


def test_tensor_parallel_model_is_unsupported():
    from tinychatengine_b200._lib import TceError
    from tinychatengine_b200.llama import GEOMETRIES, LlamaModel, shard_weights
    from tinychatengine_b200.runtime import Context

    ctx = Context(0)
    g = GEOMETRIES["tiny-gqa"]
    from tinychatengine_b200.llama import make_random_weights

    W = make_random_weights(g, torch.device("cuda", 0), 3)
    Wl, gl = shard_weights(W, g, 0, 2)
    model = LlamaModel(ctx, gl, max_ctx=128, weights=Wl, tp_rank=0, tp_size=2)
    L = ctx.L
    import ctypes as C

    assert L.tce_llama_reserve_slots(model.h, 2) == -2
    req = torch.zeros((1, 3), dtype=torch.int32, device="cuda")
    assert L.tce_llama_decode_batch(model.h, 1, C.c_void_p(req.data_ptr())) == -2
    one = (C.c_int * 1)(0)
    assert L.tce_llama_decode_batch_host(model.h, 1, one, one, one, None, None) == -2
    assert L.tce_llama_prefill_slot(model.h, 0, one, 1, 0, None, None) == -2
    assert L.tce_llama_batch_logits(model.h) is None
    with pytest.raises(TceError, match="tp_size"):
        model.reserve_slots(2)
    model.close()
    ctx.close()


def test_tensor_parallel_model_needs_the_persistent_kernel(monkeypatch):
    """tensor parallelism runs on the persistent kernel only: a tp_size = 2 shard built with TCE_PERSISTENT=0 is refused at creation"""
    monkeypatch.setenv("TCE_PERSISTENT", "0")
    from tinychatengine_b200._lib import TceError
    from tinychatengine_b200.llama import GEOMETRIES, LlamaModel, make_random_weights, shard_weights
    from tinychatengine_b200.runtime import Context

    ctx = Context(0)
    g = GEOMETRIES["tiny-gqa"]
    Wl, gl = shard_weights(make_random_weights(g, torch.device("cuda", 0), 3), g, 0, 2)
    with pytest.raises(TceError, match="persistent decode kernel"):
        LlamaModel(ctx, gl, max_ctx=128, weights=Wl, tp_rank=0, tp_size=2)
    ctx.close()


def test_multicolumn_gemv_grows_its_fixup_records():
    """45056 x 11008 at M = 2 takes 2816 row tiles x 6 K-slices of fix-up records, more than a context starts with: the launch grows them"""
    from oracle import capi
    from tinychatengine_b200.runtime import Context, random_w4

    ctx = Context(0)
    dev = torch.device("cuda", 0)
    oc, ic = 45056, 11008
    w, z, s = random_w4(oc, ic, dev, 91, random_zeros=True)
    gen = torch.Generator(device=dev)
    gen.manual_seed(92)
    x = torch.randn((2, ic), device=dev, generator=gen).to(torch.float16)
    y = ctx.w4a16_gemv(x, w, z, s)
    torch.cuda.synchronize()
    ref = capi.w4a16_gemv(x.cpu().numpy(), w.cpu().numpy().view(np.uint32), z.cpu().numpy().view(np.uint32), s.cpu().numpy())
    assert_w4_close(y.float().cpu().numpy(), ref, f"M=2 {oc}x{ic}")
    y2 = ctx.w4a16_gemv(x, w, z, s)
    torch.cuda.synchronize()
    assert torch.equal(y, y2)
    ctx.close()


def test_reserve_slots_keeps_count_and_table_together():
    """slots only grow; the cache of an existing slot survives a later reservation, and a slot past the count has no cache"""
    from tinychatengine_b200._lib import TceError

    ctx, model = _model("tiny-gqa", 128, n_slots=2)
    L = ctx.L
    assert L.tce_llama_kv_cache_slot(model.h, 1, 0, 0) is not None
    assert L.tce_llama_kv_cache_slot(model.h, 2, 0, 0) is None
    marker = torch.full_like(model.kv_cache(1, 1, 1), 0.25)
    model.kv_cache(1, 1, 1).copy_(marker)
    model.reserve_slots(5)
    model.reserve_slots(3)  # smaller: a no-op
    assert L.tce_llama_kv_cache_slot(model.h, 4, 1, 1) is not None
    assert L.tce_llama_kv_cache_slot(model.h, 5, 0, 0) is None
    assert torch.equal(model.kv_cache(1, 1, 1), marker)
    with pytest.raises(TceError):
        model.decode_batch_host([1], [0], [5])
    model.decode_batch_host([1, 2], [0, 0], [4, 1])  # the newest slot is in the device table
    assert torch.equal(model.kv_cache(1, 1, 1)[:, 1:], marker[:, 1:])
    model.close()
    ctx.close()
