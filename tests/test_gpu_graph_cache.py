"""Cached CUDA graphs against eager execution: every entry point that replays a graph (decode_host, decode, decode_batch_host, decode_batch,
generate, generate_batch) gives bit-identical logits, greedy ids and KV rows to the same model built with TCE_NO_GRAPH=1, across the first call of a
key (eager run + capture), replays, a new request tensor, an option change, batch-size changes and slot growth."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _run(monkeypatch, graphs, script, persistent="1"):
    """script(ctx, model) -> (outputs, slots used); returns the outputs and the KV caches of those slots.  TCE_DETERMINISTIC=1: no RED.ADD
    in the GEMVs, so two runs of the same work agree bit for bit"""
    from tinychatengine_b200.llama import GEOMETRIES, LlamaModel
    from tinychatengine_b200.runtime import Context

    monkeypatch.setenv("TCE_DETERMINISTIC", "1")
    monkeypatch.setenv("TCE_PERSISTENT", persistent)
    if graphs:
        monkeypatch.delenv("TCE_NO_GRAPH", raising=False)
    else:
        monkeypatch.setenv("TCE_NO_GRAPH", "1")
    ctx = Context(0)
    model = LlamaModel(ctx, GEOMETRIES["tiny-gqa"], max_ctx=128, seed=13, random_zeros=True)
    assert (model.kernels_per_step == 1) == (persistent == "1")
    try:
        out, slots = script(ctx, model)
        torch.cuda.synchronize()
        kv = [model.kv_cache(l, w, s).cpu().clone() for s in range(slots) for l in range(model.geom.num_layers) for w in (0, 1)]
    finally:
        model.close()
        ctx.close()
    return out, kv


def _assert_same(monkeypatch, script, persistent="1"):
    got, got_kv = _run(monkeypatch, True, script, persistent)
    want, want_kv = _run(monkeypatch, False, script, persistent)
    assert len(got) == len(want) and len(got_kv) == len(want_kv)
    for i, (a, b) in enumerate(zip(got, want)):
        if isinstance(a, torch.Tensor):
            assert torch.equal(a, b), f"output {i} differs between graph replay and eager execution"
        else:
            assert a == b, (i, a, b)
    for i, (a, b) in enumerate(zip(got_kv, want_kv)):
        assert torch.equal(a, b), f"KV cache {i} differs between graph replay and eager execution"


@pytest.mark.parametrize("persistent", ["1", "0"])
def test_single_sequence_graphs_match_eager(monkeypatch, persistent):
    def script(ctx, model):
        V = model.geom.vocab_size
        out = []
        lg = torch.empty(V, dtype=torch.float32)
        pos = 0
        for tok in (3, 77, 1000):  # host entry: eager + capture, then two replays
            out += [model.decode_host(tok, pos, lg), lg.clone()]
            pos += 1
        a = torch.tensor([5, pos], dtype=torch.int32, device="cuda")
        for tok in (5, 900, 17):  # device entry on one tensor, rewritten in place between calls
            a.copy_(torch.tensor([tok, pos], dtype=torch.int32))
            model.decode(a)
            out.append(model.logits().cpu().clone())
            pos += 1
        b = torch.tensor([0, 0], dtype=torch.int32, device="cuda")  # a new tensor: the result follows it, not `a`
        a.copy_(torch.tensor([1, 0], dtype=torch.int32))
        for tok in (256, 999, 42):
            b.copy_(torch.tensor([tok, pos], dtype=torch.int32))
            model.decode(b)
            out.append(model.logits().cpu().clone())
            pos += 1
        for pdl in (0, 1):  # an option change makes every captured graph stale
            ctx.set_option("use_pdl", pdl)
            for tok in (7, 8, 9):
                out += [model.decode_host(tok, pos, lg), lg.clone()]
                pos += 1
                b.copy_(torch.tensor([tok + 1, pos], dtype=torch.int32))
                model.decode(b)
                out.append(model.logits().cpu().clone())
                pos += 1
        model.reserve_slots(3)  # a new slot table: graphs that read the old one must not be replayed
        for tok in (31, 32, 33):
            out += [model.decode_host(tok, pos, lg), lg.clone()]
            pos += 1
            b.copy_(torch.tensor([tok + 1, pos], dtype=torch.int32))
            model.decode(b)
            out.append(model.logits().cpu().clone())
            pos += 1
        return out, 1

    _assert_same(monkeypatch, script, persistent)


def test_batched_graphs_match_eager(monkeypatch):
    def script(ctx, model):
        V = model.geom.vocab_size
        model.reserve_slots(3)
        pos = [0] * 8
        out = []

        def host(slots, want_logits=True):
            toks = [(37 * s + pos[s] * 11 + 1) % V for s in slots]
            lg = torch.empty((len(slots), V), dtype=torch.float32) if want_logits else None
            out.append(model.decode_batch_host(toks, [pos[s] for s in slots], slots, lg))
            if want_logits:
                out.append(lg)
            for s in slots:
                pos[s] += 1

        def device(req, slots):
            req.copy_(torch.tensor([[(53 * s + pos[s] * 7 + 2) % V, pos[s], s] for s in slots], dtype=torch.int32))
            model.decode_batch(req)
            out.append(model.batch_logits()[: len(slots)].cpu().clone())
            for s in slots:
                pos[s] += 1

        for _ in range(3):
            host([2, 0])
        for _ in range(3):
            host([2, 0], want_logits=False)  # the graph without the logits copy
        for _ in range(3):
            host([1, 2, 0])  # another batch size
        r1 = torch.zeros((2, 3), dtype=torch.int32, device="cuda")
        for _ in range(3):
            device(r1, [0, 1])
        r2 = torch.zeros((2, 3), dtype=torch.int32, device="cuda")  # a new request tensor: the result follows it, not r1
        r1.copy_(torch.tensor([[1, 0, 2], [2, 0, 1]], dtype=torch.int32))
        for _ in range(3):
            device(r2, [1, 0])
        model.reserve_slots(5)  # growing the slots drops the batch graphs (they hold the old slot table)
        for _ in range(3):
            host([4, 2, 3])
        for _ in range(3):
            device(r2, [3, 4])
        ctx.set_option("use_pdl", 0)
        for _ in range(3):
            host([4, 2, 3])
            device(r2, [0, 4])
        return out, 5

    _assert_same(monkeypatch, script)


@pytest.mark.parametrize("persistent", ["1", "0"])
def test_generate_graphs_match_eager(monkeypatch, persistent):
    def script(ctx, model):
        out = [model.generate(11, 0, 20, seed=1, top_k=20)]  # first token eager + capture, then replays
        out.append(model.generate(12, 20, 24, temp=0.0))  # the cached graph from the first call
        ctx.set_option("use_pdl", 0)  # an option change makes the graph stale
        out.append(model.generate(13, 44, 18, seed=3, top_k=40, top_p=0.9))
        model.reserve_slots(3)  # a new slot table drops it
        out.append(model.generate(14, 62, 17, seed=4))
        out.append(model.generate(15, 79, 16, seed=5, temp=0.0))
        return out, 1

    _assert_same(monkeypatch, script, persistent)


def test_generate_batch_graphs_match_eager(monkeypatch):
    def script(ctx, model):
        model.reserve_slots(3)
        rows = [dict(first_token=11, pos0=0, slot=1, n_predict=20, seed=1, top_k=20),
                dict(first_token=12, pos0=0, slot=0, n_predict=24, seed=2, temp=0.0),
                dict(first_token=13, pos0=0, slot=2, n_predict=18, seed=3, top_k=40, top_p=0.9)]
        out = [model.generate_batch(rows[:2])]  # first token eager + capture, then replays
        rows = [dict(r, first_token=r["first_token"] + 1, pos0=r["pos0"] + 30) for r in rows]
        out.append(model.generate_batch(rows[:2]))  # the cached graph from the first call
        out.append(model.generate_batch(rows[2:] + rows[:1]))  # another batch size
        model.reserve_slots(4)
        rows = [dict(r, pos0=r["pos0"] + 30) for r in rows] + [dict(first_token=5, pos0=0, slot=3, n_predict=17, seed=4)]
        out.append(model.generate_batch(rows))
        ctx.set_option("use_pdl", 0)
        rows = [dict(r, pos0=r["pos0"] + 25) for r in rows]
        out.append(model.generate_batch(rows))
        return out, 4

    _assert_same(monkeypatch, script)
