#!/usr/bin/env python
"""Batched generation on Llama-3-8B synthetic weights (32 layers, max_ctx 4096), in one process:

  (a) prompt pass of 8 prompts of 128 tokens: eight tce_llama_prefill_slot calls against one tce_llama_prefill_batch, in ms;
  (b) 8 sequences x 256 tokens with top-k sampling: tce_llama_generate_batch (batched step + device sampler per token, ids only cross PCIe)
      against a host loop of tce_llama_decode_batch_host with the [8][vocab] logits copied back plus one tce_sample per row, in aggregate
      tok/s.

    python tools/batch_generate_bench.py --repeats 3 --out result.json

Both sides of (a) and (b) run the same work on the same weights, alternating within each repeat.  Card name and power limit are read with
a query in the same run.
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

BATCH = 8
SAMPLING = dict(top_k=40, top_p=0.95, temp=0.8, repeat_penalty=1.1, frequency_penalty=0.0, presence_penalty=0.0, repeat_last_n=64)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, _, power = q.stdout.strip().splitlines()[0].partition(",") if q.returncode == 0 and q.stdout.strip() else (torch.cuda.get_device_name(0), "", "")
    return {"gpu": name.strip(), "power_limit": power.strip()}


def wall(fn):
    """host clock around a call that ends in a device synchronise"""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--prompt-len", type=int, default=128)
    ap.add_argument("--gen-len", type=int, default=256)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs an H100: there is no CPU path"
    from tinychatengine_b200.llama import GEOMETRIES, LlamaGeometry, LlamaModel
    from tinychatengine_b200.runtime import Context

    b = GEOMETRIES["llama3-8b"]
    g = LlamaGeometry("llama3-8b", args.layers, b.num_heads, b.num_kv_heads, b.embed_dim, b.hidden_dim, b.vocab_size, b.rms_eps, b.rope_theta, b.head_dim)
    ctx = Context(0)
    model = LlamaModel(ctx, g, max_ctx=4096, seed=1)
    model.reserve_slots(BATCH)
    gen = torch.Generator()
    gen.manual_seed(3)
    prompts = [torch.randint(0, g.vocab_size, (args.prompt_len,), generator=gen).tolist() for _ in range(BATCH)]
    slots = list(range(BATCH))
    out = {**card(), "model": "llama3-8b synthetic", "layers": g.num_layers, "batch": BATCH, "prompt_len": args.prompt_len, "gen_len": args.gen_len,
           "sampling": SAMPLING, "repeats": []}

    def prefill_per_call():
        return [model.prefill(p, 0, None, slot=s) for p, s in zip(prompts, slots)]

    def prefill_batch():
        return model.prefill_batch(prompts, slots)

    first = prefill_batch()
    reqs = [dict(first_token=first[s], pos0=args.prompt_len, slot=s, n_predict=args.gen_len, history=prompts[s][-64:], seed=100 + s, **SAMPLING)
            for s in range(BATCH)]

    def generate_batch():
        return model.generate_batch(reqs)

    lg = torch.empty((BATCH, g.vocab_size), dtype=torch.float32).pin_memory()

    def host_loop():
        hist = [list(r["history"]) for r in reqs]
        tok = [r["first_token"] for r in reqs]
        dev = model.batch_logits()
        for i in range(args.gen_len):
            model.decode_batch_host(tok, [args.prompt_len + i] * BATCH, slots, lg)
            for s in range(BATCH):
                t = ctx.sample(dev[s], hist[s][-64:], seed=reqs[s]["seed"], draw_index=len(hist[s]), **SAMPLING)
                hist[s].append(t)
                tok[s] = t
        return tok

    prefill_per_call(), generate_batch(), host_loop()  # warm-up: modules, graphs, expansion scratch
    for rep in range(args.repeats):
        r = {}
        r["prefill_per_call_ms"], _ = wall(prefill_per_call)
        r["prefill_batch_ms"], _ = wall(prefill_batch)
        ms, outs = wall(generate_batch)
        assert all(len(o) == args.gen_len for o in outs)
        r["generate_batch_ms"], r["generate_batch_tok_s"] = ms, BATCH * args.gen_len * 1e3 / ms
        ms, _ = wall(host_loop)
        r["host_loop_ms"], r["host_loop_tok_s"] = ms, BATCH * args.gen_len * 1e3 / ms
        r = {k: round(v, 2) for k, v in r.items()}
        out["repeats"].append(r)
        print(json.dumps(r), flush=True)
    print(json.dumps({k: v for k, v in out.items() if k != "repeats"}), flush=True)
    model.close()
    ctx.close()
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
