"""Speculative decoding on Llama-3-8B shapes (random AWQ-INT4 weights), max_ctx 4096, context 2048:

  * the span step (tce_llama_decode_span_host) at n = 1..8 tokens of one slot, against the persistent single-sequence step and the batched
    step (tce_llama_decode_batch_host) at B = n sequences;
  * the greedy prompt-lookup loop (tce_llama_generate_lookup) at three acceptance levels: no corpus, a corpus holding the exact greedy
    continuation, and one with every third token of it replaced;
  * the loop at max_draft = 0 (one host read-back per step) against generate(temp = 0) (one read-back per 16 tokens), per token: the cost
    of the loop's host round trip shows as their difference;
  * the break-even acceptance: the accepted drafts per step at which a span step of n = d + 1 rows matches d + 1 one-token steps.

Every time is a host clock around synchronous calls (each returns after its device work and copies): the median, min and max of --reps
windows.
Prints one JSON object; the card and its power limit are part of it."""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def windows(fn, reps):
    """seconds of `reps` calls of fn after one warm-up call"""
    fn()
    out = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        out.append(time.perf_counter() - t)
    return out


def spread(xs, scale=1.0):
    return {"median": scale * statistics.median(xs), "min": scale * min(xs), "max": scale * max(xs)}


def timed(fn, steps, reps):
    """median seconds per call over `reps` windows of `steps` calls"""
    def window():
        for _ in range(steps):
            fn()
    return statistics.median(windows(window, reps)) / steps


def measure(model, ctx_len=2048, steps=20, reps=5, n_predict=128):
    g = model.geom
    V = g.vocab_size
    toks = [(1009 * i + 7) % V for i in range(8)]
    res = {"persistent_step_ms": 1e3 * timed(lambda: model.decode_host(toks[0], ctx_len), steps, reps)}
    res["span_ms"] = {}
    res["batch_ms"] = {}
    for n in range(1, 9):
        res["span_ms"][n] = 1e3 * timed(lambda: model.decode_span(toks[:n], ctx_len, 0), steps, reps)
        res["batch_ms"][n] = 1e3 * timed(lambda: model.decode_batch_host(toks[:n], [ctx_len] * n, list(range(n))), steps, reps)
    # the loop: a prompt of ctx_len tokens in slot 0, then n_predict greedy ids
    prompt = [(7 * i + 3) % V for i in range(ctx_len)]
    model.prefill(prompt[:-1], 0)
    first, pos0, hist = prompt[-1], ctx_len - 1, prompt[-64:-1]
    G = model.generate(first, pos0, n_predict, history=hist, temp=0.0)
    G0, st0 = model.generate_lookup(first, pos0, n_predict, history=hist, max_draft=0)
    gen = windows(lambda: model.generate(first, pos0, n_predict, history=hist, temp=0.0), reps)
    look0 = windows(lambda: model.generate_lookup(first, pos0, n_predict, history=hist, max_draft=0), reps)
    t_gen, t_l0 = statistics.median(gen) / len(G), statistics.median(look0) / st0["steps"]
    res["generate_greedy_ms_per_token"] = spread(gen, 1e3 / len(G))
    res["lookup_max_draft0_ms_per_step"] = spread(look0, 1e3 / st0["steps"])
    res["lookup_max_draft0_minus_generate_ms"] = 1e3 * (t_l0 - t_gen)
    res["lookup_max_draft0_same_ids"] = G0 == G
    half = [t if i % 3 else (t + 1) % V for i, t in enumerate(G)]
    levels = {"none": [], "exact": [first] + G, "every_third_replaced": [first] + half}
    res["loop"] = {}
    for name, corpus in levels.items():
        ids, st = model.generate_lookup(first, pos0, n_predict, history=hist, corpus=corpus)
        w = windows(lambda: model.generate_lookup(first, pos0, n_predict, history=hist, corpus=corpus), reps)
        res["loop"][name] = {"tok_s": spread([len(ids) / x for x in w]), "ids": len(ids), **st, "tokens_per_step": len(ids) / max(1, st["steps"]),
                             "same_ids_as_greedy": ids == G}
    res["greedy_tok_s"] = spread([len(G) / x for x in gen])

    t1 = t_l0
    # accepted drafts per step at which a span step of d + 1 rows breaks even with one-token steps (round trip included on both sides)
    res["break_even_accepted"] = {d: (res["span_ms"][d + 1] / 1e3 + (t_l0 - t_gen)) / t1 - 1 for d in range(1, 8)}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--geom", default="llama3-8b")
    ap.add_argument("--ctx", type=int, default=2048)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--n-predict", type=int, default=128)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from tinychatengine_b200.llama import GEOMETRIES, LlamaModel
    from tinychatengine_b200.runtime import Context

    ctx = Context(0)
    model = LlamaModel(ctx, GEOMETRIES[args.geom], max_ctx=4096, seed=3)
    model.reserve_slots(8)
    res = {"gpu": gpu_info(), "geom": args.geom, "max_ctx": 4096, "ctx": args.ctx,
           **measure(model, args.ctx, args.steps, args.reps, args.n_predict)}
    model.close()
    ctx.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
