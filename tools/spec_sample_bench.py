"""Speculative sampling on Llama-3-8B shapes (random AWQ-INT4 weights), max_ctx 4096, context 2048, n_predict 128, at the reference chat
application's settings: temp 0.2 (its Llama-2 / CodeLLaMA path) and temp 0.7 (its Llama-3 path), both with top_k 40 and top_p 0.9.

For each temperature:
  * generate (tce_llama_generate) tok/s;
  * the sampled lookup loop (tce_llama_sample_lookup) at max_draft = 0, per token against generate: the cost of its per-step read-back;
  * the loop with no corpus, and with a corpus equal to that seed's generate output: tok/s, ids per step, accepted / drafted.
Every time is a host clock around synchronous calls: median, min and max of --reps windows after one warm-up call.

--profile instead times accept_kernel alone (tce_spec_accept on 128256-wide rows) at 1 and 8 rows, temp 0 and 0.7, with torch.profiler:
the mean device time per launch.  Run it as its own process: tracing slows the host.
Prints one JSON object; the card and its power limit are part of it."""
from __future__ import annotations

import argparse
import json
import statistics
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from spec_bench import gpu_info, spread, windows  # noqa: E402

SETTINGS = {"temp0.2": dict(temp=0.2, top_k=40, top_p=0.9), "temp0.7": dict(temp=0.7, top_k=40, top_p=0.9)}


def measure(model, ctx_len=2048, reps=5, n_predict=128, seed=11):
    V = model.geom.vocab_size
    prompt = [(7 * i + 3) % V for i in range(ctx_len)]
    model.prefill(prompt[:-1], 0)
    first, pos0, hist = prompt[-1], ctx_len - 1, prompt[-64:-1]
    res = {}
    for name, s in SETTINGS.items():
        kw = dict(history=hist, seed=seed, **s)
        G = model.generate(first, pos0, n_predict, **kw)
        gen = windows(lambda: model.generate(first, pos0, n_predict, **kw), reps)
        L0, st0 = model.generate_lookup(first, pos0, n_predict, max_draft=0, **kw)
        look0 = windows(lambda: model.generate_lookup(first, pos0, n_predict, max_draft=0, **kw), reps)
        r = {"generate_tok_s": spread([len(G) / x for x in gen]),
             "max_draft0_same_ids": L0 == G,
             "max_draft0_ms_per_token": spread(look0, 1e3 / len(L0)),
             "generate_ms_per_token": spread(gen, 1e3 / len(G)),
             "max_draft0_overhead_pct": 100.0 * (statistics.median(look0) / len(L0) / (statistics.median(gen) / len(G)) - 1.0)}
        r["loop"] = {}
        for level, corpus in (("none", []), ("generate_output", [first] + G)):
            ids, st = model.generate_lookup(first, pos0, n_predict, corpus=corpus, **kw)
            w = windows(lambda: model.generate_lookup(first, pos0, n_predict, corpus=corpus, **kw), reps)
            r["loop"][level] = {"tok_s": spread([len(ids) / x for x in w]), "ids": len(ids), **st, "tokens_per_step": len(ids) / max(1, st["steps"]),
                                "accepted_per_drafted": st["accepted"] / max(1, st["drafted"])}
        res[name] = r
    return res


def profile_accept(ctx, out_dir, launches=200):
    import torch
    from torch.profiler import ProfilerActivity, profile

    V = 128256
    g = torch.Generator(device="cuda")
    g.manual_seed(5)
    res = {}
    for rows in (1, 8):
        base = torch.randn((rows, V), device="cuda", generator=g)
        drafts = [int(t) for t in torch.argmax(base, dim=1)[:rows - 1].tolist()]
        for temp in (0.0, 0.7):
            kw = dict(top_k=40, top_p=0.9, temp=temp, repeat_penalty=1.1, repeat_last_n=64)
            lg = base.clone()
            for i in range(10):  # warm-up
                ctx.spec_accept(lg, drafts, list(range(64)), seed=i, draw_index=64, **kw)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for i in range(launches):
                    ctx.spec_accept(lg, drafts, list(range(64)), seed=i, draw_index=64, **kw)
            ev = [e for e in prof.events() if e.name.startswith("tce::(anonymous namespace)::accept_kernel") or "accept_kernel" in e.name]
            us = [e.device_time for e in ev] if ev and hasattr(ev[0], "device_time") else [e.cuda_time for e in ev]
            res[f"rows{rows}_temp{temp}"] = {"launches": len(us), "us_per_launch": spread(us) if us else None,
                                             "mean_us": statistics.mean(us) if us else None}
            if out_dir and rows == 8 and temp > 0:
                prof.export_chrome_trace(str(Path(out_dir) / "accept_kernel.pt.trace.json"))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--geom", default="llama3-8b")
    ap.add_argument("--ctx", type=int, default=2048)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--n-predict", type=int, default=128)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from tinychatengine_b200.runtime import Context

    ctx = Context(0)
    res = {"gpu": gpu_info()}
    if args.profile:
        res["accept_kernel"] = profile_accept(ctx, Path(args.out).parent if args.out else None)
    else:
        from tinychatengine_b200.llama import GEOMETRIES, LlamaModel

        model = LlamaModel(ctx, GEOMETRIES[args.geom], max_ctx=4096, seed=3)
        res.update({"geom": args.geom, "max_ctx": 4096, "ctx": args.ctx, "n_predict": args.n_predict,
                    **measure(model, args.ctx, args.reps, args.n_predict)})
        model.close()
    ctx.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
