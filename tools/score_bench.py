#!/usr/bin/env python
"""Prompt scoring against the plain prompt pass, synthetic weights, in one process:

  * Llama-3-8B (32 layers): 1 x 2048 tokens and 8 x 256;  Llama-2-13B (40 layers): 1 x 2048.
  * For each, tce_llama_prefill_batch and tce_llama_score_batch on the same prompts, alternating, after a warm-up of both (ms per call,
    host clock around the synchronous calls).
  * The lm_head chunks alone: one score_batch call under torch.profiler; the device time of the log-softmax GEMM kernels
    (gemm_wg_kernel<..., EpiRowStats>), of the merge kernel and of the chunk expansions, and the GEMM's achieved TFLOP/s for 2 n V E.

    python tools/score_bench.py --repeats 3 --out result.json

Card name and power limit are read with a query in the same run.
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

CASES = [("llama3-8b", 1, 2048), ("llama3-8b", 8, 256), ("llama2-13b", 1, 2048)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, _, power = q.stdout.strip().splitlines()[0].partition(",") if q.returncode == 0 and q.stdout.strip() else (torch.cuda.get_device_name(0), "", "")
    return {"gpu": name.strip(), "power_limit": power.strip()}


def wall(fn):
    """host clock around a call that ends in a device synchronise"""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def linear_flops(g, n):
    """2 n x (weights of every linear of the prompt pass), without the lm_head"""
    hd = g.head_dim
    per_layer = (g.num_heads + 2 * g.num_kv_heads) * hd * g.embed_dim + g.embed_dim * g.num_heads * hd + 3 * g.hidden_dim * g.embed_dim
    return 2.0 * n * per_layer * g.num_layers


def kernel_times(model, prompts, slots):
    """device time (ms) per kernel class of one score_batch call"""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        model.score_batch(prompts, slots)
        torch.cuda.synchronize()
    out = {"lm_gemm_ms": 0.0, "lm_merge_ms": 0.0, "expand_ms": 0.0, "lm_gemm_launches": 0}
    for e in prof.key_averages():
        t = e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
        if "EpiRowStats" in e.key:
            out["lm_gemm_ms"] += t
            out["lm_gemm_launches"] += e.count
        elif "lm_stats_merge" in e.key:
            out["lm_merge_ms"] += t
        elif "w4_expand" in e.key:
            out["expand_ms"] += t
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs an H100: there is no CPU path"
    from tinychatengine_b200.llama import GEOMETRIES, LlamaModel
    from tinychatengine_b200.runtime import Context

    result = {"card": card(), "cases": []}
    ctx = Context(0)
    for name in dict.fromkeys(c[0] for c in CASES):
        g = GEOMETRIES[name]
        model = LlamaModel(ctx, g, max_ctx=2048, seed=1)
        model.reserve_slots(8)
        for _, n_seqs, length in (c for c in CASES if c[0] == name):
            rng = np.random.default_rng(n_seqs)
            prompts = [[int(t) for t in rng.integers(0, g.vocab_size, length)] for _ in range(n_seqs)]
            slots = list(range(n_seqs))
            n = n_seqs * length
            prefill = lambda: model.prefill_batch(prompts, slots)
            score = lambda: model.score_batch(prompts, slots)
            prefill(), score()  # warm-up: modules, expansion scratch, scoring buffers
            r = {"model": name, "layers": g.num_layers, "prompts": n_seqs, "tokens_each": length, "prefill_batch_ms": [], "score_batch_ms": []}
            for _ in range(args.repeats):
                r["prefill_batch_ms"].append(wall(prefill))
                r["score_batch_ms"].append(wall(score))
            r.update(kernel_times(model, prompts, slots))
            lm_flop = 2.0 * n * g.vocab_size * g.embed_dim
            r["lm_head_tflop"] = lm_flop / 1e12
            r["linear_tflop"] = linear_flops(g, n) / 1e12
            r["lm_gemm_tflops"] = lm_flop / (r["lm_gemm_ms"] * 1e-3) / 1e12 if r["lm_gemm_ms"] else None
            print(json.dumps(r), flush=True)
            result["cases"].append(r)
        model.close()
        torch.cuda.empty_cache()
    ctx.close()
    result["card"] = card()  # again after the load
    print(json.dumps(result["card"]))
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
