#!/usr/bin/env python
"""BASELINE.json config 4: Llama-2-13B AWQ-INT4 prompt processing (2048 tokens) on one H100 through tce_llama_prefill.
Reports ms, tokens/s and linear-layer TFLOP/s (SURVEY.md 8(d): 2*n*12.688 G + attention 4*T^2*E*L un-masked count).
    python tools/prefill_bench.py [--model llama2-13b] [--n 2048] [--reps 3]
"""
import argparse
import json
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from tinychatengine_b200.llama import GEOMETRIES, LlamaModel  # noqa: E402
from tinychatengine_b200.runtime import Context  # noqa: E402


def prefill_once(ctx, dev, stream, model_name="llama2-13b", n=2048, peaks=None, reps=3, logits_out=None):
    """One prompt pass through tce_llama_prefill (host tokens in, greedy token out), best of `reps`, timed with CUDA events on `stream`."""
    g = GEOMETRIES[model_name]
    model = LlamaModel(ctx, g, max_ctx=n, seed=1)
    toks = [int(t) for t in torch.randint(0, g.vocab_size, (n,), generator=torch.Generator().manual_seed(7))]
    model.prefill(toks, 0, None)  # warm-up: allocations, module load
    torch.cuda.synchronize(dev)
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        model.prefill(toks, 0, None)
        e1.record(stream)
        torch.cuda.synchronize(dev)
        ts.append(e0.elapsed_time(e1) * 1e-3)
    if logits_out is not None:  # the same pass once more, untimed: the last position's logits row
        logits_out.append(torch.empty(g.vocab_size, dtype=torch.float32))
        model.prefill(toks, 0, logits_out[0])
    model.close()
    t = min(ts)
    hd = g.head_dim
    per_layer = (g.num_heads * hd + 2 * g.num_kv_heads * hd) * g.embed_dim + g.num_heads * hd * g.embed_dim + 3 * g.hidden_dim * g.embed_dim
    lin_flops = 2.0 * n * per_layer * g.num_layers
    attn_flops = 4.0 * n * n * g.num_heads * hd * g.num_layers
    out = {"model": model_name, "n": n, "ms": t * 1e3, "tok_per_s": n / t, "linear_tflops": lin_flops / t / 1e12,
           "linear_plus_attn_tflops": (lin_flops + attn_flops) / t / 1e12, "all_ms": [x * 1e3 for x in ts]}
    if peaks and "bf16_tflops" in peaks:
        out["frac_of_measured_bf16_burst"] = out["linear_tflops"] / float(peaks["bf16_tflops"])
        out["frac_of_measured_bf16_sustained"] = out["linear_tflops"] / float(peaks.get("bf16_tflops_sustained", peaks["bf16_tflops"]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="llama2-13b")
    ap.add_argument("--n", type=int, default=2048)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    pk = Path(__file__).resolve().parents[1] / "MEASURED_PEAKS.json"
    peaks = json.loads(pk.read_text()) if pk.exists() else None
    with torch.cuda.stream(stream):
        ctx = Context(0, stream)
        print(json.dumps(dict(prefill_once(ctx, dev, stream, args.model, args.n, peaks, args.reps), op="llama_prefill")))
        ctx.close()


if __name__ == "__main__":
    main()
