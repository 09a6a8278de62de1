#!/usr/bin/env python
"""Batched decode on Llama-3-8B synthetic weights (32 layers, max_ctx 4096, random-filled caches): ms per step and aggregate tok/s at
B = 1, 2, 4, 8 sequences whose positions average 2048, against the batch-1 persistent step (tce_llama_decode) in the same process, and the
kernel-per-op batch-1 step (a second model on the same weights, built with TCE_PERSISTENT=0: the batched step at batch 1 on slot 0).

    python tools/batch_decode_bench.py --steps 50 --warmup 5 --out result.json
    python tools/batch_decode_bench.py --profile --out launches.json   # GEMV launches per batched step (torch.profiler, no timing)

Bytes per step are algorithmic: the packed weights once, plus each sequence's K/V rows (the positions before it, and its own row), over
the step time against the H100 SXM data-sheet HBM rate of 3.35 TB/s.  Card name and power limit are read with a query.
"""
import argparse
import json
import os
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

HBM_TBS = 3.35
BATCHES = (1, 2, 4, 8)


def positions(batch, mean=2048, spread=2048):
    """`batch` positions evenly spread over [mean - spread/2, mean + spread/2) with mean `mean`"""
    return [mean - spread // 2 + (spread * (2 * b + 1)) // (2 * batch) for b in range(batch)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, _, power = q.stdout.strip().splitlines()[0].partition(",") if q.returncode == 0 and q.stdout.strip() else (torch.cuda.get_device_name(0), "", "")
    return {"gpu": name.strip(), "power_limit": power.strip()}


def build(args):
    from tinychatengine_b200.llama import GEOMETRIES, LlamaModel
    from tinychatengine_b200.runtime import Context

    g = GEOMETRIES["llama3-8b"]
    ctx = Context(0)
    model = LlamaModel(ctx, g, max_ctx=args.max_ctx, seed=1)
    model.reserve_slots(max(BATCHES))
    gen = torch.Generator(device="cuda")
    gen.manual_seed(5)
    for s in range(max(BATCHES)):
        for l in range(g.num_layers):
            for which in (0, 1):
                c = model.kv_cache(l, which, s)
                c.copy_((torch.randn(c.shape, device="cuda", generator=gen) * 0.5).to(torch.float16))
    torch.cuda.synchronize()
    return ctx, model


def requests(g, batch):
    return torch.tensor([[(7919 * b + 13) % g.vocab_size, p, b] for b, p in enumerate(positions(batch))], dtype=torch.int32, device="cuda")


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def per_op_model(ctx, model, max_ctx):
    """a model on the same weights whose single-sequence step is one kernel per op, its slot-0 cache a copy of `model`'s"""
    from tinychatengine_b200.llama import LlamaModel

    old = os.environ.get("TCE_PERSISTENT")
    os.environ["TCE_PERSISTENT"] = "0"
    try:
        m = LlamaModel(ctx, model.geom, max_ctx=max_ctx, weights=model.W)
    finally:
        if old is None:
            del os.environ["TCE_PERSISTENT"]
        else:
            os.environ["TCE_PERSISTENT"] = old
    for l in range(model.geom.num_layers):
        for which in (0, 1):
            m.kv_cache(l, which).copy_(model.kv_cache(l, which))
    torch.cuda.synchronize()
    return m


def measure(args):
    from tinychatengine_b200.llama import kv_bytes_per_token, weight_bytes_per_token

    ctx, model = build(args)
    g = model.geom
    wbytes = weight_bytes_per_token(g)
    out = {**card(), "model": "llama3-8b synthetic", "layers": g.num_layers, "max_ctx": args.max_ctx, "steps": args.steps, "warmup": args.warmup,
           "hbm_tbs_datasheet": HBM_TBS, "rows": []}

    def row(kind, batch, pos, ms):
        b = wbytes + sum(kv_bytes_per_token(g, p) for p in pos)
        r = {"kind": kind, "batch": batch, "positions": pos, "ms_per_step": round(ms, 4), "tok_s": round(batch * 1e3 / ms, 1),
             "gb_per_step": round(b / 1e9, 3), "frac_of_hbm_datasheet": round(b / (ms * 1e-3) / (HBM_TBS * 1e12), 3)}
        out["rows"].append(r)
        print(json.dumps(r), flush=True)

    tp = torch.tensor([321, 2048], dtype=torch.int32, device="cuda")
    row("persistent batch-1 (tce_llama_decode)", 1, [2048], timed(lambda: model.decode(tp), args.steps, args.warmup))
    per_op = per_op_model(ctx, model, args.max_ctx)
    row("kernel-per-op batch-1 (tce_llama_decode, TCE_PERSISTENT=0)", 1, [2048], timed(lambda: per_op.decode(tp), args.steps, args.warmup))
    per_op.close()
    for batch in BATCHES:
        req = requests(g, batch)
        row("batched (tce_llama_decode_batch)", batch, positions(batch), timed(lambda: model.decode_batch(req), args.steps, args.warmup))
    model.close()
    ctx.close()
    return out


def profile(args):
    """kernel-per-op launches of one batched step (no graph, so every launch is its own profiler event)"""
    os.environ["TCE_NO_GRAPH"] = "1"
    from torch.profiler import ProfilerActivity
    from torch.profiler import profile as tprofile

    ctx, model = build(args)
    g = model.geom
    out = {**card(), "model": "llama3-8b synthetic", "layers": g.num_layers, "expected_gemv_launches": 4 * g.num_layers + 1, "rows": []}
    for batch in BATCHES:
        req = requests(g, batch)
        model.decode_batch(req)
        torch.cuda.synchronize()
        with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
            model.decode_batch(req)
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        r = {"batch": batch, "gemv_launches": sum("w4a16_gemv_kernel" in n for n in names), "kernels": len(names)}
        out["rows"].append(r)
        print(json.dumps(r), flush=True)
    model.close()
    ctx.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--max-ctx", type=int, default=4096)
    ap.add_argument("--profile", action="store_true", help="count GEMV launches per batched step instead of timing")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs an H100: there is no CPU path"
    res = profile(args) if args.profile else measure(args)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
