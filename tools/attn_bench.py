#!/usr/bin/env python
"""Stand-alone decode attention at Llama-3-8B heads (32 query / 8 KV heads, head_dim 128, max_ctx 4096): device time per launch of
tce_attn_decode (one row) and of tce_attn_span at n = 1, 2, 4 and 8 rows of one sequence, with the first row at positions 512, 2048 and
4095 (lowered to max_ctx - n for a span that would run past the cache), at --chunk cached rows per split (the context's default, 256).

    python tools/attn_bench.py --launches 200 --reps 5 --out attn.json

Each figure is CUDA events around one replay of a CUDA graph of --launches back-to-back calls, so the host's cost of a call is not in it,
divided by --launches: the median, min and max of --reps replays, in microseconds.  Every call rewrites the same K / V rows with the same
bits, so the launches are alike.  Prints one JSON line per figure and one with the card's name and power limit."""
import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

H, KVH, HD, MAX_CTX = 32, 8, 128, 4096
POSITIONS = (512, 2048, 4095)
SPANS = (1, 2, 4, 8)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, _, power = q.stdout.strip().splitlines()[0].partition(",") if q.returncode == 0 and q.stdout.strip() else (torch.cuda.get_device_name(0), "", "")
    return {"gpu": name.strip(), "power_limit": power.strip()}


def per_launch_us(call, launches, reps, stream):
    call()  # sizes the context's split workspace outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=stream):
        for _ in range(launches):
            call()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    us = []
    for _ in range(reps):
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        us.append(1e3 * e0.elapsed_time(e1) / launches)
    return {"median": round(statistics.median(us), 3), "min": round(min(us), 3), "max": round(max(us), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--chunk", type=int, default=256, help="the context's attn_chunk")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs an H100: there is no CPU path"
    from oracle import capi
    from tinychatengine_b200.runtime import Context

    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    c = Context(0, stream=stream)
    c.set_option("attn_chunk", args.chunk)
    gen = torch.Generator(device=dev).manual_seed(1)
    rnd = lambda *shape: (torch.randn(shape, generator=gen, device=dev) * 0.5).half()
    kc, vc = rnd(KVH, MAX_CTX, HD), rnd(KVH, MAX_CTX, HD)
    qkv = rnd(max(SPANS), (H + 2 * KVH) * HD)
    out = torch.empty((max(SPANS), H * HD), dtype=torch.float16, device=dev)
    cosb, sinb = (torch.from_numpy(t).to(dev) for t in capi.rope_tables(MAX_CTX, HD, 500000.0))
    alpha = 1.0 / np.sqrt(HD)
    res = {**card(), "heads": [H, KVH, HD], "max_ctx": MAX_CTX, "attn_chunk": args.chunk, "launches": args.launches,
           "reps": args.reps, "rows": []}

    def row(op, n, pos, call):
        r = {"op": op, "n": n, "pos0": pos, "us": per_launch_us(call, args.launches, args.reps, stream)}
        res["rows"].append(r)
        print(json.dumps(r), flush=True)

    for p in POSITIONS:
        pos = torch.tensor([p], dtype=torch.int32, device=dev)
        row("tce_attn_decode", 1, p, lambda: c.attn_decode(qkv[0], kc, vc, cosb, sinb, pos, out[0], alpha, H, KVH, HD, MAX_CTX))
        for n in SPANS:
            p0 = min(p, MAX_CTX - n)
            row("tce_attn_span", n, p0, lambda: c.attn_span(qkv[:n], kc, vc, cosb, sinb, out[:n], alpha, n, p0, H, KVH, HD, MAX_CTX))
    c.close()
    print(json.dumps({k: v for k, v in res.items() if k != "rows"}), flush=True)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
