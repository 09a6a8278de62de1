#!/usr/bin/env python
"""Micro-benchmark of the W4A16 GEMV (tce_w4a16_gemv) at the Llama decode shapes, sweeping kernel knobs.

Weights rotate over enough distinct buffers (> 2x L2) that no launch finds its matrix in L2, as in a real decode
step where 3.9 GB stream between two uses of the same matrix.  CUDA events, 3 warm-ups.
    python tools/gemv_bench.py [--reps 40]
"""
import argparse
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from tinychatengine_b200.runtime import Context, random_w4  # noqa: E402

SHAPES = {"o_proj 4096x4096": (4096, 4096), "qkv 6144x4096": (6144, 4096), "gate_up 28672x4096": (28672, 4096),
          "down 4096x14336": (4096, 14336), "down 4096x11008": (4096, 11008), "lm_head 128256x4096": (128256, 4096)}


def alg_bytes(oc, ic):
    return oc * ic // 2 + oc * (ic // 128) * 2 + oc * (ic // 128) // 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=40)
    ap.add_argument("--configs", default="8x1s4,8x1,16x1,8x2s4,8x2")
    ap.add_argument("--m", type=int, default=1)
    ap.add_argument("--shapes", default="", help="comma separated substrings to select shapes")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    ctx = Context(0)
    peak = 6569.6
    p = Path(__file__).resolve().parents[1] / "MEASURED_PEAKS.json"
    if p.exists():
        peak = json.loads(p.read_text())["hbm_gbs"]
    rows = []
    for name, (oc, ic) in SHAPES.items():
        if args.shapes and not any(k in name for k in args.shapes.split(",")):
            continue
        nbuf = max(2, int(300e6 // alg_bytes(oc, ic)) + 1)
        bufs = [random_w4(oc, ic, dev, 100 + i) for i in range(nbuf)]
        x = torch.randn((args.m, ic), device=dev).to(torch.float16)
        y = torch.empty((args.m, oc), dtype=torch.float16, device=dev)
        for cfg in args.configs.split(","):
            if cfg == "simple":
                ctx.set_option("gemv_impl", 0)
            else:
                base, _, st = cfg.partition("s")  # "8x1s4": 8 consumer warps, 1 CTA/SM, 4-stage ring ("s" omitted: deepest that fits)
                cw, cps = base.split("x")
                ctx.set_option("gemv_stages", int(st) if st else 0)
                ctx.set_option("gemv_impl", 1)
                ctx.set_option("gemv_consumer_warps", int(cw))
                ctx.set_option("gemv_ctas_per_sm", int(cps))
            side = torch.cuda.Stream()
            ctx.set_stream(side)
            with torch.cuda.stream(side):
                for i in range(3):
                    ctx.w4a16_gemv(x, *bufs[i % nbuf], out=y)
            side.synchronize()
            # the launches are replayed from a CUDA graph so that Python / launch overhead does not hide the kernel
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=side):
                for i in range(args.reps):
                    ctx.w4a16_gemv(x, *bufs[i % nbuf], out=y)
            graph.replay()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            graph.replay()
            e1.record()
            torch.cuda.synchronize()
            us = e0.elapsed_time(e1) * 1e3 / args.reps
            gbs = alg_bytes(oc, ic) / us / 1e3
            rows.append({"shape": name, "M": args.m, "config": cfg, "us": round(us, 2), "GB/s": round(gbs, 1), "frac_of_measured_peak": round(gbs / peak, 3)})
            print(json.dumps(rows[-1]), flush=True)
        del bufs
        torch.cuda.empty_cache()
    ctx.set_option("gemv_impl", 1)
    ctx.set_option("gemv_stages", 0)


if __name__ == "__main__":
    main()
