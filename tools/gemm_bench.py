#!/usr/bin/env python
"""Micro-benchmark of the wgmma GEMMs at the prefill shapes of BASELINE.json configs 3 and 4.
W4A16: Llama-2-13B prefill (M = 2048 tokens): expansion kernel + GEMM timed together (what tce_w4a16_gemm costs), and against
torch.matmul (cuBLAS fp16) on pre-expanded weights as the library yardstick.  W8A8: Llama-2-7B shapes, M = 2048.
    python tools/gemm_bench.py [--reps 10] [--m 2048]
"""
import argparse
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from tinychatengine_b200.runtime import Context, random_w4  # noqa: E402

W4_SHAPES = {"13B qkv 15360x5120": (15360, 5120), "13B o 5120x5120": (5120, 5120), "13B gate_up 27648x5120": (27648, 5120),
             "13B down 5120x13824": (5120, 13824), "8B gate_up 28672x4096": (28672, 4096)}
W8_SHAPES = {"7B qkv/o 4096x4096": (4096, 4096), "7B fc1 11008x4096": (11008, 4096), "7B fc2 4096x11008(K=11008)": (4096, 11008)}


def timeit(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1e-3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--m", type=int, default=2048)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    ctx = Context(0)
    M = args.m
    for name, (oc, ic) in W4_SHAPES.items():
        w, z, s = random_w4(oc, ic, dev, 5, random_zeros=True)
        x = torch.randn((M, ic), device=dev).to(torch.float16)
        y = torch.empty((M, oc), dtype=torch.float16, device=dev)
        t = timeit(lambda: ctx.w4a16_gemv(x, w, z, s, out=y, gemm=True), args.reps)
        w16 = torch.randn((oc, ic), device=dev).to(torch.float16)
        t_lib = timeit(lambda: torch.matmul(x, w16.t()), args.reps)
        fl = 2.0 * M * oc * ic
        print(json.dumps({"op": "w4a16_gemm", "shape": name, "M": M, "ms": round(t * 1e3, 4), "tflops": round(fl / t / 1e12, 1),
                          "cublas_fp16_ms": round(t_lib * 1e3, 4), "cublas_tflops": round(fl / t_lib / 1e12, 1)}), flush=True)
    for name, (n, k) in W8_SHAPES.items():
        if k % 128:
            continue
        A = torch.randint(-127, 128, (M, k), dtype=torch.int8, device=dev)
        B = torch.randint(-127, 128, (n, k), dtype=torch.int8, device=dev)
        b8 = torch.randint(-127, 128, (n,), dtype=torch.int8, device=dev)
        out = torch.empty((M, n), dtype=torch.int8, device=dev)
        t = timeit(lambda: ctx.w8a8_matmul(0, A, B, b8, 0.0005, 0.02, out=out), args.reps)
        ops = 2.0 * M * n * k
        print(json.dumps({"op": "w8a8_tc", "shape": name, "M": M, "ms": round(t * 1e3, 4), "tops": round(ops / t / 1e12, 1)}), flush=True)


if __name__ == "__main__":
    main()
