#!/usr/bin/env python
"""KV-cache row copies (tce_llama_kv_copy) at Llama-3-8B shapes (32 layers, synthetic weights, max_ctx 4096), in one process:

  (a) kernel time (CUDA events around --iters back-to-back launches after a warm-up, --repeats times) and achieved GB/s of
        * a 7-way fork of 2048 rows: 2048 rows read once, written 7 times;
        * the shift of a full slot with n_keep 4 (llama.cpp rule: n_discard 2046, rows [2050, 4096) move down to 4): 2046 rows read + written;
        * the same with n_keep 5 (n_discard 2045, 2046 rows moved): source and destination overlap by one row, the one-CTA-per-slab path;
      a row is L x {K, V} x KVH x 128 x 2 B = 128 KiB; bytes over time, and as a share of the 3.35 TB/s HBM3 data-sheet rate of the H100 SXM;
  (b) time to 8 slots holding the same 2048-token prompt: prefill + fork into 7 slots, against prefill_batch of 8 copies (host clock around
      synchronised calls, alternating);
  (c) the shift of (a) against a prompt pass of the rows it keeps (n_keep + the 2046 moved rows = 2050 tokens).

    python tools/kv_copy_bench.py --repeats 5 --out result.json

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

MAX_CTX, PROMPT, N_KEEP, HBM_BPS = 4096, 2048, 4, 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, _, power = q.stdout.strip().splitlines()[0].partition(",") if q.returncode == 0 and q.stdout.strip() else (torch.cuda.get_device_name(0), "", "")
    return {"gpu": name.strip(), "power_limit": power.strip()}


def wall(fn):
    """host clock (ms) around a call that ends in a device synchronise"""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def event_ms(fn, iters):
    """device time per launch (ms): CUDA events around `iters` launches on the model's stream (torch's current stream)"""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs an H100: there is no CPU path"
    from tinychatengine_b200.llama import GEOMETRIES, LlamaModel
    from tinychatengine_b200.runtime import Context

    g = GEOMETRIES["llama3-8b"]
    row_bytes = g.num_layers * 2 * g.num_kv_heads * g.head_dim * 2
    ctx = Context(0)
    model = LlamaModel(ctx, g, max_ctx=MAX_CTX, seed=1)
    model.reserve_slots(8)
    prompt = [int(t) for t in np.random.default_rng(0).integers(0, g.vocab_size, PROMPT)]
    moved = lambda keep: MAX_CTX - keep - (MAX_CTX - keep) // 2
    fork = lambda: model.fork(0, PROMPT, range(1, 8))
    shift = lambda keep: (lambda: model.kv_shift(0, MAX_CTX, keep))
    result = {"card": card(), "model": "llama3-8b (synthetic weights)", "layers": g.num_layers, "max_ctx": MAX_CTX, "row_bytes": row_bytes}

    # (a) kernel time and achieved bandwidth
    for name, fn, nbytes in [("fork_7x2048", fork, (1 + 7) * PROMPT * row_bytes), ("shift_full_slot_keep4", shift(N_KEEP), 2 * moved(N_KEEP) * row_bytes),
                             ("shift_full_slot_keep5_overlapping", shift(N_KEEP + 1), 2 * moved(N_KEEP + 1) * row_bytes)]:
        event_ms(fn, 5)  # warm-up
        ms = [event_ms(fn, args.iters) for _ in range(args.repeats)]
        best = min(ms)
        r = {"ms": ms, "bytes": nbytes, "gbps_best": nbytes / (best * 1e-3) / 1e9, "gbps_median": nbytes / (float(np.median(ms)) * 1e-3) / 1e9,
             "floor_ms_at_3.35TBps": nbytes / HBM_BPS * 1e3, "share_of_hbm_bound_median": nbytes / HBM_BPS / (float(np.median(ms)) * 1e-3)}
        result[name] = r
        print(json.dumps({name: r}), flush=True)

    # (b) 8 slots holding the same prompt
    one = lambda: (model.prefill(prompt, 0, slot=0), fork())
    batch = lambda: model.prefill_batch([prompt] * 8, list(range(8)))
    one(), batch()  # warm-up: modules, prompt buffers and expansion scratch at both sizes
    r = {"prefill_plus_fork_ms": [], "prefill_batch_8_ms": []}
    for _ in range(args.repeats):
        r["prefill_plus_fork_ms"].append(wall(one))
        r["prefill_batch_8_ms"].append(wall(batch))
    r["speedup_median"] = float(np.median(r["prefill_batch_8_ms"]) / np.median(r["prefill_plus_fork_ms"]))
    result["eight_slots_same_prompt"] = r
    print(json.dumps({"eight_slots_same_prompt": r}), flush=True)

    # (c) shift against a prompt pass of the kept rows
    kept = [int(t) for t in np.random.default_rng(1).integers(0, g.vocab_size, N_KEEP + moved(N_KEEP))]
    repass = lambda: model.prefill(kept, 0, slot=1)
    repass()
    r = {"kept_rows": N_KEEP + moved(N_KEEP), "prompt_pass_ms": [wall(repass) for _ in range(args.repeats)],
         "shift_kernel_ms_median": float(np.median(result["shift_full_slot_keep4"]["ms"]))}
    r["ratio_median"] = float(np.median(r["prompt_pass_ms"]) / r["shift_kernel_ms_median"])
    result["shift_vs_prompt_pass"] = r
    print(json.dumps({"shift_vs_prompt_pass": r}), flush=True)

    model.close()
    ctx.close()
    result["card_after"] = card()
    print(json.dumps({"card": result["card"], "card_after": result["card_after"]}))
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
