#!/usr/bin/env python
"""Persistent decode kernel vs the kernel-per-op graph path, step by step: greedy token, appended K/V rows and logits (1-layer models)."""
import os
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from tinychatengine_b200.llama import GEOMETRIES, LlamaGeometry, LlamaModel, make_random_weights  # noqa: E402
from tinychatengine_b200.runtime import Context  # noqa: E402


def run(g, mode, steps, W, max_ctx):
    os.environ["TCE_PERSISTENT"] = mode
    ctx = Context(0)
    model = LlamaModel(ctx, g, max_ctx=max_ctx, weights=W)
    lg = torch.empty(g.vocab_size, dtype=torch.float32)
    out = []
    tok = 3
    for pos in range(steps):
        nxt = model.decode_host(tok, pos, lg)
        out.append({"logits": lg.clone(), "next": nxt, "k": model.kv_cache(0, 0)[:, :pos + 1].float().cpu().clone(),
                    "v": model.kv_cache(0, 1)[:, :pos + 1].float().cpu().clone()})
        tok = (nxt * 7 + pos) % g.vocab_size
    model.close()
    ctx.close()
    return out


def main():
    name = sys.argv[1] if len(sys.argv) > 1 else "tiny-gqa"
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 4
    layers = int(sys.argv[3]) if len(sys.argv) > 3 else 1
    g0 = GEOMETRIES[name]
    g = LlamaGeometry(g0.name, layers, g0.num_heads, g0.num_kv_heads, g0.embed_dim, g0.hidden_dim, g0.vocab_size, g0.rms_eps, g0.rope_theta)
    W = make_random_weights(g, torch.device("cuda", 0), seed=5, random_zeros=True)
    a = run(g, "0", steps, W, 256)
    b = run(g, "1", steps, W, 256)
    for pos in range(steps):
        msg = [f"pos {pos}: next {a[pos]['next']} / {b[pos]['next']}"]
        for k in ("k", "v", "logits"):
            x, y = a[pos][k], b[pos][k]
            d = (x - y).abs().max().item() / max(x.abs().max().item(), 1e-9)
            msg.append(f"{k} {d:.2e}")
        print("  ".join(msg), flush=True)


if __name__ == "__main__":
    main()
