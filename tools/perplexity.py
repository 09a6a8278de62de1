#!/usr/bin/env python
"""Perplexity of a model tree on a token file, scored in strided windows with tce_llama_score_batch.

    python tools/perplexity.py --dir models/LLaMA_3_8B_Instruct/INT4 --geom llama3-8b --tokens ids.npy --ctx 2048 --stride 512

`--tokens` is a .npy (or raw int32 .bin) array of token ids.  Windows start at 0, S, 2S, ... and hold at most C tokens; each is scored from
position 0 in its own KV-cache slot, up to 8 windows per call.  The first window counts every target, each later one only the tokens no
earlier window counted (its last S targets), so every token 1 .. N-1 is predicted exactly once, with at least C - S tokens of context
after the first window.  Prints exp(mean negative log-likelihood), the token count, the card and the wall time.
"""
import argparse
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

MAX_BATCH = 8  # TCE_LLAMA_MAX_BATCH


def window_plan(n_tokens: int, ctx: int, stride: int):
    """[(start, length, first_counted)]: window tokens [start, start + length); the targets it counts are the tokens
    first_counted .. start + length - 1 (position i of the window predicts token start + i + 1)."""
    if n_tokens < 2 or ctx < 2 or not 1 <= stride < ctx:
        raise ValueError(f"need at least 2 tokens and 1 <= stride < ctx (got n={n_tokens}, ctx={ctx}, stride={stride})")
    plan, counted_to = [], 1  # tokens below counted_to are already counted (token 0 has no prediction)
    start = 0
    while counted_to < n_tokens:
        end = min(start + ctx, n_tokens)
        plan.append((start, end - start, counted_to))
        counted_to = end
        start += stride
    return plan


def window_targets(tokens, start: int, length: int, first_counted: int):
    """Targets of one window: the next token where it is counted, -1 elsewhere (and on the last position)."""
    t = np.full(length, -1, dtype=np.int32)
    for i in range(length - 1):
        if start + i + 1 >= first_counted:
            t[i] = tokens[start + i + 1]
    return t


def score_tokens(model, tokens, ctx: int, stride: int):
    """(sum of negative log-likelihoods in float64, number of counted tokens) over the window plan."""
    tokens = np.asarray(tokens, dtype=np.int64)
    plan = window_plan(len(tokens), ctx, stride)
    model.reserve_slots(MAX_BATCH)
    nll, count = 0.0, 0
    for b0 in range(0, len(plan), MAX_BATCH):
        group = plan[b0:b0 + MAX_BATCH]
        prompts = [tokens[s:s + n].tolist() for s, n, _ in group]
        targets = [window_targets(tokens, s, n, f) for s, n, f in group]
        res = model.score_batch(prompts, list(range(len(group))), targets=targets)
        for (lp, _, _), tg in zip(res, targets):
            m = tg >= 0
            nll -= float(np.sum(lp[m].astype(np.float64)))
            count += int(m.sum())
    return nll, count


def load_tokens(path: str):
    p = Path(path)
    return np.load(p) if p.suffix == ".npy" else np.fromfile(p, dtype=np.int32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dir", required=True, help="model tree in the reference's on-disk INT4 layout")
    ap.add_argument("--geom", required=True, help="geometry name (tinychatengine_b200.llama.GEOMETRIES)")
    ap.add_argument("--tokens", required=True, help="int32 token ids, .npy or raw .bin")
    ap.add_argument("--ctx", type=int, default=2048, help="tokens per window (C)")
    ap.add_argument("--stride", type=int, default=512, help="start-to-start distance of the windows (S < C)")
    ap.add_argument("--max-ctx", type=int, default=0, help="KV-cache length of the model (default: --ctx)")
    args = ap.parse_args()
    import torch

    from tinychatengine_b200.llama import GEOMETRIES, LlamaModel
    from tinychatengine_b200.runtime import Context

    tokens = load_tokens(args.tokens)
    geom = GEOMETRIES[args.geom]
    if tokens.min() < 0 or tokens.max() >= geom.vocab_size:
        sys.exit(f"token ids outside [0, {geom.vocab_size})")
    ctx = Context(0)
    model = LlamaModel.load_dir(ctx, args.dir, geom, max_ctx=max(args.max_ctx, args.ctx))
    t0 = time.perf_counter()
    nll, count = score_tokens(model, tokens, args.ctx, args.stride)
    wall = time.perf_counter() - t0
    print(f"perplexity {np.exp(nll / count):.4f}  ({count} tokens, mean NLL {nll / count:.5f}, ctx {args.ctx}, stride {args.stride})")
    print(f"{torch.cuda.get_device_name(0)}: {wall:.2f} s")
    model.close()
    ctx.close()


if __name__ == "__main__":
    main()
