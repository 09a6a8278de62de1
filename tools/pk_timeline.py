#!/usr/bin/env python
"""Phase timeline of the persistent decode kernel (TCE_PK_DEBUG=1 makes it stamp %globaltimer per CTA and phase):
for each phase type, when the barrier opened, how long staging / consuming took, and the achieved HBM rate of the phase.
    TCE_PK_DEBUG=1 python tools/pk_timeline.py [--ctx 2048] [--model llama3-8b] [--layers 32]
"""
import argparse
import json
import os
import sys
from pathlib import Path

os.environ.setdefault("TCE_PK_DEBUG", "1")
import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from tinychatengine_b200.llama import GEOMETRIES, LlamaGeometry, LlamaModel, _tensor_from_ptr  # noqa: E402
from tinychatengine_b200.runtime import Context  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ctx", type=int, default=2048)
    ap.add_argument("--model", default="llama3-8b")
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    g0 = GEOMETRIES[args.model]
    g = LlamaGeometry(g0.name, args.layers, g0.num_heads, g0.num_kv_heads, g0.embed_dim, g0.hidden_dim, g0.vocab_size, g0.rms_eps, g0.rope_theta)
    ctx = Context(0)
    model = LlamaModel(ctx, g, max_ctx=4096, seed=1)
    for l in range(g.num_layers):
        model.kv_cache(l, 0).normal_(0, 0.5)
        model.kv_cache(l, 1).normal_(0, 0.5)
    ncta = ctx.num_sms
    nphase = 5 * g.num_layers + 1
    tp = torch.tensor([17, args.ctx], dtype=torch.int32, device="cuda")
    for _ in range(4):
        model.decode(tp)
    torch.cuda.synchronize()
    ptr = ctx.L.tce_llama_debug_buffer(model.h, 4)
    assert ptr, "no debug buffer: TCE_PK_DEBUG=1 must be set before the model is created"
    raw = _tensor_from_ptr(ptr, (ncta * nphase * 8 * 2,), torch.int32, 0).cpu().numpy().view(np.uint64).reshape(ncta, nphase, 8).astype(np.float64)
    if args.out:
        np.save(args.out.replace(".json", "") + "_raw.npy", raw)
    t0 = raw[:, 0, 0].min()
    T = (raw - t0) / 1e3  # us
    T[raw == 0] = np.nan
    hd = g.head_dim
    E, F, H, KVH = g.embed_dim, g.hidden_dim, g.num_heads, g.num_kv_heads
    bytes_of = {0: (H + 2 * KVH) * hd * E * 0.5 * 1.0390625, 1: 2 * KVH * hd * 2 * (args.ctx + 1), 2: E * H * hd * 0.5 * 1.0390625, 3: 2 * F * E * 0.5 * 1.0390625,
                4: E * F * 0.5 * 1.0390625}
    names = {0: "qkv", 1: "attn", 2: "o_proj", 3: "gate_up", 4: "down"}
    # the attention phase publishes its results from the consumer warps (no epilogue stamp): its "results written" is "phase left"
    for p in range(1, nphase - 1, 5):
        T[:, p, 3] = T[:, p, 2]
    total = np.nanmax(T[:, -1, 3]) if not np.all(np.isnan(T[:, -1, 3])) else np.nanmax(T)
    print(f"kernel span (first barrier-pass stamp -> last arrival): {total:.1f} us over {nphase} phases, ctx {args.ctx}")
    # attention sub-steps (medians over the CTAs that own chunks and over layers): time since the CTA entered the phase
    att = {4: [], 7: [], 5: [], 6: [], 2: []}
    for p in range(1, nphase - 1):
        if p % 5 == 1:
            for k in att:
                d = T[:, p, k] - T[:, p, 0]
                if not np.all(np.isnan(d)):
                    att[k].append(np.nanmedian(d))
    print("attention, since phase entry (median): q roped+bar %.2f  first stage landed %.2f  chunks done %.2f  partial written %.2f  phase left %.2f us" %
          tuple(float(np.median(att[k])) if att[k] else float("nan") for k in (4, 7, 5, 6, 2)))
    # the same sub-steps against the hand-off they wait for: the last q|k|v result of the layer (median over layers of the median / the
    # latest CTA).  The split merge ends with "phase left"; o_proj staging waits for the latest one.
    chain = {}
    for p in range(1, nphase - 1, 5):
        qkv_done = np.nanmax(T[:, p - 1, 3])
        for k, nm in ((4, "q_roped"), (7, "first_stage"), (5, "chunks_done"), (6, "partial_written"), (2, "merged")):
            d = T[:, p, k] - qkv_done
            if not np.all(np.isnan(d)):
                chain.setdefault(nm + "_med_us", []).append(np.nanmedian(d))
                chain.setdefault(nm + "_max_us", []).append(np.nanmax(d))
    chain = {k: float(np.median(v)) for k, v in chain.items()}
    print("attention, since the last q|k|v result (median / latest CTA): " +
          "  ".join(f"{nm} {chain[nm + '_med_us']:.2f}/{chain[nm + '_max_us']:.2f}" for nm in ("q_roped", "first_stage", "chunks_done", "partial_written", "merged")
                    if nm + "_med_us" in chain) + " us")
    acc = {}
    for p in range(1, nphase - 1):
        k = p % 5
        prev_done = np.nanmax(T[:, p - 1, 3])          # last CTA arrived at the previous barrier
        opened = T[:, p, 0]                             # each CTA saw the barrier open
        staged = T[:, p, 1]
        consumed = T[:, p, 2]
        arrived = T[:, p, 3]
        d = {"barrier_us": np.nanmedian(opened) - prev_done, "stage_us": np.nanmedian(staged - opened) if k != 1 else 0.0,
             "consume_us": np.nanmedian(consumed - (staged if k != 1 else opened)), "tail_us": np.nanmax(arrived) - np.nanmedian(consumed),
             "phase_us": np.nanmax(arrived) - prev_done, "skew_us": np.nanmax(consumed) - np.nanmin(consumed),
             "hop_us": (np.nanmedian(staged) if k != 1 else np.nanmedian(T[:, p, 4])) - prev_done, "etail_us": np.nanmedian(arrived - consumed)}
        acc.setdefault(k, []).append(d)
    summ = {}
    for k, lst in sorted(acc.items()):
        m = {key: float(np.median([d[key] for d in lst])) for key in lst[0]}
        m["GBps"] = bytes_of[k] / m["phase_us"] / 1e3
        m["hbm_floor_us"] = bytes_of[k] / 3.35e6  # H100 SXM data-sheet HBM3 rate, 3.35 TB/s
        summ[names[k]] = m
        print(f"{names[k]:8s} phase {m['phase_us']:6.2f} us (HBM floor {m['hbm_floor_us']:5.2f})  barrier {m['barrier_us']:5.2f}  stage {m['stage_us']:5.2f}  "
              f"consume {m['consume_us']:6.2f}  tail {m['tail_us']:5.2f}  skew {m['skew_us']:5.2f}  hop {m['hop_us']:5.2f}  etail {m['etail_us']:5.2f}  -> {m['GBps']:7.0f} GB/s")
    # GEMV sub-steps of consumer warp 0 (slots 4..6) and of the epilogue warp (7, then 3), since the CTA's input was staged (slot 1).
    # Means over the CTAs that own tiles and over the layers: the timer ticks far coarser than one ring stage, a mean over thousands of
    # intervals that start at unrelated moments still resolves it.  per_stage: (last stage released - first stage landed) / stages: slot 4
    # is stamped when the first stage has landed, before it is computed, and slot 5 after the last one is released, so the interval holds
    # the compute of every stage and, where a tile is one box (q|k|v, o_proj, gate|up at Llama-3-8B), the hand-offs of all tiles but the
    # last.  With the stages already in shared memory (q|k|v and o_proj: at most 3 per CTA, loaded while the previous phases ran) it is the
    # consumer-only cost of a ring stage.  Stages per CTA follow the kernel's layout: the two CTAs of a cluster walk the tiles of their pair
    # (partition over num_sms / 2), each over its half of the 128-groups in boxes of 16 groups (k_range) of a 32-row tile, one box per ring stage.
    tick = np.gcd.reduce(np.unique(raw[raw > 0] - raw[raw > 0].min()).astype(np.int64))
    ops = {0: (E, (H + 2 * KVH) * hd // 32), 2: (H * hd, E // 32), 3: (E, 2 * F // 32), 4: (F, E // 32)}  # IC, 32-row tiles
    sub = {}
    npair = ncta // 2
    for k, (ic, ntiles) in ops.items():
        ng, h = ic // 128, (ic // 128 + 1) // 2  # groups of a row; rank 0 takes the first h, rank 1 the rest
        tiles = np.array([(ntiles * (c // 2 + 1)) // npair - (ntiles * (c // 2)) // npair for c in range(ncta)])
        nb = np.array([(h if c % 2 == 0 else ng - h) + 15 for c in range(ncta)]) // 16  # boxes per tile
        nst = tiles * nb
        rows = {"first_landed": [], "last_released": [], "handed": [], "epi_last_in": [], "published": [], "per_stage": []}
        for p in range(k, nphase - 1, 5):
            base = T[:, p, 1]
            for nm, slot in (("first_landed", 4), ("last_released", 5), ("handed", 6), ("epi_last_in", 7), ("published", 3)):
                rows[nm].append(T[:, p, slot] - base)
            ok = nst > 0
            rows["per_stage"].append((T[ok, p, 5] - T[ok, p, 4]) / nst[ok])
        m = {nm: float(np.nanmean(np.concatenate(v))) for nm, v in rows.items()}
        m["stages_per_cta"] = f"{nst.min()}-{nst.max()}"
        sub[names[k]] = m
    print(f"GEMV sub-steps since staged (means, us; timer tick {tick} ns):")
    for nm, m in sub.items():
        print(f"  {nm:8s} stages/CTA {m['stages_per_cta']:6s} first landed {m['first_landed']:5.2f}  last released {m['last_released']:5.2f}  "
              f"handed {m['handed']:5.2f}  epilogue has last {m['epi_last_in']:5.2f}  published {m['published']:5.2f}  -> {1e3 * m['per_stage']:6.0f} ns/stage")
    summ["gemv_substeps"] = sub
    summ["timer_tick_ns"] = int(tick)
    lm = nphase - 1
    prev_done = np.nanmax(T[:, lm - 1, 3])
    print(f"lm_head  phase {np.nanmax(T[:, lm, 3]) - prev_done:6.2f} us")
    summ["lm_head_us"] = float(np.nanmax(T[:, lm, 3]) - prev_done)
    summ["kernel_us"] = float(total)
    summ["attention_chain"] = chain
    if args.out:
        Path(args.out).write_text(json.dumps(summ, indent=1))
    model.close()
    ctx.close()


if __name__ == "__main__":
    main()
