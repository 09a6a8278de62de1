#!/usr/bin/env python
"""Phase timeline of one W4A16 GEMV launch (option gemv_debug): where do the microseconds of a small GEMV go?"""
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from tinychatengine_b200.runtime import Context, random_w4  # noqa: E402

NAMES = ["entry", "tma_issued", "x_staged", "stage0_landed", "consumers_done", "epilogue_done", "first_flush"]


def main():
    dev = torch.device("cuda", 0)
    ctx = Context(0)
    ctx.set_option("gemv_debug", 1)
    for name, (oc, ic) in {"o_proj": (4096, 4096), "down": (4096, 14336), "gate_up": (28672, 4096), "lm_head": (128256, 4096)}.items():
        bufs = [random_w4(oc, ic, dev, 7 + i) for i in range(max(2, int(300e6 // (oc * ic // 2)) + 1))]
        x = torch.randn((1, ic), device=dev).to(torch.float16)
        y = torch.empty((1, oc), dtype=torch.float16, device=dev)
        for i in range(5):
            ctx.w4a16_gemv(x, *bufs[i % len(bufs)], out=y)
        torch.cuda.synchronize()
        out = np.zeros((ctx.num_sms, 8), np.uint64)
        n = ctx.L.tce_ctx_read_gemv_timing(ctx.h, out.ctypes.data_as(C.c_void_p), ctx.num_sms)
        t = out[:n].astype(np.int64)
        t0 = t[:, 0].min()
        rel = (t - t0) / 1e3
        print(f"== {name} {oc}x{ic}: per-phase time since the first CTA entry (us): min / median / max over {n} CTAs")
        for k, nm in enumerate(NAMES):
            col = rel[:, k]
            col = col[t[:, k] > 0]
            if len(col):
                print(f"   {nm:16s} {col.min():8.2f} {np.median(col):8.2f} {col.max():8.2f}")
        del bufs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
