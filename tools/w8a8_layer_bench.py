#!/usr/bin/env python
"""BASELINE.json config 3: one Int8OPTDecoderLayer-shaped W8A8 layer at Llama-2-7B shapes (E 4096, F 11008, 32 heads x 128) on one
H100, end to end through the C ABI in the order of Int8OPTDecoderLayer::forward (llm/src/nn_modules/Int8OPTDecoderLayer.cc:24-59):
LayerNormQ -> q/k/v (W8A8B8O8Linear) -> tce_opt_int8_attention (int8 KV cache in place) -> out_proj (W8A8BFP32OFP32Linear) -> residual
add -> LayerNormQ -> fc1 (W8A8B8O8LinearReLU) -> fc2 (W8A8BFP32OFP32Linear) -> residual add.  M = 1 (decode at ctx 1024: HBM-bound, GB/s
of int8 weights) and M = 2048 (prompt: tensor-bound, TOP/s).  Layers rotate over > 2x L2 of distinct weights.
    python tools/w8a8_layer_bench.py
"""
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

E, F, H, HD = 4096, 11008, 32, 128


class Layer:
    def __init__(self, dev, seed):
        g = torch.Generator(device=dev)
        g.manual_seed(seed)

        def w(n, k):
            return torch.randint(-127, 128, (n, k), dtype=torch.int8, device=dev, generator=g)

        def b8(n):
            return torch.randint(-127, 128, (n,), dtype=torch.int8, device=dev, generator=g)

        self.wq, self.wk, self.wv, self.wo = w(E, E), w(E, E), w(E, E), w(E, E)
        self.bq, self.bk, self.bv = b8(E), b8(E), b8(E)
        self.bo = torch.randn(E, device=dev, generator=g)
        self.w1, self.b1 = w(F, E), b8(F)
        self.w2, self.b2 = w(E, F), torch.randn(E, device=dev, generator=g)
        self.ln1w, self.ln1b = 1 + 0.1 * torch.randn(E, device=dev, generator=g), torch.randn(E, device=dev, generator=g)
        self.ln2w, self.ln2b = 1 + 0.1 * torch.randn(E, device=dev, generator=g), torch.randn(E, device=dev, generator=g)

    @staticmethod
    def weight_bytes():
        return 4 * E * E + 2 * E * F

    @staticmethod
    def ops(M):
        return 2 * M * (4 * E * E + 2 * E * F)


def forward(ctx, L, x, kcache, vcache, past, bufs):
    """x fp32 [M][E] -> fp32 [M][E]; kcache/vcache int8 [H][T][HD] updated in place (rows past..past+M-1)"""
    M = x.shape[0]
    # dyadic-ish scales like the reference's op tests (tests/non_cuda/test_ops.cc): products stay exact in fp32
    a_qkv, b_qkv, qk_alpha, pv_alpha, a_out, a1, b1s, a2 = 0.00050354, 0.0213013, 0.0009, 0.0078125, 0.0006, 0.00045, 0.02, 0.0007
    h8 = ctx.layernorm_q(x, L.ln1w, L.ln1b, out=bufs["h8"][:M])
    q8 = ctx.w8a8_matmul(0, h8, L.wq, L.bq, a_qkv, b_qkv, out=bufs["q8"][:M])
    k8 = ctx.w8a8_matmul(0, h8, L.wk, L.bk, a_qkv, b_qkv, out=bufs["k8"][:M])
    v8 = ctx.w8a8_matmul(0, h8, L.wv, L.bv, a_qkv, b_qkv, out=bufs["v8"][:M])
    att = ctx.opt_int8_attention(q8, k8, v8, kcache if past else None, vcache if past else None, kcache, vcache, None, qk_alpha, pv_alpha, past, H, HD)
    o = ctx.w8a8_matmul(2, att, L.wo, L.bo, a_out, 1.0, out=bufs["o"][:M])
    r = ctx.add_f32(x, o, out=bufs["r"][:M])
    h8 = ctx.layernorm_q(r, L.ln2w, L.ln2b, out=bufs["h8"][:M])
    f1 = ctx.w8a8_matmul(0, h8, L.w1, L.b1, a1, b1s, q_min=0, out=bufs["f1"][:M])  # W8A8B8O8LinearReLU: clamp at 0
    f2 = ctx.w8a8_matmul(2, f1, L.w2, L.b2, a2, 1.0, out=bufs["o"][:M])
    return ctx.add_f32(r, f2, out=bufs["y"][:M])


def w8a8_layer(ctx, dev, stream, peaks, nlayers=3, reps=4):
    hbm = float(peaks.get("hbm_gbs", 6650.0))
    T = 2048
    layers = [Layer(dev, 100 + i) for i in range(nlayers)]  # 3 x 157 MB of int8 weights: more than 2x L2
    caches = [(torch.zeros((H, T, HD), dtype=torch.int8, device=dev), torch.zeros((H, T, HD), dtype=torch.int8, device=dev)) for _ in range(nlayers)]
    bufs = {"h8": torch.empty((T, E), dtype=torch.int8, device=dev), "q8": torch.empty((T, E), dtype=torch.int8, device=dev),
            "k8": torch.empty((T, E), dtype=torch.int8, device=dev), "v8": torch.empty((T, E), dtype=torch.int8, device=dev),
            "o": torch.empty((T, E), dtype=torch.float32, device=dev), "r": torch.empty((T, E), dtype=torch.float32, device=dev),
            "f1": torch.empty((T, F), dtype=torch.int8, device=dev), "y": torch.empty((T, E), dtype=torch.float32, device=dev)}
    out = {}
    for M, past in ((2048, 0), (1, 1024)):
        x = torch.randn((M, E), device=dev) * 3

        def run():
            y = x
            for L, (kc, vc) in zip(layers, caches):
                y = forward(ctx, L, y, kc, vc, past, bufs)
            return y

        run()
        torch.cuda.synchronize(dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(reps):
            run()
        e1.record(stream)
        torch.cuda.synchronize(dev)
        ms = e0.elapsed_time(e1) / (reps * nlayers)
        if M == 1:
            gbs = Layer.weight_bytes() / (ms * 1e-3) / 1e9
            out["decode_m1_ctx1024"] = {"ms_per_layer": ms, "weight_GB_per_s": gbs, "frac_of_measured_hbm": gbs / hbm,
                                        "tok_s_at_32_layers": 1e3 / (32 * ms)}
        else:
            tops = Layer.ops(M) / (ms * 1e-3) / 1e12
            out["prefill_m2048"] = {"ms_per_layer": ms, "linear_TOP_per_s": tops, "note": "int8 wgmma (s8 x s8) GEMMs + bit-exact int8 attention + serial-order LayerNormQ"}
    out["shapes"] = "Llama-2-7B widths in the OPT W8A8 layer structure (q/k/v/o 4096x4096, fc1 11008x4096 ReLU, fc2 4096x11008, 32 heads x 128), eager launches"
    return out


def main():
    from tinychatengine_b200.runtime import Context

    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    peaks = json.loads((ROOT / "MEASURED_PEAKS.json").read_text()) if (ROOT / "MEASURED_PEAKS.json").exists() else {}
    with torch.cuda.stream(stream):
        ctx = Context(0, stream)
        print(json.dumps(w8a8_layer(ctx, dev, stream, peaks)))
        ctx.close()


if __name__ == "__main__":
    main()
