"""Llama decode runner over the C ABI (tce_llama_*): synthetic-weight builder + step API.

Geometry table = reference llm/include/model.h:71-83.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import torch

from . import _lib
from .runtime import Context, random_w4


@dataclass
class LlamaGeometry:
    name: str
    num_layers: int
    num_heads: int
    num_kv_heads: int
    embed_dim: int
    hidden_dim: int
    vocab_size: int
    rms_eps: float = 1e-5
    rope_theta: float = 10000.0
    head_dim: int = 128


GEOMETRIES = {
    "llama3-8b": LlamaGeometry("llama3-8b", 32, 32, 8, 4096, 14336, 128256, 1e-5, 500000.0),
    "llama2-7b": LlamaGeometry("llama2-7b", 32, 32, 32, 4096, 11008, 32000, 1e-6, 10000.0),
    "llama2-13b": LlamaGeometry("llama2-13b", 40, 40, 40, 5120, 13824, 32000, 1e-6, 10000.0),
    # tiny shapes for tests (same structure, GQA 4:1 like Llama-3)
    "tiny-gqa": LlamaGeometry("tiny-gqa", 2, 8, 2, 1024, 2816, 2048, 1e-5, 500000.0),
    "tiny-mha": LlamaGeometry("tiny-mha", 2, 4, 4, 512, 1408, 1024, 1e-6, 10000.0),
}


def weight_bytes_per_token(g: LlamaGeometry) -> int:
    """Algorithmic HBM bytes one decode step must read from the packed weights (nibbles + fp16 scales + 4-bit
    zeros, unpadded), SURVEY.md 8(d): 3.899 GB for Llama-3-8B."""
    hd = g.head_dim
    mats = []
    for _ in range(g.num_layers):
        mats += [(g.num_heads * hd, g.embed_dim), (g.num_kv_heads * hd, g.embed_dim), (g.num_kv_heads * hd, g.embed_dim),
                 (g.embed_dim, g.num_heads * hd), (g.hidden_dim, g.embed_dim), (g.hidden_dim, g.embed_dim), (g.embed_dim, g.hidden_dim)]
    mats.append((g.vocab_size, g.embed_dim))
    total = 0
    for oc, ic in mats:
        total += oc * ic // 2 + oc * (ic // 128) * 2 + oc * (ic // 128) // 2
    return total


def kv_bytes_per_token(g: LlamaGeometry, ctx_len: int) -> int:
    """fp16 K+V read for `ctx_len` cached positions plus the one-row append, all layers."""
    per_pos = 2 * g.num_kv_heads * g.head_dim * 2 * g.num_layers
    return per_pos * ctx_len + per_pos


def make_random_weights(geom: LlamaGeometry, dev, seed: int = 1234, random_zeros: bool = False, embed_rows: int | None = None):
    """Synthetic AWQ-INT4 Llama weights (QM_CUDA layout) as a plain dict of torch tensors on `dev`.  `embed_rows`: rows of the
    embedding table when it differs from geom.vocab_size (a tensor-parallel rank holds a vocabulary SHARD of lm_head but looks up
    GLOBAL token ids, so its table has all the rows)."""
    g = geom
    hd = g.head_dim
    gen = torch.Generator(device=dev)
    gen.manual_seed(seed)
    W = {"layers": []}
    for l in range(g.num_layers):
        s = seed * 1000 + l * 16
        L = {"q": random_w4(g.num_heads * hd, g.embed_dim, dev, s + 1, 0.02, random_zeros),
             "k": random_w4(g.num_kv_heads * hd, g.embed_dim, dev, s + 2, 0.02, random_zeros),
             "v": random_w4(g.num_kv_heads * hd, g.embed_dim, dev, s + 3, 0.02, random_zeros),
             "o": random_w4(g.embed_dim, g.num_heads * hd, dev, s + 4, 0.02, random_zeros),
             "gate": random_w4(g.hidden_dim, g.embed_dim, dev, s + 5, 0.02, random_zeros),
             "up": random_w4(g.hidden_dim, g.embed_dim, dev, s + 6, 0.02, random_zeros),
             "down": random_w4(g.embed_dim, g.hidden_dim, dev, s + 7, 0.02, random_zeros),
             "input_norm": (1.0 + 0.02 * torch.randn(g.embed_dim, device=dev, generator=gen)).float(),
             "post_norm": (1.0 + 0.02 * torch.randn(g.embed_dim, device=dev, generator=gen)).float()}
        W["layers"].append(L)
    W["embed"] = (torch.randn((embed_rows or g.vocab_size, g.embed_dim), device=dev, generator=gen) * 0.5).to(torch.float16)
    W["final_norm"] = (1.0 + 0.02 * torch.randn(g.embed_dim, device=dev, generator=gen)).float()
    W["lm_head"] = random_w4(g.vocab_size, g.embed_dim, dev, seed * 1000 + 999983, 0.02, random_zeros)
    return W


def shard_w4_rows(t, rank: int, P: int):
    """Output-channel (row) shard of a QM_CUDA tensor triple: contiguous rows [rank*OC/P, (rank+1)*OC/P)."""
    w, z, s = t
    n = w.shape[0] // P
    return tuple(x[rank * n:(rank + 1) * n].contiguous() for x in (w, z, s))


def shard_w4_cols(t, ic: int, rank: int, P: int, group: int = 128):
    """Input-channel shard (row-parallel linear): columns [rank*IC/P, (rank+1)*IC/P) repacked as a QM_CUDA tensor of
    its own: the packed words are a contiguous slice per row, scales/zeros are re-padded to the shard's zeros_width."""
    from .formats import zeros_width

    w, z, s = t
    icl = ic // P
    assert icl % group == 0
    ngl = icl // group
    zwl = zeros_width(icl, group)
    wl = w[:, rank * icl // 8:(rank + 1) * icl // 8].contiguous()
    sl = torch.zeros((w.shape[0], zwl * 8), dtype=s.dtype, device=s.device)
    sl[:, :ngl] = s[:, rank * ngl:(rank + 1) * ngl]
    zi = z.to(torch.int64) & 0xFFFFFFFF
    nib = torch.stack([(zi >> (4 * i)) & 0xF for i in range(8)], dim=2).reshape(z.shape[0], -1)  # [OC, zw*8]
    nl = torch.full((z.shape[0], zwl * 8), 8, dtype=torch.int64, device=z.device)
    nl[:, :ngl] = nib[:, rank * ngl:(rank + 1) * ngl]
    packed = torch.zeros((z.shape[0], zwl), dtype=torch.int64, device=z.device)
    for i in range(8):
        packed |= nl[:, i::8] << (4 * i)
    packed = torch.where(packed >= 2 ** 31, packed - 2 ** 32, packed).to(torch.int32)
    return wl, packed.contiguous(), sl.contiguous()


def shard_weights(W, geom: LlamaGeometry, rank: int, P: int):
    """Megatron-style shard (SURVEY.md 8e): q/k/v/gate/up/lm_head by rows, o/down by input channels."""
    hd = geom.head_dim
    gl = LlamaGeometry(geom.name, geom.num_layers, geom.num_heads // P, geom.num_kv_heads // P, geom.embed_dim, geom.hidden_dim // P,
                       geom.vocab_size // P, geom.rms_eps, geom.rope_theta, hd)
    Wl = {"layers": [], "embed": W["embed"], "final_norm": W["final_norm"], "lm_head": shard_w4_rows(W["lm_head"], rank, P)}
    for L in W["layers"]:
        Wl["layers"].append({"q": shard_w4_rows(L["q"], rank, P), "k": shard_w4_rows(L["k"], rank, P), "v": shard_w4_rows(L["v"], rank, P),
                             "o": shard_w4_cols(L["o"], geom.num_heads * hd, rank, P), "gate": shard_w4_rows(L["gate"], rank, P),
                             "up": shard_w4_rows(L["up"], rank, P), "down": shard_w4_cols(L["down"], geom.hidden_dim, rank, P),
                             "input_norm": L["input_norm"], "post_norm": L["post_norm"]})
    return Wl, gl


class LlamaModel:
    """Llama weights (synthetic by default) + tce_llama handle.  Holds the torch tensors alive (the C side borrows
    pointers).  `geom` describes the LOCAL shard when tp_size > 1 (see shard_weights)."""

    def __init__(self, ctx: Context, geom: LlamaGeometry, max_ctx: int = 4096, seed: int = 1234, random_zeros: bool = False, weights=None,
                 tp_rank: int = 0, tp_size: int = 1):
        self.ctx, self.geom, self.max_ctx = ctx, geom, max_ctx
        self.tp_rank, self.tp_size = tp_rank, tp_size
        dev = torch.device("cuda", ctx.device)
        g = geom
        hd = g.head_dim
        W = weights if weights is not None else make_random_weights(geom, dev, seed, random_zeros, embed_rows=geom.vocab_size * max(1, tp_size))
        self.W = W
        self.tensors = []

        def w4(t, oc, ic):
            assert t[0].shape == (oc, ic // 8), (t[0].shape, oc, ic)
            self.tensors.append(t)
            return _lib.W4Tensor(t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), oc, ic)

        def norm(t):
            self.tensors.append(t)
            return t.data_ptr()

        self.layers = (_lib.LlamaLayer * g.num_layers)()
        for l in range(g.num_layers):
            L, T = self.layers[l], W["layers"][l]
            L.q = w4(T["q"], g.num_heads * hd, g.embed_dim)
            L.k = w4(T["k"], g.num_kv_heads * hd, g.embed_dim)
            L.v = w4(T["v"], g.num_kv_heads * hd, g.embed_dim)
            L.o = w4(T["o"], g.embed_dim, g.num_heads * hd)
            L.gate = w4(T["gate"], g.hidden_dim, g.embed_dim)
            L.up = w4(T["up"], g.hidden_dim, g.embed_dim)
            L.down = w4(T["down"], g.embed_dim, g.hidden_dim)
            L.input_norm = norm(T["input_norm"])
            L.post_norm = norm(T["post_norm"])
        self.embed = W["embed"]
        self.final_norm = W["final_norm"]
        self.weights = _lib.LlamaWeights()
        self.weights.embed_f16 = self.embed.data_ptr()
        self.weights.layers = C.cast(self.layers, C.POINTER(_lib.LlamaLayer))
        self.weights.final_norm = self.final_norm.data_ptr()
        self.weights.lm_head = w4(W["lm_head"], g.vocab_size, g.embed_dim)
        self.weights.rope_cos = None
        self.weights.rope_sin = None
        self.cfg = _lib.LlamaConfig(g.num_layers, g.num_heads, g.num_kv_heads, hd, g.embed_dim, g.hidden_dim, g.vocab_size, max_ctx,
                                    g.rms_eps, g.rope_theta, 0.0, tp_rank, tp_size)
        h = C.c_void_p()
        _lib.check(ctx.L.tce_llama_create(ctx.h, C.byref(self.cfg), C.byref(self.weights), C.byref(h)), "tce_llama_create")
        self.h = h
        self.kernels_per_step = ctx.L.tce_llama_kernels_per_step(h)
        torch.cuda.synchronize(dev)

    @classmethod
    def load_dir(cls, ctx: Context, path, geom: LlamaGeometry, max_ctx: int = 4096):
        """Model built by the C++ loader from a parameter tree in the reference's on-disk layout (tce_llama_load_dir); the library owns the
        device copies.  `geom` plays the role of the reference's model_config."""
        self = cls.__new__(cls)
        self.ctx, self.geom, self.max_ctx = ctx, geom, max_ctx
        self.tp_rank, self.tp_size = 0, 1
        self.W, self.tensors = None, []
        g = geom
        self.cfg = _lib.LlamaConfig(g.num_layers, g.num_heads, g.num_kv_heads, g.head_dim, g.embed_dim, g.hidden_dim, g.vocab_size, max_ctx,
                                    g.rms_eps, g.rope_theta, 0.0, 0, 1)
        h = C.c_void_p()
        _lib.check(ctx.L.tce_llama_load_dir(ctx.h, str(path).encode(), C.byref(self.cfg), C.byref(h)), "tce_llama_load_dir")
        self.h = h
        self.kernels_per_step = ctx.L.tce_llama_kernels_per_step(h)
        return self

    def save_dir(self, path, rotary: bool = True):
        """Write this model's (synthetic) weights as a parameter tree in the reference's QM_CUDA on-disk layout (tests, examples):
        the inverse of load_dir.  q|k|v are written merged under self_attn/qkv_proj, as llm/tools/llama_qkv_merger.py leaves them."""
        from pathlib import Path

        import numpy as np

        from . import formats

        root = Path(path)
        W = self.W

        def f32(t, p):
            p.parent.mkdir(parents=True, exist_ok=True)
            t.detach().float().cpu().numpy().astype(np.float32).tofile(p)

        def w4(t, p):
            formats.save_qm_cuda_dir(p, t[0].cpu().numpy().view(np.uint32), t[1].cpu().numpy().view(np.uint32), t[2].cpu().numpy())

        f32(W["embed"], root / "decoder" / "embed_tokens" / "weight.bin")
        f32(W["final_norm"], root / "decoder" / "norm" / "weight.bin")
        for l, T in enumerate(W["layers"]):
            lp = root / "decoder" / f"layer{l}"
            f32(T["input_norm"], lp / "input_layernorm" / "weight.bin")
            f32(T["post_norm"], lp / "post_attention_layernorm" / "weight.bin")
            merged = tuple(torch.cat([T[n][i] for n in ("q", "k", "v")], dim=0) for i in range(3))
            w4(merged, lp / "self_attn" / "qkv_proj")
            w4(T["o"], lp / "self_attn" / "o_proj")
            for n in ("gate", "up", "down"):
                w4(T[n], lp / f"{n}_proj")
        w4(W["lm_head"], root / "lm_head")
        if rotary:
            # rotary_emb tables and the qk scale as the reference trees carry them (fp16; llm/tools/rotary_emb_exporter.py, read by
            # RotaryPosEmb_cuda's constructor and Int4llamaAttention.cu:82): a tree with tables overrides rope_theta on load
            g = self.geom
            hd = g.head_dim
            inv = 1.0 / (g.rope_theta ** (np.arange(0, hd, 2, dtype=np.float64) / hd))
            ang = np.arange(self.max_ctx)[:, None] * inv[None, :]
            emb = np.concatenate([ang, ang], axis=1)
            for l in range(g.num_layers):
                sa = root / "decoder" / f"layer{l}" / "self_attn"
                (sa / "rotary_emb").mkdir(parents=True, exist_ok=True)
                (sa / "qk_bmm").mkdir(parents=True, exist_ok=True)
                np.cos(emb).astype(np.float16).tofile(sa / "rotary_emb" / "cos_cached_half.bin")
                np.sin(emb).astype(np.float16).tofile(sa / "rotary_emb" / "sin_cached_half.bin")
                np.array([1.0 / np.sqrt(hd)], dtype=np.float16).tofile(sa / "qk_bmm" / "alpha_half.bin")

    def tp_connect(self, group=None):
        """Exchange the IPC handles of the peer-visible buffers over torch.distributed and map the peers."""
        import torch.distributed as dist

        mine = (C.c_ubyte * 64)()
        _lib.check(self.ctx.L.tce_llama_tp_handle(self.h, C.cast(mine, C.c_void_p)), "tce_llama_tp_handle")
        t = torch.tensor(list(mine), dtype=torch.uint8)
        backend = dist.get_backend(group)
        if backend == "nccl":
            t = t.cuda(self.ctx.device)
        out = [torch.empty_like(t) for _ in range(self.tp_size)]
        dist.all_gather(out, t, group=group)
        blob = b"".join(bytes(o.cpu().tolist()) for o in out)
        buf = (C.c_ubyte * len(blob)).from_buffer_copy(blob)
        _lib.check(self.ctx.L.tce_llama_tp_connect(self.h, C.cast(buf, C.c_void_p)), "tce_llama_tp_connect")
        dist.barrier(group=group)

    def layer_tensors(self, l: int):
        """(q, k, v, o, gate, up, down) each as (w, zeros, scales) torch tensors, plus the two norm gammas."""
        per = 9
        base = l * per
        t = self.tensors[base: base + per]
        return {"q": t[0], "k": t[1], "v": t[2], "o": t[3], "gate": t[4], "up": t[5], "down": t[6], "input_norm": t[7], "post_norm": t[8]}

    def decode(self, tokpos_dev: torch.Tensor):
        _lib.check(self.ctx.L.tce_llama_decode(self.h, C.c_void_p(tokpos_dev.data_ptr())), "tce_llama_decode")

    def decode_host(self, token: int, pos: int, logits_host=None):
        nxt = C.c_int(-1)
        p = None if logits_host is None else C.c_void_p(logits_host.data_ptr())
        _lib.check(self.ctx.L.tce_llama_decode_host(self.h, int(token), int(pos), p, C.byref(nxt)), "tce_llama_decode_host")
        return nxt.value

    def generate(self, first_token: int, pos0: int, n_predict: int, *, history=(), eos_id: int = -1, top_k=40, top_p=0.95, temp=0.8, repeat_penalty=1.1,
                 frequency_penalty=0.0, presence_penalty=0.0, repeat_last_n=64, seed=0, n_keep=None):
        """Device generate loop (decode + sample per token, only the ids come back); defaults are the reference's opt_params.  n_keep: when
        the context fills before n_predict ids, shift slot 0 with kv_shift(0, max_ctx, n_keep) and carry on (the reference's opt_params.n_keep);
        None stops at max_ctx."""
        import numpy as np

        cfg = _lib.Sampling(int(top_k), float(top_p), float(temp), float(repeat_penalty), float(frequency_penalty), float(presence_penalty),
                            int(repeat_last_n), int(seed))

        def run(first, p0, budget, hist_ids):
            hist = np.ascontiguousarray(np.asarray(list(hist_ids), dtype=np.int32))
            out = np.zeros(max(1, budget), dtype=np.int32)
            n = C.c_int(0)
            _lib.check(self.ctx.L.tce_llama_generate(self.h, int(first), int(p0), int(budget), C.byref(cfg),
                                                     hist.ctypes.data_as(C.c_void_p) if hist.size else None, int(hist.size), int(eos_id),
                                                     out.ctypes.data_as(C.c_void_p), C.byref(n)), "tce_llama_generate")
            return out[:n.value].tolist()

        self._check_n_keep(n_keep)
        ids = run(first_token, pos0, n_predict, history)
        p0, seg = pos0, len(ids)
        while self._context_full(n_keep, p0, seg, n_predict - (len(ids) - seg), ids, eos_id):
            p0 = self.kv_shift(0, self.max_ctx, n_keep)
            more = run(ids[-1], p0, n_predict - len(ids), (list(history) + ids)[-self.max_ctx:])
            ids += more
            seg = len(more)
        return ids

    def _check_n_keep(self, n_keep):
        if n_keep is not None and not (0 <= n_keep and (self.max_ctx - n_keep) // 2 >= 1):
            raise ValueError(f"n_keep = {n_keep}: the context shift needs 0 <= n_keep and (max_ctx - n_keep) // 2 >= 1 (max_ctx = {self.max_ctx})")

    def _context_full(self, n_keep, pos0, n_seg, budget, ids, eos_id) -> bool:
        """A generate call that returned n_seg ids from pos0 with this budget stopped only because the context filled (and n_keep asks to
        shift and continue)."""
        return n_keep is not None and n_seg > 0 and pos0 + n_seg == self.max_ctx and n_seg < budget and ids[-1] != eos_id

    def kv_copy(self, src_slot: int, src_pos: int, n: int, dst_slots, dst_pos=None):
        """Copy KV-cache rows src_pos .. src_pos + n - 1 of src_slot to rows dst_pos[i] .. of dst_slots[i] (up to MAX_BATCH destinations;
        default: the same positions), every layer, K and V; K rows are re-rotated by the position change (tce_llama_kv_copy).  Asynchronous,
        ordered with the other calls on the model's stream."""
        dst_slots = [int(s) for s in dst_slots]
        dst_pos = [int(src_pos)] * len(dst_slots) if dst_pos is None else [int(p) for p in dst_pos]
        if len(dst_pos) != len(dst_slots):
            raise ValueError("kv_copy: one destination position per destination slot")
        arr = lambda v: (C.c_int * max(1, len(v)))(*v)
        _lib.check(self.ctx.L.tce_llama_kv_copy(self.h, int(src_slot), int(src_pos), int(n), len(dst_slots), arr(dst_slots), arr(dst_pos)),
                   "tce_llama_kv_copy")

    def fork(self, src_slot: int, n_rows: int, dst_slots):
        """Rows 0 .. n_rows - 1 of src_slot (a prompt pass's cache) into each of dst_slots at the same positions."""
        self.kv_copy(src_slot, 0, n_rows, dst_slots)

    def kv_shift(self, slot: int, n_past: int, n_keep: int, n_discard=None) -> int:
        """Context shift of a slot holding n_past rows: keep [0, n_keep), drop the next n_discard (default (n_past - n_keep) // 2, the llama.cpp
        rule) and move [n_keep + n_discard, n_past) down to n_keep, K re-rotated.  Returns the new n_past."""
        if n_discard is None:
            n_discard = (n_past - n_keep) // 2
        if n_discard < 1 or n_keep < 0 or n_keep + n_discard > n_past:
            raise ValueError(f"kv_shift: n_past = {n_past}, n_keep = {n_keep}, n_discard = {n_discard}: needs n_discard >= 1, n_keep >= 0 and "
                             "n_keep + n_discard <= n_past")
        self.kv_copy(slot, n_keep + n_discard, n_past - n_keep - n_discard, [slot], [n_keep])
        return n_past - n_discard

    def prefill(self, tokens, pos0: int = 0, logits_host=None, slot: int = 0) -> int:
        """Prompt processing: all `tokens` (host ints) at positions pos0.. in one pass into KV-cache slot `slot`; returns the greedy next
        token."""
        arr = (C.c_int * len(tokens))(*[int(t) for t in tokens])
        nxt = C.c_int(-1)
        p = None if logits_host is None else C.c_void_p(logits_host.data_ptr())
        if slot == 0:
            _lib.check(self.ctx.L.tce_llama_prefill(self.h, arr, len(tokens), int(pos0), p, C.byref(nxt)), "tce_llama_prefill")
        else:
            _lib.check(self.ctx.L.tce_llama_prefill_slot(self.h, int(slot), arr, len(tokens), int(pos0), p, C.byref(nxt)), "tce_llama_prefill_slot")
        return nxt.value

    MAX_BATCH = 8  # TCE_LLAMA_MAX_BATCH

    def reserve_slots(self, n_slots: int):
        """Grow the number of KV-cache slots to `n_slots` (slot 0 is the single-sequence cache; never shrinks)."""
        _lib.check(self.ctx.L.tce_llama_reserve_slots(self.h, int(n_slots)), "tce_llama_reserve_slots")

    def decode_batch(self, req_dev: torch.Tensor):
        """One batched step from a device int32 [batch, 3] tensor of {token, position, slot}; logits land in batch_logits()."""
        assert req_dev.dtype == torch.int32 and req_dev.is_contiguous() and req_dev.dim() == 2 and req_dev.shape[1] == 3
        _lib.check(self.ctx.L.tce_llama_decode_batch(self.h, int(req_dev.shape[0]), C.c_void_p(req_dev.data_ptr())), "tce_llama_decode_batch")

    def decode_batch_host(self, tokens, positions, slots, logits_host=None):
        """One batched step from host lists; fills logits_host (float32 [batch, vocab], may be None) and returns the greedy tokens."""
        n = len(tokens)
        arr = lambda v: (C.c_int * max(1, n))(*[int(x) for x in v])
        nxt = (C.c_int * max(1, n))()
        p = None if logits_host is None else C.c_void_p(logits_host.data_ptr())
        _lib.check(self.ctx.L.tce_llama_decode_batch_host(self.h, n, arr(tokens), arr(positions), arr(slots), p, nxt), "tce_llama_decode_batch_host")
        return list(nxt[:n])

    def decode_span(self, tokens, pos0: int, slot: int = 0, logits_host=None) -> list[int]:
        """Span step: up to MAX_BATCH consecutive tokens (host ints) at positions pos0.. of one slot in one pass over the weights; fills
        logits_host (float32 [len(tokens), vocab], may be None; row i = the logits after tokens[i]) and returns the greedy ids of every row."""
        n = len(tokens)
        arr = (C.c_int * max(1, n))(*[int(t) for t in tokens])
        nxt = (C.c_int * max(1, n))()
        p = None if logits_host is None else C.c_void_p(logits_host.data_ptr())
        _lib.check(self.ctx.L.tce_llama_decode_span_host(self.h, int(slot), int(pos0), n, arr, p, nxt), "tce_llama_decode_span_host")
        return list(nxt[:n])

    def generate_lookup(self, first_token: int, pos0: int, n_predict: int, *, history=(), corpus=(), max_draft=7, ngram=(1, 3), eos_id: int = -1,
                        repeat_penalty=1.1, frequency_penalty=0.0, presence_penalty=0.0, repeat_last_n=64, temp=0.0, top_k=40, top_p=0.95, seed=0):
        """Generation on slot 0 with prompt-lookup drafts verified by the span step, in fewer passes over the weights when the continuation
        repeats corpus / history / earlier output.  temp <= 0 (tce_llama_generate_lookup): the ids of generate(temp=0) with the same penalties.
        temp > 0 (tce_llama_sample_lookup): drafts are accepted by speculative sampling, so the ids have the distribution of
        generate(temp=temp, ...) with the same fields, and at max_draft = 0 they are its ids for the same seed.
        Returns (ids, {"steps", "drafted", "accepted"})."""
        import numpy as np

        if temp > 0:
            cfg = _lib.Sampling(int(top_k), float(top_p), float(temp), float(repeat_penalty), float(frequency_penalty), float(presence_penalty),
                                int(repeat_last_n), int(seed))
            fn, name = self.ctx.L.tce_llama_sample_lookup, "tce_llama_sample_lookup"
        else:
            cfg = _lib.Sampling(40, 0.95, 0.0, float(repeat_penalty), float(frequency_penalty), float(presence_penalty), int(repeat_last_n), 0)
            fn, name = self.ctx.L.tce_llama_generate_lookup, "tce_llama_generate_lookup"
        lk = _lib.Lookup(int(max_draft), int(ngram[0]), int(ngram[1]))
        hist = np.ascontiguousarray(np.asarray(list(history), dtype=np.int32))
        corp = np.ascontiguousarray(np.asarray(list(corpus), dtype=np.int32))
        out = np.zeros(max(1, int(n_predict)), dtype=np.int32)
        n = C.c_int(0)
        st = _lib.LookupStats()
        ptr = lambda a: a.ctypes.data_as(C.c_void_p) if a.size else None
        _lib.check(fn(self.h, int(first_token), int(pos0), int(n_predict), C.byref(cfg), ptr(hist), int(hist.size), ptr(corp), int(corp.size), C.byref(lk),
                      int(eos_id), out.ctypes.data_as(C.c_void_p), C.byref(n), C.byref(st)), name)
        return out[:n.value].tolist(), {"steps": st.steps, "drafted": st.drafted, "accepted": st.accepted}

    def prefill_batch(self, prompts, slots, pos0s=None, logits_host=None) -> list[int]:
        """Prompt processing of up to MAX_BATCH prompts (lists of host ints) in one pass over the weights, prompt s into KV-cache slot
        slots[s] at positions pos0s[s].. (default 0); fills logits_host (float32 [n_prompts, vocab], may be None) with the logits of each
        prompt's last position and returns the greedy next tokens."""
        n = len(prompts)
        pos0s = [0] * n if pos0s is None else list(pos0s)
        flat = [int(t) for p in prompts for t in p]
        arr = lambda v: (C.c_int * max(1, len(v)))(*[int(x) for x in v])
        nxt = (C.c_int * max(1, n))()
        p = None if logits_host is None else C.c_void_p(logits_host.data_ptr())
        _lib.check(self.ctx.L.tce_llama_prefill_batch(self.h, n, arr(flat), arr([len(q) for q in prompts]), arr(pos0s), arr(slots), p, nxt),
                   "tce_llama_prefill_batch")
        return list(nxt[:n])

    def score_batch(self, prompts, slots, pos0s=None, targets=None, logits=None):
        """Teacher-forced scoring of up to MAX_BATCH prompts in one prompt pass (the KV rows prefill_batch would write are written too).
        targets: per prompt, the token whose log-probability each position reports (-1 for none); default: the next token of the prompt,
        -1 at its last position.  logits: optional CUDA float32 tensor [n, vocab] (n = all positions of all prompts) that receives every
        position's logits.  Returns, per prompt, (logprobs float32, greedy ids int32, greedy logprobs float32) numpy arrays; logprobs are
        NaN where the target is -1."""
        import numpy as np

        n_seqs = len(prompts)
        pos0s = [0] * n_seqs if pos0s is None else list(pos0s)
        lengths = [len(q) for q in prompts]
        n = sum(lengths)
        flat = np.ascontiguousarray(np.asarray([int(t) for q in prompts for t in q] or [0], dtype=np.int32))
        arr = lambda v: (C.c_int * max(1, len(v)))(*[int(x) for x in v])
        tg = None
        if targets is not None:
            if [len(t) for t in targets] != lengths:
                raise ValueError("score_batch: targets must have one entry per prompt position")
            tg = np.ascontiguousarray(np.asarray([int(t) for q in targets for t in q] or [0], dtype=np.int32))
        lp = np.empty(max(1, n), dtype=np.float32)
        gr = np.empty(max(1, n), dtype=np.int32)
        glp = np.empty(max(1, n), dtype=np.float32)
        lg = None
        if logits is not None:
            V = self.geom.vocab_size
            if not (logits.is_cuda and logits.dtype == torch.float32 and logits.is_contiguous() and tuple(logits.shape) == (n, V)):
                raise ValueError(f"score_batch: logits must be a contiguous CUDA float32 tensor of shape ({n}, {V})")
            lg = C.c_void_p(logits.data_ptr())
        ptr = lambda a: a.ctypes.data_as(C.c_void_p)
        _lib.check(self.ctx.L.tce_llama_score_batch(self.h, n_seqs, ptr(flat), arr(lengths), arr(pos0s), arr(slots),
                                                    None if tg is None else ptr(tg), ptr(lp), ptr(gr), ptr(glp), lg), "tce_llama_score_batch")
        out, r = [], 0
        for m in lengths:
            out.append((lp[r:r + m].copy(), gr[r:r + m].copy(), glp[r:r + m].copy()))
            r += m
        return out

    def generate_batch(self, requests, n_keep=None) -> list[list[int]]:
        """Device generate loop of up to MAX_BATCH sequences (one batched step + one sampler launch per token, only the ids come back).
        Each request is a dict with first_token, pos0, slot, n_predict and optional history, eos_id and the sampling fields of generate(),
        with the same defaults (the reference's opt_params).  n_keep: a sequence that stops only because its slot filled is shifted with
        kv_shift(slot, max_ctx, n_keep) and continues in the next call, with the rest of its budget; None stops it at max_ctx."""
        self._check_n_keep(n_keep)
        outs = self._generate_batch(requests)
        if n_keep is None:
            return outs
        ids = [list(o) for o in outs]
        active = list(enumerate(requests))
        while True:
            cont = []
            for (i, r), seg in zip(active, outs):
                if self._context_full(n_keep, r["pos0"], len(seg), r["n_predict"], ids[i], r.get("eos_id", -1)):
                    p0 = self.kv_shift(r["slot"], self.max_ctx, n_keep)
                    hist = (list(requests[i].get("history", ())) + ids[i])[-self.max_ctx:]
                    cont.append((i, dict(r, first_token=ids[i][-1], pos0=p0, n_predict=r["n_predict"] - len(seg), history=hist)))
            if not cont:
                return ids
            active = cont
            outs = self._generate_batch([r for _, r in active])
            for (i, _), seg in zip(active, outs):
                ids[i] += seg

    def _generate_batch(self, requests) -> list[list[int]]:
        defaults = dict(history=(), eos_id=-1, top_k=40, top_p=0.95, temp=0.8, repeat_penalty=1.1, frequency_penalty=0.0, presence_penalty=0.0,
                        repeat_last_n=64, seed=0)
        n = len(requests)
        reqs = (_lib.GenRequest * max(1, n))()
        keep = []
        for i, r in enumerate(requests):
            unknown = set(r) - set(defaults) - {"first_token", "pos0", "slot", "n_predict"}
            if unknown:
                raise TypeError(f"generate_batch: unknown request fields {sorted(unknown)}")
            q = {**defaults, **r}
            hist = (C.c_int * max(1, len(q["history"])))(*[int(t) for t in q["history"]])
            keep.append(hist)
            reqs[i] = _lib.GenRequest(int(q["first_token"]), int(q["pos0"]), int(q["slot"]), int(q["n_predict"]), int(q["eos_id"]),
                                      C.cast(hist, C.POINTER(C.c_int)) if len(q["history"]) else None, len(q["history"]),
                                      _lib.Sampling(int(q["top_k"]), float(q["top_p"]), float(q["temp"]), float(q["repeat_penalty"]),
                                                    float(q["frequency_penalty"]), float(q["presence_penalty"]), int(q["repeat_last_n"]), int(q["seed"])))
        stride = max([1] + [max(0, int(r["n_predict"])) for r in requests])
        out = (C.c_int * (max(1, n) * stride))()
        n_out = (C.c_int * max(1, n))()
        _lib.check(self.ctx.L.tce_llama_generate_batch(self.h, n, reqs, out, stride, n_out), "tce_llama_generate_batch")
        return [list(out[i * stride:i * stride + n_out[i]]) for i in range(n)]

    def batch_logits(self) -> torch.Tensor:
        """View of the device logits of the batched step (float32 [MAX_BATCH, vocab])."""
        ptr = self.ctx.L.tce_llama_batch_logits(self.h)
        if not ptr:
            raise _lib.TceError("tce_llama_batch_logits: no batched-step buffers (tensor-parallel model?)")
        return _tensor_from_ptr(ptr, (self.MAX_BATCH, self.geom.vocab_size), torch.float32, self.ctx.device)

    def logits(self) -> torch.Tensor:
        """View of the device logits buffer (float32 [vocab])."""
        ptr = self.ctx.L.tce_llama_logits(self.h)
        return _tensor_from_ptr(ptr, (self.geom.vocab_size,), torch.float32, self.ctx.device)

    def kv_cache(self, layer: int, which: int, slot: int = 0) -> torch.Tensor:
        ptr = self.ctx.L.tce_llama_kv_cache(self.h, layer, which) if slot == 0 else self.ctx.L.tce_llama_kv_cache_slot(self.h, slot, layer, which)
        if slot != 0 and not ptr:
            raise _lib.TceError(f"no KV cache for slot {slot}, layer {layer}, which {which}")
        return _tensor_from_ptr(ptr, (self.geom.num_kv_heads, self.max_ctx, self.geom.head_dim), torch.float16, self.ctx.device)

    def debug_buffer(self, which: int) -> torch.Tensor:
        """0..3: the batched step's residual (float32 [MAX_BATCH, E]), q|k|v, attention output and SiLU*up (float16 [MAX_BATCH, ...]),
        row b = request b of the last batched or span step; 5: the persistent kernel's hand-off words as int32 [n, 2] {payload, tag} (cut
        into its vectors by handoff_views)."""
        g = self.geom
        B = self.MAX_BATCH
        if which == 5:
            shape, dt = (sum(self._handoff_words().values()), 2), torch.int32
        else:
            shape, dt = {0: ((B, g.embed_dim), torch.float32), 1: ((B, (g.num_heads + 2 * g.num_kv_heads) * g.head_dim), torch.float16),
                         2: ((B, g.num_heads * g.head_dim), torch.float16), 3: ((B, g.hidden_dim), torch.float16)}[which]
        ptr = self.ctx.L.tce_llama_debug_buffer(self.h, which)
        if not ptr:
            raise _lib.TceError(f"debug buffer {which}: " + ("this model has no persistent kernel" if which == 5 else
                                                              "the kernel-per-op step has not run on this model"))
        return _tensor_from_ptr(ptr, shape, dt, self.ctx.device)

    def attn_nsplit_max(self) -> int:
        """Split records per head of the persistent kernel's attention (pk::attn_nsplit_max): #CTAs / KVH, at most one per 64-row chunk."""
        return min(max(1, self.ctx.num_sms // self.geom.num_kv_heads), -(-self.max_ctx // 64))

    def _handoff_words(self) -> dict:
        """Words of each hand-off vector, in the order LlamaDecoder::build_persistent lays them out (tensor parallel: the o_proj /
        down_proj words live in the peer-visible buffer instead)."""
        g = self.geom
        n = {"qkv": (g.num_heads + 2 * g.num_kv_heads) * 64, "attn": g.num_heads * 64, "act": g.hidden_dim // 2,
             "part": g.num_heads * self.attn_nsplit_max() * 130}
        if self.tp_size == 1:
            n.update(delta0=g.embed_dim, delta1=g.embed_dim)
        return n

    def handoff_views(self) -> dict:
        """The persistent kernel's hand-off words after a step (they hold the last layer's vectors): name -> (payload, tag).  qkv, attn,
        act: fp16 [2 * words] (two halfs per word); part: fp32 [H, nsplit_max, 130] (per split: output[128], max, sum); delta0 / delta1:
        the o_proj / down_proj outputs, fp32 [E].  tag: int64 per word (same shape as the words: [H, nsplit_max, 130] for part)."""
        words = self.debug_buffer(5)
        out, o = {}, 0
        for name, n in self._handoff_words().items():
            w = words[o:o + n]
            o += n
            pay = w[:, 0].contiguous()
            tag = w[:, 1].to(torch.int64) & 0xFFFFFFFF
            if name in ("qkv", "attn", "act"):
                out[name] = (pay.view(torch.float16), tag)
            elif name == "part":
                shape = (self.geom.num_heads, self.attn_nsplit_max(), 130)
                out[name] = (pay.view(torch.float32).reshape(shape), tag.reshape(shape))
            else:
                out[name] = (pay.view(torch.float32), tag)
        return out

    def close(self):
        if self.h:
            self.ctx.L.tce_llama_destroy(self.h)
            self.h = None


class _CudaArrayHolder:
    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (ptr, False), "version": 3}


def _tensor_from_ptr(ptr: int, shape, dtype, device: int) -> torch.Tensor:
    typestr = {torch.float32: "<f4", torch.float16: "<f2", torch.int32: "<i4", torch.int8: "|i1"}[dtype]
    return torch.as_tensor(_CudaArrayHolder(ptr, tuple(shape), typestr), device=torch.device("cuda", device))
