"""Device-side plumbing on top of the C ABI: contexts, torch tensors as raw device pointers, synthetic weights.

torch supplies memory + streams; every computation goes through libtce_b200.so.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from .formats import GROUP, zeros_width


def _ptr(t):
    if t is None:
        return None
    if not t.is_contiguous():  # the C ABI takes dense row-major buffers; a strided view would be read as garbage
        raise _lib.TceError(f"non-contiguous tensor passed to libtce_b200 (shape {tuple(t.shape)}, strides {t.stride()})")
    return C.c_void_p(t.data_ptr())


class Context:
    """One tce_ctx per (device, stream)."""

    def __init__(self, device: int | None = None, stream: torch.cuda.Stream | None = None):
        if not torch.cuda.is_available():
            raise _lib.TceError("no CUDA device: tinychatengine_b200 has no CPU fallback")
        self.device = torch.cuda.current_device() if device is None else device
        self.L = _lib.lib()
        h = C.c_void_p()
        _lib.check(self.L.tce_ctx_create(self.device, C.byref(h)), "tce_ctx_create")
        self.h = h
        self.stream = None
        self.set_stream(stream if stream is not None else torch.cuda.current_stream(self.device))

    def set_stream(self, stream: torch.cuda.Stream):
        self.stream = stream
        _lib.check(self.L.tce_ctx_set_stream(self.h, C.c_void_p(stream.cuda_stream)), "tce_ctx_set_stream")

    def set_option(self, name: str, value: int):
        _lib.check(self.L.tce_ctx_set_option(self.h, name.encode(), int(value)), "tce_ctx_set_option")

    def synchronize(self):
        _lib.check(self.L.tce_ctx_synchronize(self.h), "tce_ctx_synchronize")

    @property
    def num_sms(self) -> int:
        return self.L.tce_ctx_num_sms(self.h)

    def close(self):
        if self.h:
            self.L.tce_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- ops (thin: argument marshalling only) ----
    def w4a16_gemv(self, x, w, zeros, scales, out=None, group: int = GROUP, gemm: bool = False):
        M, IC = x.shape
        OC = w.shape[0]
        if out is None:
            out = torch.empty((M, OC), dtype=torch.float16, device=x.device)
        fn = self.L.tce_w4a16_gemm if gemm else self.L.tce_w4a16_gemv
        _lib.check(fn(self.h, _ptr(x), _ptr(w), _ptr(zeros), _ptr(scales), _ptr(out), M, IC, OC, group), "tce_w4a16_gemv")
        return out

    def w8a8_matmul(self, variant: int, A, B, bias=None, alpha=1.0, beta=1.0, q_min=-128, q_max=127, batch=False, out=None):
        M, K = A.shape
        N = B.shape[-2]
        if out is None:
            out = torch.empty((M, N), dtype=torch.int8 if variant in (0, 1) else torch.float32, device=A.device)
        _lib.check(self.L.tce_w8a8_matmul(self.h, variant, int(batch), _ptr(A), _ptr(B), _ptr(bias), _ptr(out), M, N, K, alpha, beta, q_min, q_max),
                   "tce_w8a8_matmul")
        return out

    def naive_fp16_int4(self, A, B, scales, block: int = GROUP):
        M, IC = A.shape
        OC = scales.shape[1]
        out = torch.empty((M, OC), dtype=torch.float16, device=A.device)
        _lib.check(self.L.tce_naive_fp16_int4(self.h, _ptr(A), _ptr(B), _ptr(scales), _ptr(out), M, IC, OC, block), "tce_naive_fp16_int4")
        return out

    def f32_matmul_transposed(self, A, B):
        M, K = A.shape
        N = B.shape[0]
        out = torch.empty((M, N), dtype=torch.float32, device=A.device)
        _lib.check(self.L.tce_f32_matmul_transposed(self.h, _ptr(A), _ptr(B), _ptr(out), M, N, K), "tce_f32_matmul_transposed")
        return out

    def opt_int8_attention(self, q8, k8, v8, past_k, past_v, final_k, final_v, mask, qk_alpha, pv_alpha, past: int, H: int, hd: int):
        """final_k/final_v: int8 [H][>=past+sqlen][hd] tensors (may be the same storage as past_k/past_v -> in place)."""
        sqlen = q8.shape[0]
        out = torch.empty((sqlen, H * hd), dtype=torch.int8, device=q8.device)
        phs = past_k.stride(0) if past_k is not None else 0
        _lib.check(self.L.tce_opt_int8_attention(self.h, _ptr(q8), _ptr(k8), _ptr(v8), _ptr(past_k), _ptr(past_v), phs, _ptr(final_k), _ptr(final_v),
                                                 final_k.stride(0), _ptr(mask), qk_alpha, pv_alpha, sqlen, past, H, hd, _ptr(out)),
                   "tce_opt_int8_attention")
        return out

    def attn_decode(self, qkv, k_cache, v_cache, cos, sin, pos_dev, out, alpha, H, KVH, hd, max_ctx):
        _lib.check(self.L.tce_attn_decode(self.h, _ptr(qkv), _ptr(k_cache), _ptr(v_cache), _ptr(cos), _ptr(sin), _ptr(pos_dev), _ptr(out), alpha, H, KVH,
                                          hd, max_ctx), "tce_attn_decode")
        return out

    def attn_span(self, qkv, k_cache, v_cache, cos, sin, out, alpha, n, pos0, H, KVH, hd, max_ctx):
        _lib.check(self.L.tce_attn_span(self.h, _ptr(qkv), _ptr(k_cache), _ptr(v_cache), _ptr(cos), _ptr(sin), _ptr(out), alpha, n, pos0, H, KVH, hd,
                                        max_ctx), "tce_attn_span")
        return out

    def attn_prefill(self, qkv, k_cache, v_cache, cos, sin, out, alpha, n, pos0, H, KVH, hd, max_ctx):
        _lib.check(self.L.tce_attn_prefill(self.h, _ptr(qkv), _ptr(k_cache), _ptr(v_cache), _ptr(cos), _ptr(sin), _ptr(out), alpha, n, pos0, H, KVH, hd,
                                           max_ctx), "tce_attn_prefill")
        return out

    def rmsnorm_f16(self, x, gamma, eps, out=None):
        if out is None:
            out = torch.empty_like(x)
        _lib.check(self.L.tce_rmsnorm_f16(self.h, _ptr(x), _ptr(gamma), _ptr(out), x.shape[0], x.shape[1], eps), "tce_rmsnorm_f16")
        return out

    def layernorm_q(self, x, weight, bias, out=None):
        if out is None:
            out = torch.empty(x.shape, dtype=torch.int8, device=x.device)
        _lib.check(self.L.tce_layernorm_q(self.h, _ptr(x), _ptr(weight), _ptr(bias), _ptr(out), x.shape[0], x.shape[1]), "tce_layernorm_q")
        return out

    def add_f32(self, a, b, out=None):
        if out is None:
            out = torch.empty_like(a)
        _lib.check(self.L.tce_add_f32(self.h, _ptr(a), _ptr(b), _ptr(out), a.numel()), "tce_add_f32")
        return out

    def sample(self, logits, window=(), *, top_k=40, top_p=0.95, temp=0.8, repeat_penalty=1.1, frequency_penalty=0.0, presence_penalty=0.0,
               repeat_last_n=64, seed=0, draw_index=0, candidates=False):
        """One device sampling step on `logits` (float32 CUDA tensor, penalised in place); defaults are the reference's opt_params.
        Returns the token, or (token, ids, probs) with candidates=True."""
        import ctypes as C

        import numpy as np

        cfg = _lib.Sampling(int(top_k), float(top_p), float(temp), float(repeat_penalty), float(frequency_penalty), float(presence_penalty),
                            int(repeat_last_n), int(seed))
        win = np.ascontiguousarray(np.asarray(list(window), dtype=np.int32))
        tok, cnt = C.c_int(-1), C.c_int(0)
        kcap = max(1, min(1024, int(top_k) if top_k > 0 else logits.numel()))
        ids = np.zeros(kcap, dtype=np.int32)
        probs = np.zeros(kcap, dtype=np.float32)
        _lib.check(self.L.tce_sample(self.h, _ptr(logits), logits.numel(), win.ctypes.data_as(C.c_void_p) if win.size else None, int(win.size), C.byref(cfg),
                                     int(draw_index), C.byref(tok), ids.ctypes.data_as(C.c_void_p) if candidates else None,
                                     probs.ctypes.data_as(C.c_void_p) if candidates else None, C.byref(cnt) if candidates else None), "tce_sample")
        if candidates:
            return tok.value, ids[:cnt.value].copy(), probs[:cnt.value].copy()
        return tok.value

    def spec_accept(self, logits, drafts=(), window=(), *, top_k=40, top_p=0.95, temp=0.8, repeat_penalty=1.1, frequency_penalty=0.0,
                    presence_penalty=0.0, repeat_last_n=64, seed=0, draw_index=0, eos_id=-1, budget=None):
        """The acceptance rule of one speculative step (tce_spec_accept) on `logits` (float32 CUDA tensor [len(drafts) + 1, V], penalised in
        place).  Returns (ids, accepted, stop, q)."""
        import ctypes as C

        import numpy as np

        rows = len(drafts) + 1
        assert logits.dim() == 2 and logits.shape[0] == rows and logits.stride(1) == 1
        cfg = _lib.Sampling(int(top_k), float(top_p), float(temp), float(repeat_penalty), float(frequency_penalty), float(presence_penalty),
                            int(repeat_last_n), int(seed))
        dr = np.ascontiguousarray(np.asarray(list(drafts), dtype=np.int32))
        win = np.ascontiguousarray(np.asarray(list(window), dtype=np.int32))
        ids = np.zeros(rows, dtype=np.int32)
        q = np.zeros(rows, dtype=np.float32)
        n, acc, stop = C.c_int(0), C.c_int(0), C.c_int(0)
        ptr = lambda a: a.ctypes.data_as(C.c_void_p) if a.size else None
        _lib.check(self.L.tce_spec_accept(self.h, _ptr(logits), rows, logits.stride(0), logits.shape[1], ptr(dr), ptr(win), int(win.size), C.byref(cfg),
                                          int(draw_index), int(eos_id), int(rows if budget is None else budget), ptr(ids), C.byref(n), C.byref(acc),
                                          C.byref(stop), ptr(q)), "tce_spec_accept")
        return ids[:n.value].tolist(), acc.value, stop.value, q

    def argmax_f32(self, x, out=None):
        if out is None:
            out = torch.empty((1,), dtype=torch.int32, device=x.device)
        _lib.check(self.L.tce_argmax_f32(self.h, _ptr(x), x.numel(), _ptr(out)), "tce_argmax_f32")
        return out


def random_w4(oc: int, ic: int, device, seed: int, scale: float = 0.02, random_zeros: bool = False, group: int = GROUP):
    """Synthetic QM_CUDA tensors generated on the device: uniform nibbles, per-group fp16 scales such that the
    dequantised weights have std ~ `scale`, zero points 8 (or random)."""
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    zw = zeros_width(ic, group)
    w = torch.randint(-(2**31), 2**31 - 1, (oc, ic // 8), dtype=torch.int32, device=device, generator=g)
    ng = ic // group
    s = torch.zeros((oc, zw * 8), dtype=torch.float16, device=device)
    # uniform nibbles minus 8 have std ~4.6
    s[:, :ng] = ((0.5 + torch.rand((oc, ng), device=device, generator=g)) * (scale / 4.6)).to(torch.float16)
    if random_zeros:
        z = torch.randint(-(2**31), 2**31 - 1, (oc, zw), dtype=torch.int32, device=device, generator=g)
    else:
        z = torch.full((oc, zw), -0x77777778, dtype=torch.int32, device=device)  # 0x88888888
    return w, z, s
