"""Helpers for the -m gpu parity tests: everything goes through the C ABI of libtgis_engine.so."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from vllm_tgis_adapter_b200.engine import _lib

KV_BLOCK = 32
HEAD_DIM = 128

SAMPLE_ROW_DTYPE = np.dtype([
    ("flags", "<i4"), ("n_topn", "<i4"), ("temperature", "<f4"), ("top_k", "<i4"), ("top_p", "<f4"),
    ("typical_p", "<f4"), ("rep_penalty", "<f4"), ("len_decay_factor", "<f4"), ("eos_id", "<i4"), ("n_out", "<i4"),
    ("min_tokens", "<i4"), ("seq_slot", "<i4"), ("seed_lo", "<u4"), ("seed_hi", "<u4"), ("step", "<u4"),
    ("logits_row", "<i4"),
])
SAMPLE_OUT_DTYPE = np.dtype([
    ("token", "<i4"), ("logprob", "<f4"), ("rank", "<i4"), ("n_topn", "<i4"), ("topn_ids", "<i4", (12,)),
    ("topn_lps", "<f4", (12,)),
])
SAMPLE_GREEDY, SAMPLE_LOGPROBS, SAMPLE_TYPICAL, SAMPLE_LENPEN, SAMPLE_SEEDED = 1, 2, 4, 8, 16
SAMPLE_MASKED = 64


def lib():
    return _lib.load_library()


def kerr() -> str:
    return (lib().tgis_k_last_error() or b"").decode()


def ptr(t: torch.Tensor) -> C.c_void_p:
    return C.c_void_p(t.data_ptr())


def i32p(a: np.ndarray):
    return a.ctypes.data_as(C.POINTER(C.c_int32))


def gemm(x: torch.Tensor, w: torch.Tensor, impl: int = 0, iters: int = 1, out_f32: bool = False, swiglu: bool = False
         ) -> tuple[torch.Tensor, float]:
    T, K = x.shape
    N = w.shape[0]
    rows = max(T, 256)
    xp = torch.zeros(rows, K, dtype=torch.bfloat16, device="cuda")
    xp[:T] = x
    mode = 2 if swiglu else (1 if out_f32 else 0)
    y = torch.empty(T, N // 2 if swiglu else N, dtype=torch.float32 if out_f32 else torch.bfloat16, device="cuda")
    ms = C.c_float(0)
    rc = lib().tgis_k_gemm(ptr(xp), ptr(w), ptr(y), T, N, K, rows, impl, iters, C.byref(ms), mode)
    assert rc == 0, kerr()
    return y, ms.value


def bf16_ulp_diff(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """|a-b| measured in bf16 ulps of max(|a|,|b|)."""
    a32, b32 = a.float(), b.float()
    mag = torch.maximum(a32.abs(), b32.abs()).clamp_min(1e-30)
    ulp = torch.exp2(torch.floor(torch.log2(mag)) - 7)
    return (a32 - b32).abs() / ulp


def attention_reference_f64(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, first_pos: int, scale: float
                            ) -> torch.Tensor:
    """float64 softmax(q k^T * scale) v of one sequence, causal by absolute position (query i sits at first_pos + i).
    q [q_len, n_q, 128], k / v [kv_len, n_kv, 128] (bf16, any device) -> float64 [q_len, n_q, 128] on q's device."""
    q_len, n_q, _ = q.shape
    kv_len, n_kv, _ = k.shape
    G = n_q // n_kv
    k, v = k.to(q.device), v.to(q.device)
    future = torch.arange(kv_len, device=q.device)[None, :] > (first_pos + torch.arange(q_len, device=q.device))[:, None]
    out = torch.empty(q_len, n_q, HEAD_DIM, dtype=torch.float64, device=q.device)
    for h in range(n_kv):  # one kv head at a time bounds the [G, q_len, kv_len] score tensor
        s = q[:, h * G:(h + 1) * G].double().transpose(0, 1) @ k[:, h].double().t() * scale
        p = torch.softmax(s.masked_fill_(future, float("-inf")), dim=-1)
        out[:, h * G:(h + 1) * G] = (p @ v[:, h].double()).transpose(0, 1)
    return out


def attention_floor_scale(first_pos: int, q_len: int) -> torch.Tensor:
    """Per query row of one sequence, the factor on attention_bar's 2^-16 floor: keys accumulated in one pass / 2048,
    at least 1.  The tensor-core MMA does not round its fp32 accumulation like an FADD, so the error of O grows with
    the number of MMAs chained into one accumulator.  A prefill row chains its whole context (2 MMAs per 16 keys,
    hi and lo); decode restarts every 128-token split and merges the splits in ordinary fp32 arithmetic (q_len 1: 1).
    Measured on H100: a chunk at context 7680 .. 8191 misses the plain 2^-16 floor by up to ~2x on a few elements."""
    if q_len == 1:
        return torch.ones(1, 1, 1, dtype=torch.float64)
    keys = first_pos + 1 + torch.arange(q_len, dtype=torch.float64)
    return (keys / 2048).clamp_min(1.0)[:, None, None]


def attention_bar(out: torch.Tensor, ref: torch.Tensor, floor_scale: torch.Tensor | None = None
                  ) -> tuple[int, float, str]:
    """The accuracy bar of the attention kernels (P reaches the tensor cores as bf16 hi + lo, ~16 mantissa bits):
    every element within one bf16 ulp of the float64 reference, or within 2^-16 * floor_scale of its row's largest
    |ref| (the floor for near-cancelling outputs; floor_scale broadcasts against ref[..., :1], attention_floor_scale).
    out bf16 [..., 128], ref float64, same shape.
    Returns (elements over the bar, fraction bit-exact to bf16(ref), description of the worst element, which also
    gives the largest error / floor ratio)."""
    o = out.to(ref.device).double()
    err = (o - ref).abs()
    ulp = torch.exp2(torch.floor(torch.log2(ref.abs().clamp_min(1e-30))) - 7)
    floor = 2.0 ** -16 * ref.abs().amax(dim=-1, keepdim=True)
    if floor_scale is not None:
        floor = floor * floor_scale.to(ref.device)
    bad = (err > ulp) & (err > floor)
    exact = float((out.to(ref.device) == ref.to(torch.bfloat16)).double().mean())
    over_ulp = err > ulp
    ratio = float(torch.where(over_ulp, err / floor.clamp_min(1e-300), torch.zeros_like(err)).max()) if bool(
        over_ulp.any()) else 0.0
    worst = f"max error / floor where over 1 ulp: {ratio:.2f}"
    n_bad = int(bad.sum())
    if n_bad:
        i = int(torch.argmax(torch.where(bad, err / ulp, torch.zeros_like(err))))
        idx = np.unravel_index(i, tuple(ref.shape))
        worst += (f"; worst at {tuple(int(j) for j in idx)}: out {float(o.flatten()[i])!r} "
                  f"ref {float(ref.flatten()[i])!r} ({float((err / ulp).flatten()[i]):.1f} ulp)")
    return n_bad, exact, worst


def k_cache_from_dense(k: torch.Tensor, n_blocks: int) -> torch.Tensor:
    """k: [tokens, n_kv, 128] (already placed: token t lives in slot t) -> engine K layout
    [blocks][n_kv][16 chunks][32 tok][8]."""
    t, n_kv, _ = k.shape
    pad = torch.zeros(n_blocks * KV_BLOCK, n_kv, HEAD_DIM, dtype=k.dtype, device=k.device)
    pad[:t] = k
    x = pad.view(n_blocks, KV_BLOCK, n_kv, 16, 8).permute(0, 2, 3, 1, 4).contiguous()
    return x


def v_cache_from_dense(v: torch.Tensor, n_blocks: int) -> torch.Tensor:
    """-> engine V layout [blocks][n_kv][32 tok][16 chunks ^ (tok & 7)][8]."""
    t, n_kv, _ = v.shape
    pad = torch.zeros(n_blocks * KV_BLOCK, n_kv, HEAD_DIM, dtype=v.dtype, device=v.device)
    pad[:t] = v
    x = pad.view(n_blocks, KV_BLOCK, n_kv, 16, 8).permute(0, 2, 1, 3, 4).contiguous()  # [b][kv][tok][chunk][8]
    tok = torch.arange(KV_BLOCK, device=v.device)
    chunk = torch.arange(16, device=v.device)
    src = (chunk[None, :] ^ (tok[:, None] & 7))  # physical p holds logical p ^ (tok&7)
    idx = src[None, None, :, :, None].expand(n_blocks, n_kv, KV_BLOCK, 16, 8)
    return torch.gather(x, 3, idx).contiguous()


def dense_from_k_cache(kc: torch.Tensor) -> torch.Tensor:
    nb, n_kv = kc.shape[0], kc.shape[1]
    return kc.permute(0, 3, 1, 2, 4).reshape(nb * KV_BLOCK, n_kv, HEAD_DIM)


def dense_from_v_cache(vc: torch.Tensor) -> torch.Tensor:
    nb, n_kv = vc.shape[0], vc.shape[1]
    tok = torch.arange(KV_BLOCK, device=vc.device)
    chunk = torch.arange(16, device=vc.device)
    src = (chunk[None, :] ^ (tok[:, None] & 7))
    idx = src[None, None, :, :, None].expand(nb, n_kv, KV_BLOCK, 16, 8)
    x = torch.gather(vc, 3, idx)  # xor is an involution
    return x.permute(0, 2, 1, 3, 4).reshape(nb * KV_BLOCK, n_kv, HEAD_DIM)


def run_sampler(logits: torch.Tensor, rows: np.ndarray, bitmap: torch.Tensor | None = None, iters: int = 1,
                return_us: bool = False, allow: torch.Tensor | None = None):
    """logits: fp32 (golden fixtures) or bf16 (the product path's dtype) [rows, V] on the device."""
    assert rows.dtype == SAMPLE_ROW_DTYPE and rows.dtype.itemsize == lib().tgis_k_sizeof_sample_row()
    assert SAMPLE_OUT_DTYPE.itemsize == lib().tgis_k_sizeof_sample_out()
    assert logits.dtype in (torch.float32, torch.bfloat16)
    out = np.zeros(len(rows), dtype=SAMPLE_OUT_DTYPE)
    us = C.c_float(0)
    # allow: [slots, ceil(V/32)] int32 guided-decoding bitmask on the device, used by rows flagged SAMPLE_MASKED
    rc = lib().tgis_k_sampler_masked(ptr(logits), 1 if logits.dtype == torch.bfloat16 else 0, logits.stride(0),
                                     logits.shape[1], rows.ctypes.data_as(C.c_void_p), len(rows),
                                     ptr(bitmap) if bitmap is not None else None,
                                     ptr(allow) if allow is not None else None, out.ctypes.data_as(C.c_void_p),
                                     iters, C.byref(us))
    assert rc == 0, kerr()
    return (out, us.value) if return_us else out
