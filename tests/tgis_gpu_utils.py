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


# ------------------------------------------------------------------------------ RMSNorm / LayerNorm restatements
# The summation order of rmsnorm_kernel (csrc/elementwise.cu) and opt_layernorm_kernel (csrc/opt.cu) restated with fp32
# torch ops on the device, so that the kernels can be compared with torch.equal.  On the device torch.rsqrt is the
# kernels' rsqrtf, and the division by a 0-dim CUDA tensor is IEEE division like the kernels' (torch divides by a Python
# number by multiplying with its reciprocal, which is not the same for widths that are not powers of two).
NORM_THREADS = 256


def rmsnorm_vectors(hidden: int) -> int:
    """NORM_MAX_VEC of the rmsnorm_kernel instantiation rmsnorm_launch picks: 16-byte vectors per thread"""
    return 1 if hidden <= NORM_THREADS * 8 else 2 if hidden <= NORM_THREADS * 16 else 4


def layernorm_geometry(hidden: int) -> tuple[int, int]:
    """(LN_THREADS, LN_MAX_VEC) of the opt_layernorm_kernel instantiation opt_layernorm_launch picks"""
    if hidden <= 1024:
        return 128, 1
    return (256, 1) if hidden <= 2048 else (256, 2) if hidden <= 4096 else (256, 4)


def norm_slices(v: torch.Tensor, threads: int, nvec: int) -> list[torch.Tensor]:
    """v [T, H] -> the [T, threads] slices in the order every thread visits its elements: thread tid owns the 8-element
    vectors i = tid + threads * j (j < nvec) and goes through them j by j, element by element.  Past H: zeros."""
    T, H = v.shape
    pad = torch.zeros(T, nvec * threads * 8, dtype=v.dtype, device=v.device)
    pad[:, :H] = v
    p = pad.view(T, nvec, threads, 8)
    return [p[:, j, :, e] for j in range(nvec) for e in range(8)]


def _xor_butterfly(v: torch.Tensor) -> torch.Tensor:
    """[..., 32] lanes -> [...]: v += shfl_xor(v, o) for o = 16, 8, 4, 2, 1 (every lane ends with the same sum)"""
    while v.shape[-1] > 1:
        h = v.shape[-1] // 2
        v = v[..., :h] + v[..., h:]
    return v[..., 0]


def norm_block_sum(partials: torch.Tensor) -> torch.Tensor:
    """block_sum / bsum: [T, threads] per-thread fp32 partials -> [T].  Each warp's butterfly; the warp sums in lanes
    0 .. threads / 32 - 1 and zeros in the other lanes; the same butterfly over those 32 lanes."""
    T, threads = partials.shape
    lanes = torch.zeros(T, 32, dtype=torch.float32, device=partials.device)
    lanes[:, :threads // 32] = _xor_butterfly(partials.view(T, threads // 32, 32))
    return _xor_butterfly(lanes)


def f32(x: float, like: torch.Tensor) -> torch.Tensor:
    """x as a 0-dim fp32 tensor on like's device (an operand, not a Python scalar: see above)"""
    return torch.tensor(x, dtype=torch.float32, device=like.device)


def rmsnorm_sum_of_squares(z: torch.Tensor) -> torch.Tensor:
    """z [T, H] bf16 -> rmsnorm_kernel's fp32 sum of squares [T].  Each thread adds its squares to 0 one at a time; a
    bf16 square is exact in fp32, so the kernel's fused multiply-add rounds like this multiply then add."""
    zf = z.float()
    sq = zf * zf
    s = torch.zeros(z.shape[0], NORM_THREADS, dtype=torch.float32, device=z.device)
    for part in norm_slices(sq, NORM_THREADS, rmsnorm_vectors(z.shape[1])):
        s = s + part
    return norm_block_sum(s)


def rmsnorm_restated(x: torch.Tensor, w: torch.Tensor, eps: float, residual: torch.Tensor | None = None,
                     mult: float = 1.0, divisor: int | None = None) -> tuple[torch.Tensor, torch.Tensor | None]:
    """rmsnorm_kernel<ADD, NORM_MAX_VEC, MULT> in torch.  x [T, H] bf16, w [H] bf16.  With a residual (ADD):
    z = bf16(bf16(x * m) + r) for m != 1, else bf16(x + r); without: z = x.  Then rs = rsqrt(sum of squares / H + eps)
    and out = bf16(bf16(z * rs) * w).  Returns (out, z): z is what ADD writes back to the residual (None without).
    divisor replaces H (the tests' mutants)."""
    if residual is not None:
        xf = x.float()
        if mult != 1.0:
            xf = (xf * f32(mult, x)).bfloat16().float()
        z = (xf + residual.float()).bfloat16()
    else:
        z = x
    n = f32(divisor or z.shape[1], z)
    rs = torch.rsqrt(rmsnorm_sum_of_squares(z) / n + f32(eps, z))
    out = ((z.float() * rs[:, None]).bfloat16().float() * w.float()).bfloat16()
    return out, (z if residual is not None else None)


def fma_f32(a: torch.Tensor, b: torch.Tensor, c: torch.Tensor) -> torch.Tensor:
    """fp32 a * b + c rounded once, as an FFMA does.  The product of two fp32 values is exact in float64; the float64
    sum's own rounding error is recovered (TwoSum) and decides the rounding where that sum lies exactly halfway between
    two fp32 values (rounding it to fp32 as it stands would round twice)."""
    p, cd = a.double() * b.double(), c.double()
    s = p + cd
    bv = s - p
    err = (p - (s - bv)) + (cd - bv)
    f = s.float()
    inf = torch.full_like(f, float("inf"))
    other = torch.nextafter(f, torch.where(s > f.double(), inf, -inf))      # the fp32 neighbour on s's side of f
    tie = (s == (f.double() + other.double()) * 0.5) & (err != 0)
    dinf = torch.full_like(s, float("inf"))
    s = torch.where(tie, torch.nextafter(s, torch.where(err > 0, dinf, -dinf)), s)
    return s.float()


def layernorm_restated(resid: torch.Tensor, w: torch.Tensor, b: torch.Tensor, eps: float,
                       acc: torch.Tensor | None = None, acc_bias: torch.Tensor | None = None,
                       var_divisor: int | None = None) -> tuple[torch.Tensor, torch.Tensor | None]:
    """opt_layernorm_kernel<ADD, LN_THREADS, LN_MAX_VEC> in torch.  resid [T, H] bf16, w / b [H] bf16.  With acc (ADD;
    fp32 [T, H], acc_bias [H] bf16): z = bf16(r + bf16(acc + acc_bias)); without: z = resid.  Thread partials as
    norm_slices, summed with norm_block_sum: mean = sum(z) / H; q += d * d with d = z - mean (an FFMA: fma_f32);
    rstd = rsqrt(sum(q) / H + eps); out = bf16(fma(d * rstd, w, b)).  Returns (out, z if ADD else None).
    var_divisor replaces H in the variance (the tests' mutants)."""
    T, H = resid.shape
    threads, nvec = layernorm_geometry(H)
    if acc is not None:
        z = (resid.float() + (acc + acc_bias.float()).bfloat16().float()).bfloat16()
    else:
        z = resid
    zf = z.float()
    n = f32(H, zf)
    s = torch.zeros(T, threads, dtype=torch.float32, device=z.device)
    for part in norm_slices(zf, threads, nvec):
        s = s + part
    mean = norm_block_sum(s) / n
    d = zf - mean[:, None]
    q = torch.zeros_like(s)
    for part in norm_slices(d, threads, nvec):      # past H: d = 0, and fma(0, 0, q) = q
        q = fma_f32(part, part, q)
    rstd = torch.rsqrt(norm_block_sum(q) / f32(var_divisor or H, zf) + f32(eps, zf))
    out = fma_f32(d * rstd[:, None], w.float().expand(T, H), b.float().expand(T, H)).bfloat16()
    return out, (z if acc is not None else None)


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


# ------------------------------------------------------------------------------------ paged attention cases, any D
# Shared by the sliding-window and long-context tests: the cache is built on the device from a seeded generator (no
# per-token Python loop: a case holds up to a few hundred thousand tokens), and the float64 reference runs on the device.
POISON_K, POISON_V = 32.0, 512.0
EXTREME_K, EXTREME_V = 16384.0, 32768.0
Q_BIAS = 0.5
MIN_EXACT = 0.99
REF_SCORE_BYTES = 256 << 20   # the largest float64 score tensor the reference builds at once
DECODE_SPLIT = 128            # tokens per decode split (kernels.h)


def attention_scale(D: int) -> float:
    import math

    return float(np.float32(1.0 / math.sqrt(D)))


def paged_k_cache(k: torch.Tensor, n_blocks: int) -> torch.Tensor:
    """k [n_blocks * 32, n_kv, D] (token t in slot t) -> [blocks][n_kv][D / 8 chunks][32 tok][8]"""
    n_kv, D = k.shape[1], k.shape[2]
    return k.view(n_blocks, 32, n_kv, D // 8, 8).permute(0, 2, 3, 1, 4).contiguous()


def paged_v_cache(v: torch.Tensor, n_blocks: int) -> torch.Tensor:
    """-> [blocks][n_kv][32 tok][v_chunk(D / 8 chunks, tok)][8]: chunk ^ (tok & 7); at D = 96 chunks 8..11 are xor-ed
    among themselves by (tok >> 1) & 3 (kernels.h v_chunk).  Both are involutions, so the gather index is the map."""
    n_kv, D = v.shape[1], v.shape[2]
    C_ = D // 8
    x = v.view(n_blocks, 32, n_kv, C_, 8).permute(0, 2, 1, 3, 4).contiguous()
    tok = torch.arange(32, device=v.device)[:, None]
    chunk = torch.arange(C_, device=v.device)[None, :]
    src = chunk ^ (tok & 7)
    if D == 96:
        src = torch.where(chunk < 8, src, 8 + ((chunk - 8) ^ ((tok >> 1) & 3)))
    return torch.gather(x, 3, src[None, None, :, :, None].expand(n_blocks, n_kv, 32, C_, 8)).contiguous()


def masked_reference_f64(q, k, v, first_pos, window, D):
    """float64 softmax(q k^T / sqrt(D)) v of one sequence with the causal and window masks.  One kv head at a time, and
    the query rows in chunks, so that no score tensor exceeds REF_SCORE_BYTES."""
    q_len, n_q, _ = q.shape
    kv_len, n_kv, _ = k.shape
    G = n_q // n_kv
    rows = max(1, REF_SCORE_BYTES // (8 * G * kv_len))
    kpos = torch.arange(kv_len, device=q.device)[None, :]
    out = torch.empty(q_len, n_q, D, dtype=torch.float64, device=q.device)
    for h in range(n_kv):
        kh, vh = k[:, h].double(), v[:, h].double()
        for r0 in range(0, q_len, rows):
            r1 = min(q_len, r0 + rows)
            qpos = first_pos + torch.arange(r0, r1, device=q.device)[:, None]
            hidden = kpos > qpos
            if window:
                hidden = hidden | (kpos <= qpos - window)
            s = q[r0:r1, h * G:(h + 1) * G].double().transpose(0, 1) @ kh.t() * attention_scale(D)
            p = torch.softmax(s.masked_fill_(hidden, float("-inf")), dim=-1)
            out[r0:r1, h * G:(h + 1) * G] = (p @ vh).transpose(0, 1)
            del s, p
    return out


def needle_positions(kv_len: int) -> list[int]:
    """keys in decode splits 70 and 700 and in the last split (those the sequence has)"""
    last = (kv_len - 1) // DECODE_SPLIT
    pos = [sp * DECODE_SPLIT + off for sp, off in ((70, 37), (700, 91)) if sp < last]
    return pos + [last * DECODE_SPLIT + min(5, kv_len - 1 - last * DECODE_SPLIT)]


def paged_seq_kv(mode, kv_len, n_kv, D, gen):
    """K / V of one sequence, drawn on the device.  The queries are randn + Q_BIAS in every dimension, so a key along
    the all-ones direction scores about Q_BIAS * sqrt(D) per unit of its value (in units of the softmax's e-fold):
      rand       K ~ 1.5 randn, V ~ randn
      peak_last  K scaled by 4 and the last key lifted by 8
      wide_v     V spread over 2^-12 .. 2^12
      needles    rand plus keys in decode splits 70, 700 and the last one that score about 11 - 13 above the mean, each
                 as heavy as a large part of the 8k - 128k bulk: the output depends on every chunk of 64 splits
      rising     rand plus a ramp that lifts the scores by about 40 from the first key to the last: the running maximum
                 moves from chunk to chunk, so the merge's exp2(m_split - m_final) rescaling carries the result
      cliff      rand with the last split's keys lifted by about 200 (290 in the kernel's log2 domain; the spread over the
                 query heads is 2 / sqrt(D) of that per standard deviation): a merge that took the row maximum without
                 that split would overflow exp2f to inf in the typical head (NaN out)"""
    k = torch.randn(kv_len, n_kv, D, generator=gen, device="cuda") * 1.5
    v = torch.randn(kv_len, n_kv, D, generator=gen, device="cuda")
    unit = 1.0 / (Q_BIAS * D ** 0.5)   # K value per unit of expected score along the all-ones direction
    if mode == "peak_last":
        k = k * 4.0
        k[kv_len - 1] += 8.0
    elif mode == "wide_v":
        v = v * torch.exp2(torch.randint(-12, 13, v.shape, generator=gen, device="cuda").float())
    elif mode == "needles":
        for i, p in enumerate(needle_positions(kv_len)):
            k[p] = (11.0 + i) * unit
    elif mode == "rising":
        k += (40.0 * unit / kv_len) * torch.arange(kv_len, device="cuda", dtype=torch.float32)[:, None, None]
    elif mode == "cliff":
        k[(kv_len - 1) // DECODE_SPLIT * DECODE_SPLIT:] += 200.0 * unit
    else:
        assert mode == "rand", mode
    return k.bfloat16(), v.bfloat16()


class PagedCase:
    """specs = [(context before this step, q_len[, K / V mode])] over one paged cache of D-dim heads, blocks scattered
    over a permuted pool; a spec without a mode takes modes[index % len(modes)].  Poisoned for `window`:
      * every cache block wholly below the lowest position any row of the sequence sees is NaN (K and V): the kernels
        must never load it, since a NaN value times p = 0 is still NaN;
      * the positions of the block holding that lowest visible position that lie below it hold finite extremes (K 2^14,
        V 2^15): loaded, and they must be masked;
      * slots outside every sequence hold a finite poison (K 32, V 512)."""

    def __init__(self, D, n_q, n_kv, specs, window, seed, modes=("rand", "peak_last", "wide_v")):
        self.D, self.n_q, self.n_kv, self.window = D, n_q, n_kv, window
        self.specs = [(s[0], s[1]) for s in specs]
        self.modes = [s[2] if len(s) > 2 else modes[i % len(modes)] for i, s in enumerate(specs)]
        gen = torch.Generator(device="cuda").manual_seed(seed)
        T = sum(q for _, q in self.specs)
        self.q = (torch.randn(T, n_q, D, generator=gen, device="cuda") + Q_BIAS).bfloat16()
        self.qkv = torch.zeros(T, n_q + 2 * n_kv, D, dtype=torch.bfloat16, device="cuda")
        self.qkv[:, :n_q] = self.q
        nbs = [(c + q + 31) // 32 for c, q in self.specs]
        self.bt_stride = max(nbs)
        n_blocks = sum(nbs) + 8
        order = torch.from_numpy(np.random.RandomState(seed).permutation(n_blocks)).cuda()
        k_pool = torch.full((n_blocks * 32, n_kv, D), POISON_K, dtype=torch.bfloat16, device="cuda")
        v_pool = torch.full((n_blocks * 32, n_kv, D), POISON_V, dtype=torch.bfloat16, device="cuda")
        self.bt = np.zeros((len(self.specs), self.bt_stride), dtype=np.int32)
        self.seqs = np.zeros((len(self.specs), 4), dtype=np.int32)
        self.kv = []
        self.n_nan_blocks = 0
        cur, q_start = 0, 0
        for s, ((ctx, ql), nb, mode) in enumerate(zip(self.specs, nbs, self.modes)):
            blocks = order[cur: cur + nb]
            cur += nb
            self.bt[s, :nb] = blocks.cpu().numpy()
            kv_len = ctx + ql
            k, v = paged_seq_kv(mode, kv_len, n_kv, D, gen)
            pos = torch.arange(kv_len, device="cuda")
            slots = blocks[pos // 32] * 32 + pos % 32
            k_pool[slots], v_pool[slots] = k, v
            if window:
                lo = max(0, ctx - window + 1)   # the lowest position the first query row sees
                hid = pos < lo
                nan = pos < (lo // 32) * 32
                self.n_nan_blocks += lo // 32
                k_pool[slots[hid]], v_pool[slots[hid]] = EXTREME_K, EXTREME_V
                k_pool[slots[nan]], v_pool[slots[nan]] = float("nan"), float("nan")
            self.kv.append((k, v))
            self.seqs[s] = (q_start, ql, kv_len, s)
            q_start += ql
        self.kc = paged_k_cache(k_pool, n_blocks)
        self.vc = paged_v_cache(v_pool, n_blocks)
        del k_pool, v_pool

    def run(self, mode=0, window=None):
        """tgis_k_attention_window: mode 0 every prefill tile on the plain kernel, 1 on the split-context kernel, 2 the
        engine's selection; decode rows (q_len 1) on the decode kernel and the split merge in every mode"""
        out = torch.zeros(self.q.shape, dtype=torch.bfloat16, device="cuda")
        rc = lib().tgis_k_attention_window(self.D, ptr(self.qkv), ptr(self.kc), ptr(self.vc),
                                           i32p(self.seqs.reshape(-1)), len(self.specs), i32p(self.bt.reshape(-1)),
                                           len(self.specs), self.bt_stride, ptr(out), self.n_q, self.n_kv,
                                           attention_scale(self.D), mode, self.window if window is None else window)
        assert rc == 0, kerr()
        return out

    def reference(self, floor=attention_floor_scale):
        """float64 reference [T, n_q, D] and the per-row floor factor, floor(context, q_len) per sequence"""
        ref = torch.empty(self.q.shape, dtype=torch.float64, device="cuda")
        scale = torch.empty(self.q.shape[0], 1, 1, dtype=torch.float64)
        for (ctx, ql), (k, v), (q0, *_) in zip(self.specs, self.kv, self.seqs):
            ref[q0: q0 + ql] = masked_reference_f64(self.q[q0: q0 + ql], k, v, ctx, self.window, self.D)
            scale[q0: q0 + ql] = floor(ctx, ql)
        return ref, scale


def assert_attention_bar(out, ref, floor, what):
    """attention_bar with no element over it, no NaN and at least MIN_EXACT bit-exact; returns the worst-element text"""
    assert not bool(torch.isnan(out).any()), f"{what}: NaN in the output"
    n_bad, exact, worst = attention_bar(out, ref, floor)
    print(f"{what}: {exact * 100:.2f} % bit-exact, {n_bad} over the bar ({worst})")
    assert n_bad == 0, f"{what}: {n_bad} elements over the bar; {worst}"
    assert exact >= MIN_EXACT, f"{what}: only {exact * 100:.2f} % bit-exact"
    return worst


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
