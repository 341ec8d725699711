"""-m gpu: sliding-window attention in the decode (+ split merge), prefill, chunked prefill and split-context prefill
kernels, at 128- and 64-dim heads, through tgis_k_attention_window.

The query at position p sees the keys p - W < k <= p.  Every output is held to the bar of
tests/test_attention_precision_gpu.py against a float64 reference with that mask: within one bf16 ulp, or within 2^-16 of
the row's largest |reference| times the chained-key factor, and at least 99 % bit-exact.  The cache is poisoned so that a
kernel that reads what it must not shows it:
  * every cache block wholly below the lowest position any row of the sequence sees is NaN (K and V): the kernels must
    never load it, since a NaN value times p = 0 is still NaN;
  * the positions of the block holding that lowest visible position that lie below it hold finite extremes (K 2^14,
    V 2^15): loaded, and they must be masked;
  * slots outside every sequence hold the finite poison of the full-attention tests.
A window no shorter than the context is bit-identical to window 0, and two launches give the same bits.
"""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

POISON_K, POISON_V = 32.0, 512.0
EXTREME_K, EXTREME_V = 16384.0, 32768.0
Q_BIAS = 0.5
MIN_EXACT = 0.99
HEADS = {128: [(32, 8), (8, 2), (64, 8), (6, 2), (4, 4)], 64: [(32, 8), (8, 2), (16, 2), (4, 4)]}
HEAD_CASES = [(d, nq, nkv) for d in (128, 64) for nq, nkv in HEADS[d]]


@pytest.fixture(scope="module")
def g():
    import tgis_gpu_utils as gpu_utils

    assert torch.cuda.is_available()
    return gpu_utils


def _scale(D):
    return float(np.float32(1.0 / math.sqrt(D)))


# ------------------------------------------------------------------------------------------------ layout helpers
def k_cache_from_dense(k, n_blocks):
    """k [n_blocks * 32, n_kv, D] (token t in slot t) -> [blocks][n_kv][D / 8 chunks][32 tok][8]"""
    n_kv, D = k.shape[1], k.shape[2]
    return k.view(n_blocks, 32, n_kv, D // 8, 8).permute(0, 2, 3, 1, 4).contiguous()


def v_cache_from_dense(v, n_blocks):
    """-> [blocks][n_kv][32 tok][D / 8 chunks ^ (tok & 7)][8]"""
    n_kv, D = v.shape[1], v.shape[2]
    C = D // 8
    x = v.view(n_blocks, 32, n_kv, C, 8).permute(0, 2, 1, 3, 4).contiguous()
    tok = torch.arange(32, device=v.device)
    src = torch.arange(C, device=v.device)[None, :] ^ (tok[:, None] & 7)
    return torch.gather(x, 3, src[None, None, :, :, None].expand(n_blocks, n_kv, 32, C, 8)).contiguous()


def reference_f64(q, k, v, first_pos, window, D):
    """float64 softmax(q k^T / sqrt(D)) v of one sequence with the causal and window masks"""
    q_len, n_q, _ = q.shape
    kv_len, n_kv, _ = k.shape
    G = n_q // n_kv
    qpos = first_pos + torch.arange(q_len, device=q.device)[:, None]
    kpos = torch.arange(kv_len, device=q.device)[None, :]
    hidden = kpos > qpos
    if window:
        hidden = hidden | (kpos <= qpos - window)
    out = torch.empty(q_len, n_q, D, dtype=torch.float64, device=q.device)
    for h in range(n_kv):
        s = q[:, h * G:(h + 1) * G].double().transpose(0, 1) @ k[:, h].double().t() * _scale(D)
        p = torch.softmax(s.masked_fill_(hidden, float("-inf")), dim=-1)
        out[:, h * G:(h + 1) * G] = (p @ v[:, h].double()).transpose(0, 1)
    return out


def _seq_kv(mode, kv_len, n_kv, D, gen):
    k = torch.randn(kv_len, n_kv, D, generator=gen, device="cuda") * 1.5
    v = torch.randn(kv_len, n_kv, D, generator=gen, device="cuda")
    if mode == "peak_last":
        k = k * 4.0
        k[kv_len - 1] += 8.0
    elif mode == "wide_v":
        v = v * torch.exp2(torch.randint(-12, 13, v.shape, generator=gen, device="cuda").float())
    else:
        assert mode == "rand", mode
    return k.bfloat16(), v.bfloat16()


class Case:
    """specs = [(context before this step, q_len)] over one paged cache of D-dim heads, blocks scattered over a permuted
    pool; poisoned as the module docstring says for `window`"""

    def __init__(self, g, D, n_q, n_kv, specs, window, seed, modes=("rand", "peak_last", "wide_v")):
        self.g, self.D, self.n_q, self.n_kv, self.specs, self.window = g, D, n_q, n_kv, specs, window
        gen = torch.Generator(device="cuda").manual_seed(seed)
        T = sum(q for _, q in specs)
        self.q = (torch.randn(T, n_q, D, generator=gen, device="cuda") + Q_BIAS).bfloat16()
        self.qkv = torch.zeros(T, n_q + 2 * n_kv, D, dtype=torch.bfloat16, device="cuda")
        self.qkv[:, :n_q] = self.q
        nbs = [(c + q + 31) // 32 for c, q in specs]
        self.bt_stride = max(nbs)
        n_blocks = sum(nbs) + 8
        order = torch.from_numpy(np.random.RandomState(seed).permutation(n_blocks)).cuda()
        k_pool = torch.full((n_blocks * 32, n_kv, D), POISON_K, dtype=torch.bfloat16, device="cuda")
        v_pool = torch.full((n_blocks * 32, n_kv, D), POISON_V, dtype=torch.bfloat16, device="cuda")
        self.bt = np.zeros((len(specs), self.bt_stride), dtype=np.int32)
        self.seqs = np.zeros((len(specs), 4), dtype=np.int32)
        self.kv = []
        self.n_nan_blocks = 0
        cur, q_start = 0, 0
        for s, ((ctx, ql), nb) in enumerate(zip(specs, nbs)):
            blocks = order[cur: cur + nb]
            cur += nb
            self.bt[s, :nb] = blocks.cpu().numpy()
            kv_len = ctx + ql
            k, v = _seq_kv(modes[s % len(modes)], kv_len, n_kv, D, gen)
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
        self.kc = k_cache_from_dense(k_pool, n_blocks)
        self.vc = v_cache_from_dense(v_pool, n_blocks)

    def run(self, mode=0, window=None):
        out = torch.zeros(self.q.shape, dtype=torch.bfloat16, device="cuda")
        g = self.g
        rc = g.lib().tgis_k_attention_window(self.D, g.ptr(self.qkv), g.ptr(self.kc), g.ptr(self.vc),
                                             g.i32p(self.seqs.reshape(-1)), len(self.specs),
                                             g.i32p(self.bt.reshape(-1)), len(self.specs), self.bt_stride, g.ptr(out),
                                             self.n_q, self.n_kv, _scale(self.D), mode,
                                             self.window if window is None else window)
        assert rc == 0, g.kerr()
        return out

    def reference(self):
        ref = torch.empty(self.q.shape, dtype=torch.float64, device="cuda")
        floor = torch.empty(self.q.shape[0], 1, 1, dtype=torch.float64)
        for (ctx, ql), (k, v), (q0, *_) in zip(self.specs, self.kv, self.seqs):
            ref[q0: q0 + ql] = reference_f64(self.q[q0: q0 + ql], k, v, ctx, self.window, self.D)
            floor[q0: q0 + ql] = self.g.attention_floor_scale(ctx, ql)
        return ref, floor


def _assert_bar(g, out, ref, floor, what):
    assert not bool(torch.isnan(out).any()), f"{what}: NaN in the output (a block below the window was read)"
    n_bad, exact, worst = g.attention_bar(out, ref, floor)
    print(f"{what}: {exact * 100:.2f} % bit-exact, {n_bad} over the bar ({worst})")
    assert n_bad == 0, f"{what}: {n_bad} elements over the bar; {worst}"
    assert exact >= MIN_EXACT, f"{what}: only {exact * 100:.2f} % bit-exact"


def _decode_lengths(W):
    lengths = [1, W - 1, W, W + 1, W + 31, W + 32, W + 127, W + 128, W + 129, 2 * W + 5, 8192]
    if W == 4096:
        lengths.append(32768)
    return [n for n in lengths if n >= 1]


# ------------------------------------------------------------------------------------------------ decode
@pytest.mark.parametrize("W", [40, 100, 4096])
@pytest.mark.parametrize("D,n_q,n_kv", HEAD_CASES)
def test_windowed_decode_meets_float64_bar(g, D, n_q, n_kv, W):
    """kv_len at and around the window, its block and split boundaries, and far past it; blocks wholly below the window
    are NaN.  Two launches give the same bits."""
    specs = [(n - 1, 1) for n in _decode_lengths(W)]
    case = Case(g, D, n_q, n_kv, specs, W, seed=W * 7 + n_q * 3 + n_kv + D)
    assert case.n_nan_blocks > 0
    out = case.run()
    _assert_bar(g, out, *case.reference(), f"decode D={D} ({n_q}, {n_kv}) W={W}")
    assert torch.equal(out, case.run()), "two launches differ"


@pytest.mark.parametrize("D,n_q,n_kv", [(128, 32, 8), (64, 32, 8), (128, 6, 2)])
def test_window_not_shorter_than_the_context_is_bit_identical_to_full_attention(g, D, n_q, n_kv):
    """decode, prefill and split-context prefill: with W >= every kv_len the same bits as window 0"""
    specs = [(0, 1), (126, 1), (127, 1), (4096, 1), (8191, 1), (0, 300), (1100, 17), (2000, 100), (40, 2)]
    case = Case(g, D, n_q, n_kv, specs, 0, seed=n_q + D)
    for mode in (0, 1, 2):
        full = case.run(mode, window=0)
        for W in (8192, 8193, 1 << 30):
            assert torch.equal(case.run(mode, window=W), full), (mode, W)
    # and a window that does bite changes the output (the test above would pass for a kernel ignoring the window)
    assert not torch.equal(case.run(0, window=100), case.run(0, window=0))


# ------------------------------------------------------------------------------------------------ prefill
PREFILL_WINDOWS = [40, 100, 4096]


def _prefill_specs(W):
    """whole prompts and chunks whose windows cross tile (16), block (32) and split-context rank boundaries, contexts off
    the grid, and decode rows in the same call"""
    return [(0, 2 * W + 37), (W + 5, 64), (3 * W + 17, 17), (1000, 1000), (7680, 512), (W - 1, 2), (4097, 33),
            (33, 17), (0, 1), (8191, 1), (W + 40, 1), (2 * W, 16)]


@pytest.mark.parametrize("W", PREFILL_WINDOWS)
@pytest.mark.parametrize("D,n_q,n_kv", HEAD_CASES)
def test_windowed_prefill_and_chunked_prefill_meet_float64_bar(g, D, n_q, n_kv, W):
    case = Case(g, D, n_q, n_kv, _prefill_specs(W), W, seed=W + n_q * 11 + n_kv + D)
    out = case.run(0)
    _assert_bar(g, out, *case.reference(), f"prefill + decode D={D} ({n_q}, {n_kv}) W={W}")
    assert torch.equal(out, case.run(0)), "two launches differ"


def _split_specs(W):
    """short suffixes over long contexts (the engine's split-context shape), with windows that leave some of the 8 ranks
    no visible block (W = 40: 2 or 3 visible blocks per tile) and rows whose window starts inside a rank's share"""
    return [(1024, 128), (1024, 1), (8000, 100), (4097, 17), (2048, 16), (1500, 33), (3, 5), (0, 40), (40, 2),
            (W + 3, 20), (6 * W + 1, 64)]


@pytest.mark.parametrize("W", PREFILL_WINDOWS)
@pytest.mark.parametrize("D,n_q,n_kv", HEAD_CASES)
def test_windowed_split_context_prefill_meets_float64_bar(g, D, n_q, n_kv, W):
    """every prefill sequence on the split-context cluster kernel (mode 1), then the engine's selection (mode 2)"""
    case = Case(g, D, n_q, n_kv, _split_specs(W), W, seed=W * 3 + n_q * 7 + n_kv + D)
    ref, floor = case.reference()
    for mode in (1, 2):
        out = case.run(mode)
        _assert_bar(g, out, ref, floor, f"split-context prefill D={D} mode {mode} ({n_q}, {n_kv}) W={W}")
        assert torch.equal(out, case.run(mode)), "two launches differ"


def test_negative_window_is_refused(g):
    case = Case(g, 128, 4, 4, [(9, 1)], 0, seed=1)
    out = torch.zeros(1, 4, 128, dtype=torch.bfloat16, device="cuda")
    rc = g.lib().tgis_k_attention_window(128, g.ptr(case.qkv), g.ptr(case.kc), g.ptr(case.vc),
                                         g.i32p(case.seqs.reshape(-1)), 1, g.i32p(case.bt.reshape(-1)), 1,
                                         case.bt_stride, g.ptr(out), 4, 4, _scale(128), 0, -1)
    assert rc != 0 and "window" in g.kerr()
