"""-m gpu: the 64-dim-head instantiations of the RoPE + KV writer and of the attention kernels (decode + split merge,
prefill, chunked prefill, split-context prefill), through the tgis_k_*_hd hooks.

The cache layout at D = 64 is the 128-dim one at half the width: K tile [8 chunks][32 tok][8], V tile
[32 tok][8 chunks ^ (tok & 7)][8], 4 KiB each.  The dense <-> cache helpers below restate it independently of the kernels.
Attention is held to the bar of tests/test_attention_precision_gpu.py: every element within one bf16 ulp of a float64
reference or within 2^-16 of its row's largest |reference| (tgis_gpu_utils.attention_bar), at least 99 % bit-exact, with
the same poison (aligned keys, values of 512, all finite) in every slot a sequence must not see.
"""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

D = 64
CHUNKS = D // 8
SCALE = float(np.float32(1.0 / math.sqrt(D)))
HEADS = [(32, 8), (8, 2), (16, 2), (4, 4)]  # Llama-3.2-1B (G = 4), its quarter, G = 8, G = 1
DEC_CTAS_PER_SM, DEC_WARPS = 2, 4
POISON_K, POISON_V = 32.0, 512.0
Q_BIAS = 0.5
MIN_EXACT = 0.99


@pytest.fixture(scope="module")
def g():
    import tgis_gpu_utils as gpu_utils

    assert torch.cuda.is_available()
    return gpu_utils


# ------------------------------------------------------------------------------------------------ layout helpers
def k_cache_from_dense(k, n_blocks):
    """k [n_blocks * 32, n_kv, 64] (token t in slot t) -> [blocks][n_kv][8 chunks][32 tok][8]"""
    n_kv = k.shape[1]
    return k.view(n_blocks, 32, n_kv, CHUNKS, 8).permute(0, 2, 3, 1, 4).contiguous()


def _swizzle(n_blocks, n_kv, device):
    tok = torch.arange(32, device=device)
    chunk = torch.arange(CHUNKS, device=device)
    src = chunk[None, :] ^ (tok[:, None] & 7)   # physical chunk p of token t holds logical chunk p ^ (t & 7)
    return src[None, None, :, :, None].expand(n_blocks, n_kv, 32, CHUNKS, 8)


def v_cache_from_dense(v, n_blocks):
    """-> [blocks][n_kv][32 tok][8 chunks ^ (tok & 7)][8]"""
    n_kv = v.shape[1]
    x = v.view(n_blocks, 32, n_kv, CHUNKS, 8).permute(0, 2, 1, 3, 4).contiguous()
    return torch.gather(x, 3, _swizzle(n_blocks, n_kv, v.device)).contiguous()


def dense_from_k_cache(kc):
    nb, n_kv = kc.shape[:2]
    return kc.permute(0, 3, 1, 2, 4).reshape(nb * 32, n_kv, D)


def dense_from_v_cache(vc):
    nb, n_kv = vc.shape[:2]
    x = torch.gather(vc, 3, _swizzle(nb, n_kv, vc.device))   # the xor is an involution
    return x.permute(0, 2, 1, 3, 4).reshape(nb * 32, n_kv, D)


def reference_f64(q, k, v, first_pos):
    """float64 causal softmax(q k^T / sqrt(64)) v of one sequence: q [q_len, n_q, 64], k / v [kv_len, n_kv, 64]"""
    q_len, n_q, _ = q.shape
    kv_len, n_kv, _ = k.shape
    G = n_q // n_kv
    future = torch.arange(kv_len, device=q.device)[None, :] > (first_pos + torch.arange(q_len, device=q.device))[:, None]
    out = torch.empty(q_len, n_q, D, dtype=torch.float64, device=q.device)
    for h in range(n_kv):
        s = q[:, h * G:(h + 1) * G].double().transpose(0, 1) @ k[:, h].double().t() * SCALE
        p = torch.softmax(s.masked_fill_(future, float("-inf")), dim=-1)
        out[:, h * G:(h + 1) * G] = (p @ v[:, h].double()).transpose(0, 1)
    return out


# ------------------------------------------------------------------------------------------------ RoPE + KV writer
@pytest.mark.parametrize("n_q,n_kv", [(32, 8), (4, 2), (3, 3)])
def test_rope_and_kv_writer_at_64_dim_heads_match_the_oracle_bit_for_bit(g, n_q, n_kv):
    """q / k rotated exactly as the oracle's _rope does (pairs (i, i + 32), every product rounded to bf16), v untouched;
    k / v land in their slots of the 64-dim cache layout (read back through the dense helpers above), slots < 0 are not
    cached, and no other slot is written."""
    from oracle.llama_oracle import LlamaConfig, LlamaOracle

    T, n_blocks, max_pos = 70, 9, 512
    gen = torch.Generator(device="cuda").manual_seed(n_q)
    qkv0 = (torch.randn(T, n_q + 2 * n_kv, D, generator=gen, device="cuda") * 1.5).bfloat16()
    table = (torch.rand(max_pos, D, generator=gen, device="cuda") * 2 - 1).bfloat16()
    rng = np.random.RandomState(n_q)
    positions = rng.randint(0, max_pos, T).astype(np.int32)
    slot_map = rng.permutation(n_blocks * 32)[:T].astype(np.int32)
    slot_map[5] = slot_map[40] = -1
    sentinel = 7.0
    kc = torch.full((n_blocks, n_kv, CHUNKS, 32, 8), sentinel, dtype=torch.bfloat16, device="cuda")
    vc = torch.full((n_blocks, n_kv, 32, CHUNKS, 8), sentinel, dtype=torch.bfloat16, device="cuda")
    qkv = qkv0.clone()
    rc = g.lib().tgis_k_rope_kv_hd(D, g.ptr(qkv), g.i32p(positions), g.i32p(slot_map), g.ptr(table), g.ptr(kc),
                                   g.ptr(vc), T, n_q, n_kv)
    assert rc == 0, g.kerr()

    cfg = LlamaConfig(n_layers=1, hidden=64, n_q_heads=n_q, n_kv_heads=n_kv, ffn=64, vocab=8, head_dim=D, max_model_len=8)
    ora = LlamaOracle.__new__(LlamaOracle)   # only _rope is used: needs cfg and the table
    ora.cfg, ora.cos_sin = cfg, table
    pos = torch.from_numpy(positions).long().cuda()
    want_qk = ora._rope(qkv0[:, :n_q + n_kv], pos)
    assert torch.equal(qkv[:, :n_q + n_kv], want_qk)
    assert torch.equal(qkv[:, n_q + n_kv:], qkv0[:, n_q + n_kv:])
    k_dense, v_dense = dense_from_k_cache(kc), dense_from_v_cache(vc)
    want_k = torch.full_like(k_dense, sentinel)
    want_v = torch.full_like(v_dense, sentinel)
    live = torch.from_numpy(slot_map >= 0).cuda()
    sl = torch.from_numpy(slot_map).long().cuda()[live]
    want_k[sl] = want_qk[live][:, n_q:]
    want_v[sl] = qkv0[live][:, n_q + n_kv:]
    assert torch.equal(k_dense, want_k) and torch.equal(v_dense, want_v)
    # and the helpers invert each other, so the layout above is the one the attention tests feed
    assert torch.equal(k_cache_from_dense(k_dense, n_blocks), kc) and torch.equal(v_cache_from_dense(v_dense, n_blocks), vc)


# ------------------------------------------------------------------------------------------------ attention
def _seq_kv(mode, ctx, q_len, n_kv, gen):
    """value patterns of tests/test_attention_precision_gpu.py at 64 dims"""
    kv_len = ctx + q_len
    k = torch.randn(kv_len, n_kv, D, generator=gen, device="cuda") * 1.5
    v = torch.randn(kv_len, n_kv, D, generator=gen, device="cuda")
    if mode in ("peak_last", "peak_first"):
        k = k * 4.0
        j = 0 if mode == "peak_first" else int(torch.randint(((kv_len - 1) // 32) * 32, kv_len, (1,), generator=gen,
                                                             device="cuda"))
        k[j] += 8.0
    elif mode == "uniform":
        k = k[:1].expand(kv_len, n_kv, D).clone()
    elif mode == "wide_v":
        v = v * torch.exp2(torch.randint(-12, 13, v.shape, generator=gen, device="cuda").float())
    elif mode == "ramp":
        step = 0.04 / (SCALE * Q_BIAS * D)
        ramp = (torch.arange(q_len, device="cuda", dtype=torch.float32) - (q_len - 1) / 2) * step
        k[ctx:] += ramp[:, None, None]
    else:
        assert mode == "rand", mode
    return k.bfloat16(), v.bfloat16()


class Case:
    """specs = [(context before this step, q_len, mode)] over one paged 64-dim cache; blocks scattered over a permuted pool,
    every slot outside a sequence's kv_len is poison"""

    def __init__(self, g, n_q, n_kv, specs, seed):
        self.g, self.n_q, self.n_kv, self.specs = g, n_q, n_kv, specs
        gen = torch.Generator(device="cuda").manual_seed(seed)
        T = sum(q for _, q, _ in specs)
        self.q = (torch.randn(T, n_q, D, generator=gen, device="cuda") + Q_BIAS).bfloat16()
        self.qkv = torch.zeros(T, n_q + 2 * n_kv, D, dtype=torch.bfloat16, device="cuda")
        self.qkv[:, :n_q] = self.q
        nbs = [(c + q + 31) // 32 for c, q, _ in specs]
        self.bt_stride = max(nbs)
        n_blocks = sum(nbs) + 8
        order = torch.from_numpy(np.random.RandomState(seed).permutation(n_blocks)).cuda()
        k_pool = torch.full((n_blocks * 32, n_kv, D), POISON_K, dtype=torch.bfloat16, device="cuda")
        v_pool = torch.full((n_blocks * 32, n_kv, D), POISON_V, dtype=torch.bfloat16, device="cuda")
        self.bt = np.zeros((len(specs), self.bt_stride), dtype=np.int32)
        self.seqs = np.zeros((len(specs), 4), dtype=np.int32)
        self.kv = []
        cur, q_start = 0, 0
        for s, ((ctx, ql, mode), nb) in enumerate(zip(specs, nbs)):
            blocks = order[cur: cur + nb]
            cur += nb
            self.bt[s, :nb] = blocks.cpu().numpy()
            k, v = _seq_kv(mode, ctx, ql, n_kv, gen)
            pos = torch.arange(ctx + ql, device="cuda")
            slots = blocks[pos // 32] * 32 + pos % 32
            k_pool[slots], v_pool[slots] = k, v
            self.kv.append((k, v))
            self.seqs[s] = (q_start, ql, ctx + ql, s)
            q_start += ql
        self.kc = k_cache_from_dense(k_pool, n_blocks)
        self.vc = v_cache_from_dense(v_pool, n_blocks)

    def run(self, mode=0):
        out = torch.zeros(self.q.shape, dtype=torch.bfloat16, device="cuda")
        g = self.g
        rc = g.lib().tgis_k_attention_split_hd(D, g.ptr(self.qkv), g.ptr(self.kc), g.ptr(self.vc),
                                               g.i32p(self.seqs.reshape(-1)), len(self.specs),
                                               g.i32p(self.bt.reshape(-1)), len(self.specs), self.bt_stride, g.ptr(out),
                                               self.n_q, self.n_kv, SCALE, mode)
        assert rc == 0, g.kerr()
        return out

    def reference(self):
        ref = torch.empty(self.q.shape, dtype=torch.float64, device="cuda")
        scale = torch.empty(self.q.shape[0], 1, 1, dtype=torch.float64)
        for (ctx, ql, _), (k, v), (q0, *_) in zip(self.specs, self.kv, self.seqs):
            ref[q0: q0 + ql] = reference_f64(self.q[q0: q0 + ql], k, v, ctx)
            scale[q0: q0 + ql] = self.g.attention_floor_scale(ctx, ql)
        return ref, scale


def _assert_bar(g, out, ref, floor_scale, what):
    n_bad, exact, worst = g.attention_bar(out, ref, floor_scale)
    print(f"{what}: {exact * 100:.2f} % bit-exact, {n_bad} over the bar ({worst})")
    assert n_bad == 0, f"{what}: {n_bad} elements over the bar; {worst}"
    assert exact >= MIN_EXACT, f"{what}: only {exact * 100:.2f} % bit-exact"


DEC_MODES = ["rand", "peak_last", "rand", "peak_first", "uniform", "wide_v"]


@pytest.mark.parametrize("n_q,n_kv", HEADS)
def test_decode_at_64_dim_heads_meets_float64_bar(g, n_q, n_kv):
    """Contexts 1, 127, 128, 129, 4097 (one split, the split boundary, 33 splits through the merge kernel) and enough
    further sequences that every warp slot takes several work items, so the six-deep tile ring runs across item
    boundaries; two launches give the same bits."""
    slots = DEC_CTAS_PER_SM * DEC_WARPS * torch.cuda.get_device_properties(0).multi_processor_count
    lengths = [1, 2, 31, 32, 33, 127, 128, 129, 4097, 8192]
    rng = np.random.RandomState(n_q * 100 + n_kv)
    while sum((n + 127) // 128 for n in lengths) * n_kv <= 3 * slots:
        lengths.append(int(rng.randint(1, 8193)))
    specs = [(n - 1, 1, DEC_MODES[i % len(DEC_MODES)]) for i, n in enumerate(lengths)]
    case = Case(g, n_q, n_kv, specs, seed=n_q * 10 + n_kv)
    out = case.run()
    _assert_bar(g, out, *case.reference(), f"decode D=64 ({n_q}, {n_kv}), {len(lengths)} sequences")
    assert torch.equal(out, case.run()), "two launches differ"


PREFILL_SPECS = [
    (0, 2048, "ramp"), (7680, 512, "ramp"),
    (4097, 2, "ramp"), (4097, 17, "peak_last"), (3001, 1000, "ramp"),
    (33, 17, "wide_v"), (4095, 2, "peak_first"), (1000, 17, "uniform"), (0, 17, "rand"), (500, 1000, "peak_last"),
    (8191, 1, "rand"), (4096, 1, "peak_last"), (128, 1, "wide_v"), (0, 1, "rand"), (30, 1, "uniform"),
]


@pytest.mark.parametrize("n_q,n_kv", HEADS)
def test_prefill_and_chunked_prefill_at_64_dim_heads_meet_float64_bar(g, n_q, n_kv):
    """whole prompts, chunks over contexts up to 8191 off the 16 / 32 grid, and decode rows in the same call"""
    case = Case(g, n_q, n_kv, PREFILL_SPECS, seed=n_q * 1000 + n_kv)
    out = case.run()
    _assert_bar(g, out, *case.reference(), f"prefill + decode D=64 ({n_q}, {n_kv})")
    assert torch.equal(out, case.run()), "two launches differ"


SPLIT_SPECS = [
    (1024, 128, "ramp"), (1024, 1, "rand"), (8000, 100, "peak_last"), (4097, 17, "peak_first"), (2048, 16, "uniform"),
    (1500, 33, "wide_v"), (3, 5, "rand"), (0, 40, "ramp"), (40, 2, "rand"),   # the last three: ranks with no blocks
]


@pytest.mark.parametrize("n_q,n_kv", HEADS)
def test_split_context_prefill_at_64_dim_heads_meets_float64_bar(g, n_q, n_kv):
    """every prefill sequence on the split-context cluster kernel (mode 1), then the engine's selection (mode 2: the
    short suffixes over >= 1024 tokens on the cluster kernel, the rest on the existing one)"""
    case = Case(g, n_q, n_kv, SPLIT_SPECS, seed=n_q * 7 + n_kv)
    ref, floor = case.reference()
    for mode in (1, 2):
        out = case.run(mode)
        _assert_bar(g, out, ref, floor, f"split-context prefill D=64 mode {mode} ({n_q}, {n_kv})")
        assert torch.equal(out, case.run(mode)), "two launches differ"


def test_group_size_3_is_refused_at_64_dim_heads_not_run(g):
    """(head_dim 64, G = 3) is not instantiated: the decode launcher reports it instead of running another kernel"""
    case = Case(g, 4, 4, [(9, 1, "rand")], seed=1)
    case.n_q, case.n_kv = 6, 2   # G = 3; nothing is launched, so the buffers' shapes do not matter
    out = torch.zeros(1, 6, D, dtype=torch.bfloat16, device="cuda")
    rc = g.lib().tgis_k_attention_hd(D, g.ptr(case.qkv), g.ptr(case.kc), g.ptr(case.vc), g.i32p(case.seqs.reshape(-1)),
                                     1, g.i32p(case.bt.reshape(-1)), 1, case.bt_stride, g.ptr(out), 6, 2, SCALE)
    assert rc != 0 and "invalid" in g.kerr().lower()
