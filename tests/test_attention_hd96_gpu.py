"""The 96-dim-head (Phi-3-mini) instantiations of the RoPE + KV writer and of the attention kernels (decode + split merge,
prefill, chunked prefill, split-context prefill), through the tgis_k_*_hd / _window hooks, and the V-tile chunk
permutation they share.

At D = 96 a K tile is [12 chunks][32 tok][8] and a V tile [32 tok][12 chunks, permuted][8], 6 KiB each.  The V
permutation (kernels.h v_chunk<96>) stores logical chunk c of token t at physical chunk
  c < 8:   c ^ (t & 7)
  c >= 8:  8 + ((c - 8) ^ ((t >> 1) & 3))
an involution that keeps every chunk inside the token's 192-byte row (c ^ (t & 7) would not, for c = 8..11).  The dense
<-> cache helpers below restate it independently of the kernels.  Attention is held to the bar of
tests/test_attention_hd64_gpu.py (tgis_gpu_utils.attention_bar: one bf16 ulp of a float64 reference or 2^-16 of the
row's largest |reference|, at least 99 % bit-exact), with and without a sliding window; slots a sequence must not see
hold finite poison, and blocks wholly below a window hold NaN.

The bank-group check of the readers' ldmatrix.trans addresses runs without a GPU.
"""
import math

import numpy as np
import pytest
import torch

D = 96
CHUNKS = D // 8
SCALE = float(np.float32(1.0 / math.sqrt(D)))
HEADS = [(32, 32), (8, 4), (16, 4), (16, 2)]   # Phi-3-mini (G = 1), G = 2, 4, 8
POISON_K, POISON_V = 32.0, 512.0
EXTREME_K, EXTREME_V = 16384.0, 32768.0
Q_BIAS = 0.5
MIN_EXACT = 0.99


def v_chunk(c, t):
    """physical 16-byte chunk of logical chunk c of token t (ints or integer arrays)"""
    return np.where(c < 8, c ^ (t & 7), 8 + ((c - 8) ^ ((t >> 1) & 3)))


# ------------------------------------------------------------------------------------------------ swizzle (no GPU)
def test_v_chunk_is_an_involution_inside_the_row():
    c, t = np.meshgrid(np.arange(CHUNKS), np.arange(32), indexing="ij")
    p = v_chunk(c, t)
    assert p.min() == 0 and p.max() == CHUNKS - 1
    for tok in range(32):
        assert sorted(p[:, tok].tolist()) == list(range(CHUNKS))
    assert np.array_equal(v_chunk(p, t), c)
    # and the plain xor would leave the row for chunks 8..11
    assert (c ^ (t & 7)).max() == 15


def _bank_groups(addrs):
    return sorted(((a // 16) % 8) for a in addrs)


def test_readers_ldmatrix_trans_matrices_hit_eight_distinct_bank_groups():
    """Each 8-lane phase of ldmatrix.x4.trans reads one 8 x 16-byte matrix; it is conflict-free when its 8 row addresses
    fall in 8 distinct 16-byte bank groups.  The addresses are those of attention.cu: decode tok = kk*16 + (mi>>1)*8 + ri,
    chunk 2(md+u) + (mi&1); prefill tok = kk*16 + (mi&1)*8 + ri, chunk nd + (mi>>1); byte offset tok*192 +
    v_chunk(chunk, tok)*16."""
    n_mat = 0
    for kk in range(2):
        for mi in range(4):
            for md in range(0, D // 16, 2):
                for u in range(2):
                    rows = [(kk * 16 + (mi >> 1) * 8 + ri, 2 * (md + u) + (mi & 1)) for ri in range(8)]
                    assert _bank_groups([t * 2 * D + int(v_chunk(c, t)) * 16 for t, c in rows]) == list(range(8))
                    n_mat += 1
            for nd in range(0, D // 8, 2):
                rows = [(kk * 16 + (mi & 1) * 8 + ri, nd + (mi >> 1)) for ri in range(8)]
                assert _bank_groups([t * 2 * D + int(v_chunk(c, t)) * 16 for t, c in rows]) == list(range(8))
                n_mat += 1
    assert n_mat == 2 * 4 * (6 + 6)


def test_writer_thread_mapping_is_exact():
    """96 threads per CTA = 16 heads x 6 threads: every (head, chunk) of a CTA is written by exactly one thread and no
    thread maps to a head of the next CTA"""
    CH, threads = D // 16, 96
    seen = {(tid // CH, tid % CH) for tid in range(threads)}
    assert len(seen) == threads and max(h for h, _ in seen) == 15


# ------------------------------------------------------------------------------------------------ layout helpers
def _perm(n_blocks, n_kv, device):
    c = torch.arange(CHUNKS, device=device)[None, :]
    t = torch.arange(32, device=device)[:, None]
    src = torch.where(c < 8, c ^ (t & 7), 8 + ((c - 8) ^ ((t >> 1) & 3)))   # an involution: phys p holds logical src
    return src[None, None, :, :, None].expand(n_blocks, n_kv, 32, CHUNKS, 8)


def k_cache_from_dense(k, n_blocks):
    n_kv = k.shape[1]
    return k.view(n_blocks, 32, n_kv, CHUNKS, 8).permute(0, 2, 3, 1, 4).contiguous()


def v_cache_from_dense(v, n_blocks):
    n_kv = v.shape[1]
    x = v.view(n_blocks, 32, n_kv, CHUNKS, 8).permute(0, 2, 1, 3, 4).contiguous()
    return torch.gather(x, 3, _perm(n_blocks, n_kv, v.device)).contiguous()


def dense_from_k_cache(kc):
    nb, n_kv = kc.shape[:2]
    return kc.permute(0, 3, 1, 2, 4).reshape(nb * 32, n_kv, D)


def dense_from_v_cache(vc):
    nb, n_kv = vc.shape[:2]
    x = torch.gather(vc, 3, _perm(nb, n_kv, vc.device))
    return x.permute(0, 2, 1, 3, 4).reshape(nb * 32, n_kv, D)


@pytest.fixture(scope="module")
def g():
    import tgis_gpu_utils as gpu_utils

    assert torch.cuda.is_available()
    return gpu_utils


# ------------------------------------------------------------------------------------------------ RoPE + KV writer
@pytest.mark.gpu
@pytest.mark.parametrize("n_q,n_kv", [(32, 32), (4, 2), (3, 3), (16, 2)])
def test_rope_and_kv_writer_at_96_dim_heads_match_the_oracle_bit_for_bit(g, n_q, n_kv):
    """q / k rotated as the oracle's _rope (pairs (i, i + 48)), v untouched; k / v in their slots of the 96-dim layout,
    slots < 0 not cached, no other slot written.  (3, 3) and (4, 2) leave the last CTA's 16 heads partly empty."""
    from oracle.llama_oracle import LlamaConfig, LlamaOracle

    T, n_blocks, max_pos = 70, 9, 512
    gen = torch.Generator(device="cuda").manual_seed(n_q + 7 * n_kv)
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
    cfg = LlamaConfig(n_layers=1, hidden=96, n_q_heads=n_q, n_kv_heads=n_kv, ffn=64, vocab=8, head_dim=D,
                      max_model_len=8)
    ora = LlamaOracle.__new__(LlamaOracle)
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
    assert torch.equal(k_cache_from_dense(k_dense, n_blocks), kc) and torch.equal(v_cache_from_dense(v_dense, n_blocks), vc)


# ------------------------------------------------------------------------------------------------ attention
def reference_f64(q, k, v, first_pos, window):
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
        s = q[:, h * G:(h + 1) * G].double().transpose(0, 1) @ k[:, h].double().t() * SCALE
        p = torch.softmax(s.masked_fill_(hidden, float("-inf")), dim=-1)
        out[:, h * G:(h + 1) * G] = (p @ v[:, h].double()).transpose(0, 1)
    return out


def _seq_kv(mode, kv_len, n_kv, gen):
    k = torch.randn(kv_len, n_kv, D, generator=gen, device="cuda") * 1.5
    v = torch.randn(kv_len, n_kv, D, generator=gen, device="cuda")
    if mode == "peak_last":
        k = k * 4.0
        k[kv_len - 1] += 8.0
    elif mode == "wide_v":
        v = v * torch.exp2(torch.randint(-12, 13, v.shape, generator=gen, device="cuda").float())
    elif mode == "uniform":
        k = k[:1].expand(kv_len, n_kv, D).clone()
    else:
        assert mode == "rand", mode
    return k.bfloat16(), v.bfloat16()


class Case:
    """specs = [(context before this step, q_len)] over one paged 96-dim cache, blocks scattered over a permuted pool"""

    def __init__(self, g, n_q, n_kv, specs, window, seed, modes=("rand", "peak_last", "wide_v", "uniform")):
        self.g, self.n_q, self.n_kv, self.specs, self.window = g, n_q, n_kv, specs, window
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
        cur, q_start = 0, 0
        for s, ((ctx, ql), nb) in enumerate(zip(specs, nbs)):
            blocks = order[cur: cur + nb]
            cur += nb
            self.bt[s, :nb] = blocks.cpu().numpy()
            kv_len = ctx + ql
            k, v = _seq_kv(modes[s % len(modes)], kv_len, n_kv, gen)
            pos = torch.arange(kv_len, device="cuda")
            slots = blocks[pos // 32] * 32 + pos % 32
            k_pool[slots], v_pool[slots] = k, v
            if window:
                lo = max(0, ctx - window + 1)
                hid, nan = pos < lo, pos < (lo // 32) * 32
                k_pool[slots[hid]], v_pool[slots[hid]] = EXTREME_K, EXTREME_V
                k_pool[slots[nan]], v_pool[slots[nan]] = float("nan"), float("nan")
            self.kv.append((k, v))
            self.seqs[s] = (q_start, ql, kv_len, s)
            q_start += ql
        self.kc = k_cache_from_dense(k_pool, n_blocks)
        self.vc = v_cache_from_dense(v_pool, n_blocks)

    def run(self, mode=0):
        out = torch.zeros(self.q.shape, dtype=torch.bfloat16, device="cuda")
        g = self.g
        rc = g.lib().tgis_k_attention_window(D, g.ptr(self.qkv), g.ptr(self.kc), g.ptr(self.vc),
                                             g.i32p(self.seqs.reshape(-1)), len(self.specs),
                                             g.i32p(self.bt.reshape(-1)), len(self.specs), self.bt_stride, g.ptr(out),
                                             self.n_q, self.n_kv, SCALE, mode, self.window)
        assert rc == 0, g.kerr()
        return out

    def reference(self):
        ref = torch.empty(self.q.shape, dtype=torch.float64, device="cuda")
        floor = torch.empty(self.q.shape[0], 1, 1, dtype=torch.float64)
        for (ctx, ql), (k, v), (q0, *_) in zip(self.specs, self.kv, self.seqs):
            ref[q0: q0 + ql] = reference_f64(self.q[q0: q0 + ql], k, v, ctx, self.window)
            floor[q0: q0 + ql] = self.g.attention_floor_scale(ctx, ql)
        return ref, floor


def _assert_bar(g, out, ref, floor, what):
    assert not bool(torch.isnan(out).any()), f"{what}: NaN in the output"
    n_bad, exact, worst = g.attention_bar(out, ref, floor)
    print(f"{what}: {exact * 100:.2f} % bit-exact, {n_bad} over the bar ({worst})")
    assert n_bad == 0, f"{what}: {n_bad} elements over the bar; {worst}"
    assert exact >= MIN_EXACT, f"{what}: only {exact * 100:.2f} % bit-exact"


@pytest.mark.gpu
@pytest.mark.parametrize("W", [0, 40])
@pytest.mark.parametrize("n_q,n_kv", HEADS)
def test_decode_at_96_dim_heads_meets_float64_bar(g, n_q, n_kv, W):
    """contexts at the block and split boundaries and through the merge kernel (33 splits), and enough sequences that
    every warp slot takes several items, so the tile ring runs across item boundaries; two launches give the same bits"""
    slots = 2 * 4 * torch.cuda.get_device_properties(0).multi_processor_count
    lengths = [1, 2, 31, 32, 33, 127, 128, 129, 4097, 8192]
    rng = np.random.RandomState(n_q * 100 + n_kv + W)
    while sum((n + 127) // 128 for n in lengths) * n_kv <= 3 * slots:
        lengths.append(int(rng.randint(1, 8193)))
    case = Case(g, n_q, n_kv, [(n - 1, 1) for n in lengths], W, seed=n_q * 10 + n_kv + W)
    out = case.run()
    _assert_bar(g, out, *case.reference(), f"decode D=96 ({n_q}, {n_kv}) W={W}, {len(lengths)} sequences")
    assert torch.equal(out, case.run()), "two launches differ"


PREFILL_SPECS = [(0, 2048), (7680, 512), (4097, 2), (4097, 17), (3001, 1000), (33, 17), (4095, 2), (1000, 17), (0, 17),
                 (500, 1000), (8191, 1), (4096, 1), (128, 1), (0, 1), (30, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("W", [0, 100])
@pytest.mark.parametrize("n_q,n_kv", HEADS)
def test_prefill_and_chunked_prefill_at_96_dim_heads_meet_float64_bar(g, n_q, n_kv, W):
    case = Case(g, n_q, n_kv, PREFILL_SPECS, W, seed=n_q * 1000 + n_kv + W)
    out = case.run(0)
    _assert_bar(g, out, *case.reference(), f"prefill + decode D=96 ({n_q}, {n_kv}) W={W}")
    assert torch.equal(out, case.run(0)), "two launches differ"


SPLIT_SPECS = [(1024, 128), (1024, 1), (8000, 100), (4097, 17), (2048, 16), (1500, 33), (3, 5), (0, 40), (40, 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("W", [0, 100])
@pytest.mark.parametrize("n_q,n_kv", HEADS)
def test_split_context_prefill_at_96_dim_heads_meets_float64_bar(g, n_q, n_kv, W):
    """every prefill sequence on the split-context cluster kernel (mode 1), then the engine's selection (mode 2)"""
    case = Case(g, n_q, n_kv, SPLIT_SPECS, W, seed=n_q * 7 + n_kv + W)
    ref, floor = case.reference()
    for mode in (1, 2):
        out = case.run(mode)
        _assert_bar(g, out, ref, floor, f"split-context prefill D=96 mode {mode} ({n_q}, {n_kv}) W={W}")
        assert torch.equal(out, case.run(mode)), "two launches differ"


@pytest.mark.gpu
@pytest.mark.parametrize("n_q,n_kv", [(6, 2), (10, 2)])
def test_uninstantiated_groups_are_refused_at_96_dim_heads_not_run(g, n_q, n_kv):
    """(head_dim 96, G = 3 or 5) is not instantiated: the decode launcher reports it instead of running another kernel"""
    case = Case(g, 4, 4, [(9, 1)], 0, seed=1)
    out = torch.zeros(1, n_q, D, dtype=torch.bfloat16, device="cuda")
    rc = g.lib().tgis_k_attention_hd(D, g.ptr(case.qkv), g.ptr(case.kc), g.ptr(case.vc), g.i32p(case.seqs.reshape(-1)),
                                     1, g.i32p(case.bt.reshape(-1)), 1, case.bt_stride, g.ptr(out), n_q, n_kv, SCALE)
    assert rc != 0 and "invalid" in g.kerr().lower()
