"""-m gpu: both attention kernels against a float64 reference at the precision they are built for, at serving shapes.

The decode and prefill kernels feed the probabilities P to the tensor cores as a bf16 hi + lo pair (~16 mantissa bits),
so their outputs track softmax(q k^T / sqrt(d)) v computed in float64 from the same bf16 inputs far more closely than a
plain bf16-P flash kernel would.  The bar (tgis_gpu_utils.attention_bar), for every output element: within one bf16 ulp
of the reference, or within 2^-16 of the largest |reference| of its 128-dim row (times keys / 2048 for a prefill row
over more than 2048 keys, tgis_gpu_utils.attention_floor_scale); and per case at least 99 % of the elements bit-exact
to bf16(reference).  A kernel that rounds P to bf16 alone misses the second part by a wide margin.

Cache slots that a sequence must not see hold poison: keys aligned with the queries (scores in the hundreds) and values
of 512, all finite (the decode kernel relies on finite slots).  A read past a mask therefore moves an output by O(1).
"""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SCALE = float(np.float32(1.0 / math.sqrt(128)))  # the fp32 value the kernels receive
HEADS = [(32, 8), (8, 2), (64, 8), (6, 2), (4, 4)]  # Llama-3-8B, its TP-4 shard, G = 8, G = 3, G = 1
DEC_CTAS_PER_SM, DEC_WARPS = 2, 4  # attention.cu TGIS_DEC_MINB, DEC_WARPS: one decode work item per warp slot and round
POISON_K, POISON_V = 32.0, 512.0
Q_BIAS = 0.5  # every query leans towards +1 in every dim, so POISON_K * ones scores ~ 0.088 * 32 * 64 = 180
MIN_EXACT = 0.99


@pytest.fixture(scope="module")
def g():
    import tgis_gpu_utils as gpu_utils

    assert torch.cuda.is_available()
    return gpu_utils


def _seq_kv(mode, ctx, q_len, n_kv, gen):
    """K / V of one sequence (bf16 [kv_len, n_kv, 128] on the device) for a value pattern:
    rand       k ~ 1.5 N(0, 1), v ~ N(0, 1)
    peak_last  scores ~ +-20 (k ~ 6 N(0, 1)) and a key in the sequence's last block that is every head's row maximum
               (~ +45), so the running maximum changes in the last block of the last split
    peak_first the same with the maximum at key 0
    uniform    one key repeated: every score of a row is equal
    wide_v     v spans 2^-12 .. 2^12 elementwise
    ramp       a key component along the query bias that grows by 0.04 in score per position of this step's chunk
               (centred on the chunk): a causal off-by-one lets the next, more attractive key in"""
    kv_len = ctx + q_len
    dev = "cuda"
    k = torch.randn(kv_len, n_kv, 128, generator=gen, device=dev) * 1.5
    v = torch.randn(kv_len, n_kv, 128, generator=gen, device=dev)
    if mode in ("peak_last", "peak_first"):
        k = k * 4.0
        j = 0 if mode == "peak_first" else int(torch.randint(((kv_len - 1) // 32) * 32, kv_len, (1,), generator=gen,
                                                             device=dev))
        k[j] += 8.0
    elif mode == "uniform":
        k = k[:1].expand(kv_len, n_kv, 128).clone()
    elif mode == "wide_v":
        v = v * torch.exp2(torch.randint(-12, 13, v.shape, generator=gen, device=dev).float())
    elif mode == "ramp":
        step = 0.04 / (SCALE * Q_BIAS * 128)  # score per position along the query bias
        ramp = (torch.arange(q_len, device=dev, dtype=torch.float32) - (q_len - 1) / 2) * step
        k[ctx:] += ramp[:, None, None]
    else:
        assert mode == "rand", mode
    return k.bfloat16(), v.bfloat16()


class Case:
    """A batch of sequences over one paged cache: specs = [(context before this step, q_len, mode)].  Each sequence's
    blocks are scattered over a permuted physical pool (plus spare blocks); every slot outside a sequence's kv_len is
    poison."""

    def __init__(self, g, n_q, n_kv, specs, seed):
        self.g, self.n_q, self.n_kv, self.specs = g, n_q, n_kv, specs
        gen = torch.Generator(device="cuda").manual_seed(seed)
        T = sum(q for _, q, _ in specs)
        self.q = (torch.randn(T, n_q, 128, generator=gen, device="cuda") + Q_BIAS).bfloat16()
        self.qkv = torch.zeros(T, n_q + 2 * n_kv, 128, dtype=torch.bfloat16, device="cuda")
        self.qkv[:, :n_q] = self.q
        nbs = [(c + q + 31) // 32 for c, q, _ in specs]
        self.bt_stride = max(nbs)
        n_blocks = sum(nbs) + 8
        order = torch.from_numpy(np.random.RandomState(seed).permutation(n_blocks)).cuda()
        k_pool = torch.full((n_blocks * 32, n_kv, 128), POISON_K, dtype=torch.bfloat16, device="cuda")
        v_pool = torch.full((n_blocks * 32, n_kv, 128), POISON_V, dtype=torch.bfloat16, device="cuda")
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
        self.kc = g.k_cache_from_dense(k_pool, n_blocks)
        self.vc = g.v_cache_from_dense(v_pool, n_blocks)

    def run(self):
        out = torch.zeros(self.q.shape, dtype=torch.bfloat16, device="cuda")
        g = self.g
        rc = g.lib().tgis_k_attention(g.ptr(self.qkv), g.ptr(self.kc), g.ptr(self.vc), g.i32p(self.seqs.reshape(-1)),
                                      len(self.specs), g.i32p(self.bt.reshape(-1)), len(self.specs), self.bt_stride,
                                      g.ptr(out), self.n_q, self.n_kv, SCALE)
        assert rc == 0, g.kerr()
        return out

    def reference(self):
        """float64 reference [T, n_q, 128] and the per-row floor factor (tgis_gpu_utils.attention_floor_scale)"""
        ref = torch.empty(self.q.shape, dtype=torch.float64, device="cuda")
        scale = torch.empty(self.q.shape[0], 1, 1, dtype=torch.float64)
        for (ctx, ql, _), (k, v), (q0, *_) in zip(self.specs, self.kv, self.seqs):
            ref[q0: q0 + ql] = self.g.attention_reference_f64(self.q[q0: q0 + ql], k, v, ctx, SCALE)
            scale[q0: q0 + ql] = self.g.attention_floor_scale(ctx, ql)
        return ref, scale


def _assert_bar(g, out, ref, floor_scale, what):
    n_bad, exact, worst = g.attention_bar(out, ref, floor_scale)
    print(f"{what}: {exact * 100:.2f} % bit-exact, {n_bad} over the bar ({worst})")
    assert n_bad == 0, f"{what}: {n_bad} elements over the bar; {worst}"
    assert exact >= MIN_EXACT, f"{what}: only {exact * 100:.2f} % bit-exact"


DEC_MODES = ["rand", "peak_last", "rand", "peak_first", "uniform", "wide_v"]


@pytest.mark.parametrize("n_q,n_kv", HEADS)
def test_decode_at_scale_meets_float64_bar(g, n_q, n_kv):
    """Enough decode sequences (1 .. 8192 tokens, up to 64 splits) that every warp slot works through at least three
    rounds of the boustrophedon schedule, so the issue cursor and the consumer cross item boundaries; two launches give
    the same bits."""
    slots = DEC_CTAS_PER_SM * DEC_WARPS * torch.cuda.get_device_properties(0).multi_processor_count
    lengths = [1, 2, 31, 32, 33, 127, 128, 129, 4095, 4096, 4097, 8191, 8192]
    rng = np.random.RandomState(n_q * 100 + n_kv)
    while sum((n + 127) // 128 for n in lengths) * n_kv <= 3 * slots:
        lengths.append(int(rng.randint(1, 8193)))
    specs = [(n - 1, 1, DEC_MODES[i % len(DEC_MODES)]) for i, n in enumerate(lengths)]
    case = Case(g, n_q, n_kv, specs, seed=n_q * 10 + n_kv)
    out = case.run()
    _assert_bar(g, out, *case.reference(), f"decode ({n_q}, {n_kv}), {len(lengths)} sequences")
    assert torch.equal(out, case.run()), "two launches differ"


PREFILL_SPECS = [
    (0, 2048, "ramp"),          # the largest chunk, no context
    (7680, 512, "ramp"),        # a chunk ending at 8192
    (4097, 2, "ramp"), (4097, 17, "peak_last"), (3001, 1000, "ramp"),  # contexts off the 16 / 32 grid
    (33, 17, "wide_v"), (4095, 2, "peak_first"), (1000, 17, "uniform"), (0, 17, "rand"), (500, 1000, "peak_last"),
    (8191, 1, "rand"), (4096, 1, "peak_last"), (128, 1, "wide_v"), (0, 1, "rand"), (30, 1, "uniform"),  # decode rows
]


@pytest.mark.parametrize("n_q,n_kv", HEADS)
def test_prefill_and_chunked_prefill_meet_float64_bar(g, n_q, n_kv):
    """Prefill chunks of up to 2048 rows over contexts up to 8191 (256 KV blocks through the 2-stage ring), ragged
    contexts, and decode rows in the same call (decode launch + merge, then prefill, as the engine issues them)."""
    case = Case(g, n_q, n_kv, PREFILL_SPECS, seed=n_q * 1000 + n_kv)
    out = case.run()
    _assert_bar(g, out, *case.reference(), f"prefill + decode ({n_q}, {n_kv})")
    assert torch.equal(out, case.run()), "two launches differ"


# 124 splits x 8 kv heads = 992 decode items: no more than the warp slots of an H100 (1056), so every warp starts on its
# own item and the many short last splits (tail block among the first tiles a warp streams) sit inside the window of
# cache reads before the grid-dependency wait
CHAIN_LENGTHS = [1, 2, 17, 31, 32, 33, 40, 63, 64, 65, 96, 100, 127, 128, 129, 150, 161, 200, 255, 256, 257, 289, 300,
                 400, 513, 600, 1000, 1025, 1300, 1537, 2049, 2100]


@pytest.mark.parametrize("writer", [0, 1], ids=["rope_kvwrite", "gemm_fused_rope"])
def test_cache_write_then_attention_on_one_stream(g, writer, monkeypatch):
    """The engine's decode layer step (Llama-3-8B heads, 32 sequences): the step's K / V rows are written into the cache
    (by rope_kvwrite, or by the qkv GEMM's fused RoPE + scatter epilogue, the production decode path) and attention
    follows on the same stream with no synchronisation.  The decode kernel streams cache blocks of earlier steps before
    its grid-dependency wait; the newest slot starts as poison, so a read of it before the writer is done shows.  The
    result must meet the float64 bar over the written cache, and equal bit for bit the run without pre-wait reads
    (TGIS_ATTN_PREFETCH=0) and the unchained writer-then-attention calls."""
    n_q, n_kv, K = 32, 8, 4096
    G, T = n_q // n_kv, len(CHAIN_LENGTHS)
    slots = DEC_CTAS_PER_SM * DEC_WARPS * torch.cuda.get_device_properties(0).multi_processor_count
    if sum((n + 127) // 128 for n in CHAIN_LENGTHS) * n_kv > slots:
        pytest.skip("fewer decode warp slots than items on this device: the short tails would not start a warp")
    lib = g.lib()
    gen = torch.Generator(device="cuda").manual_seed(17 + writer)
    x = torch.zeros(256, K, dtype=torch.bfloat16, device="cuda")
    x[:T] = (torch.randn(T, K, generator=gen, device="cuda") * 0.5).bfloat16()
    w = (torch.randn((n_q + 2 * n_kv) * 128, K, generator=gen, device="cuda") * 0.05).bfloat16()
    qkv0 = (torch.randn(T, n_q + 2 * n_kv, 128, generator=gen, device="cuda") * 1.5).bfloat16()
    table = (torch.rand(8192, 128, generator=gen, device="cuda") * 2 - 1).bfloat16()
    positions = np.array([n - 1 for n in CHAIN_LENGTHS], dtype=np.int32)
    nbs = [(n + 31) // 32 for n in CHAIN_LENGTHS]
    n_blocks, bt_stride = sum(nbs), max(nbs)
    order = np.random.RandomState(3).permutation(n_blocks).astype(np.int32)
    bt = np.zeros((T, bt_stride), dtype=np.int32)
    seqs = np.zeros((T, 4), dtype=np.int32)
    cur = 0
    for s, nb in enumerate(nbs):
        bt[s, :nb] = order[cur: cur + nb]
        cur += nb
        seqs[s] = (s, 1, CHAIN_LENGTHS[s], s)
    slot_map = np.array([bt[s, p // 32] * 32 + p % 32 for s, p in enumerate(positions)], dtype=np.int32)

    def write_alone(qkv, kc, vc):
        if writer == 0:
            qkv.copy_(qkv0)
            rc = lib.tgis_k_rope_kv(g.ptr(qkv), g.i32p(positions), g.i32p(slot_map), g.ptr(table), g.ptr(kc), g.ptr(vc),
                                    T, n_q, n_kv)
        else:
            rc = lib.tgis_k_gemm_rope(g.ptr(x), g.ptr(w), g.ptr(qkv), T, n_q, n_kv, K, 256, g.i32p(positions),
                                      g.i32p(slot_map), g.ptr(table), g.ptr(kc), g.ptr(vc))
            if rc == 1:
                pytest.skip("the launch plan does not split every qkv weight tile on this device: no fused epilogue")
        assert rc == 0, g.kerr()

    # the roped queries come out of the writer: run it once to aim the poison at them
    qkv_r = torch.zeros_like(qkv0)
    scratch = torch.zeros(n_blocks * 32, n_kv, 128, dtype=torch.bfloat16, device="cuda")
    write_alone(qkv_r, g.k_cache_from_dense(scratch, n_blocks), g.v_cache_from_dense(scratch, n_blocks))
    q_sign = torch.sign(qkv_r[:, :n_q].float().view(T, n_kv, G, 128).sum(2))  # [T, n_kv, 128]
    k_pool = (torch.randn(n_blocks * 32, n_kv, 128, generator=gen, device="cuda") * 1.5).bfloat16()
    v_pool = torch.randn(n_blocks * 32, n_kv, 128, generator=gen, device="cuda").bfloat16()
    for s, n in enumerate(CHAIN_LENGTHS):  # the newest slot and the unused rest of its block: aligned keys, large values
        tail = torch.arange(n - 1, nbs[s] * 32, device="cuda")
        sl = torch.from_numpy(bt[s]).cuda()[tail // 32] * 32 + tail % 32
        k_pool[sl] = (POISON_K * q_sign[s]).bfloat16()
        v_pool[sl] = POISON_V
    kc0, vc0 = g.k_cache_from_dense(k_pool, n_blocks), g.v_cache_from_dense(v_pool, n_blocks)

    def chained():
        qkv, kc, vc = qkv0.clone(), kc0.clone(), vc0.clone()
        out = torch.zeros(T, n_q, 128, dtype=torch.bfloat16, device="cuda")
        rc = lib.tgis_k_rope_attention(writer, g.ptr(x), g.ptr(w), K, 256, g.ptr(qkv), g.i32p(positions),
                                       g.i32p(slot_map), g.ptr(table), g.ptr(kc), g.ptr(vc), g.i32p(seqs.reshape(-1)), T,
                                       g.i32p(bt.reshape(-1)), T, bt_stride, g.ptr(out), n_q, n_kv, SCALE)
        assert rc == 0, g.kerr()
        return out, qkv, kc, vc

    monkeypatch.setenv("TGIS_ATTN_PREFETCH", "1")
    out, qkv, kc, vc = chained()
    monkeypatch.setenv("TGIS_ATTN_PREFETCH", "0")
    out_nopre, *_ = chained()
    monkeypatch.delenv("TGIS_ATTN_PREFETCH")
    qkv_u, kc_u, vc_u = qkv0.clone(), kc0.clone(), vc0.clone()
    write_alone(qkv_u, kc_u, vc_u)
    out_u = torch.zeros(T, n_q, 128, dtype=torch.bfloat16, device="cuda")
    assert lib.tgis_k_attention(g.ptr(qkv_u), g.ptr(kc_u), g.ptr(vc_u), g.i32p(seqs.reshape(-1)), T,
                                g.i32p(bt.reshape(-1)), T, bt_stride, g.ptr(out_u), n_q, n_kv, SCALE) == 0, g.kerr()
    # the chained writer wrote what the stand-alone one writes, over the poison
    assert torch.equal(qkv, qkv_u) and torch.equal(kc, kc_u) and torch.equal(vc, vc_u)
    k_dense, v_dense = g.dense_from_k_cache(kc), g.dense_from_v_cache(vc)
    assert not bool((v_dense[torch.from_numpy(slot_map).long().cuda()] == POISON_V).any())
    ref = torch.empty(T, n_q, 128, dtype=torch.float64, device="cuda")
    for s, n in enumerate(CHAIN_LENGTHS):
        pos = torch.arange(n, device="cuda")
        sl = torch.from_numpy(bt[s]).cuda()[pos // 32] * 32 + pos % 32
        ref[s: s + 1] = g.attention_reference_f64(qkv[s: s + 1, :n_q], k_dense[sl], v_dense[sl], n - 1, SCALE)
    _assert_bar(g, out, ref, None, f"write + attention chain (writer {writer})")  # decode rows only: no floor factor
    assert torch.equal(out, out_nopre), "cache reads before the grid-dependency wait changed the result"
    assert torch.equal(out, out_u), "the chained step differs from the unchained calls"
