"""-m gpu parity tests, one per hot-path kernel: CUDA (through the C ABI) vs the CPU oracle on the same seeded inputs.

Tolerances (written here, per the task contract):
  * integer / index results (greedy token ids, ranks, top-n ids, KV-cache placement, RoPE bits): bit-exact
  * bf16 tensor results whose fp32 accumulation ORDER differs from the oracle's (GEMM): <= 1 bf16 ulp per element
  * RMSNorm and SiLU * mul: bit-exact (RMSNorm against tgis_gpu_utils.rmsnorm_restated, its summation order)
  * attention (both kernels feed P to the tensor cores as bf16 hi + lo): against a float64 softmax from the same bf16
    inputs, <= 1 bf16 ulp per element or <= 2^-16 of the row's largest output, and >= 99 % bit-exact
    (tgis_gpu_utils.attention_bar; tests/test_attention_precision_gpu.py runs the same bar at serving shapes)
  * logprobs: 1e-3 absolute (BASELINE.json north_star)
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def g():
    import tgis_gpu_utils as gpu_utils

    assert torch.cuda.is_available()
    torch.backends.cuda.matmul.allow_tf32 = False
    return gpu_utils


GEMM_SHAPES = [
    (1, 128, 64), (7, 256, 512), (16, 384, 4096), (32, 6144, 4096), (33, 1000, 520), (64, 4096, 14336),
    (100, 2048, 1024), (128, 1024, 4096), (200, 512, 256), (256, 28672, 4096), (300, 768, 512), (1024, 2048, 1024),
    (32, 128256, 4096), (4, 1024, 256),
]


@pytest.mark.parametrize("T,N,K", GEMM_SHAPES)
def test_gemm_tcgen05_matches_fp32_reference(g, T, N, K):
    gen = torch.Generator(device="cuda").manual_seed(T * 7 + N + K)
    x = (torch.randn(T, K, generator=gen, device="cuda") * 0.5).bfloat16()
    w = (torch.randn(N, K, generator=gen, device="cuda") * 0.05).bfloat16()
    y, _ = g.gemm(x, w)
    ref = x.float() @ w.float().t()
    ulp = g.bf16_ulp_diff(y, ref.bfloat16())
    # fp32 accumulation order differs from cuBLAS': a result sitting on a rounding boundary may land 1 ulp away
    bad = (ulp > 1.01) & ((y.float() - ref).abs() > 1e-3 * ref.abs().mean())
    assert int(bad.sum()) == 0, f"max ulp {float(ulp.max())} bad={int(bad.sum())}"
    frac_exact = float((ulp == 0).float().mean())
    assert frac_exact > 0.97, frac_exact
    # bit-deterministic across launches (stream-K fix-up sums in fixed CTA order)
    y2, _ = g.gemm(x, w)
    assert torch.equal(y, y2)


def test_gemm_fp32_output_for_logits(g):
    """lm_head path: the epilogue stores the fp32 accumulator (no bf16 round trip)."""
    gen = torch.Generator(device="cuda").manual_seed(1)
    x = (torch.randn(24, 512, generator=gen, device="cuda")).bfloat16()
    w = (torch.randn(5000, 512, generator=gen, device="cuda") * 0.02).bfloat16()
    y, _ = g.gemm(x, w, out_f32=True)
    ref = x.float() @ w.float().t()
    assert float((y - ref).abs().max()) < 2e-5 * float(ref.abs().max()) + 1e-5


@pytest.mark.parametrize("T,F,K", [(32, 1536, 512), (7, 14336, 4096), (300, 1024, 256)])
def test_gemm_fused_swiglu_epilogue(g, T, F, K):
    """gate_up GEMM with SwiGLU fused in the epilogue (rows interleaved gate_j, up_j) == GEMM -> bf16 -> silu*mul."""
    gen = torch.Generator(device="cuda").manual_seed(T + F)
    x = (torch.randn(T, K, generator=gen, device="cuda") * 0.5).bfloat16()
    wg = (torch.randn(F, K, generator=gen, device="cuda") * 0.05).bfloat16()
    wu = (torch.randn(F, K, generator=gen, device="cuda") * 0.05).bfloat16()
    w = torch.stack([wg, wu], dim=1).reshape(2 * F, K).contiguous()   # row 2j = gate_j, row 2j+1 = up_j
    act, _ = g.gemm(x, w, swiglu=True)
    gate = (x.float() @ wg.float().t()).bfloat16()
    up = (x.float() @ wu.float().t()).bfloat16()
    ref = torch.nn.functional.silu(gate) * up
    ulp = g.bf16_ulp_diff(act, ref)
    # A gate/up accumulator that lands within fp32 summation noise of a bf16 rounding midpoint may round the other way
    # than torch's (different summation order): that 1-ulp flip of the INTERMEDIATE moves the output by up to ~4 ulp.
    # So: nothing beyond 6 ulp (above an absolute floor), and at most 1e-4 of the elements beyond 2 ulp.
    floor = (act.float() - ref.float()).abs() > 2e-3 * ref.float().abs().mean()
    bad = (ulp > 6.01) & floor
    if int(bad.sum()):
        idx = torch.nonzero(bad)[:5]
        info = [(int(t), int(j), float(act[t, j]), float(ref[t, j]), float(gate[t, j]), float(up[t, j]),
                 float((x[t].float() @ wg[j].float())), float((x[t].float() @ wu[j].float()))) for t, j in idx]
        raise AssertionError(f"max ulp {float(ulp.max())}; (t, j, act, ref, gate_bf16, up_bf16, gate_f32, up_f32): {info}")
    assert float(((ulp > 2.01) & floor).float().mean()) < 1e-4
    assert float((ulp == 0).float().mean()) > 0.95
    act2, _ = g.gemm(x, w, swiglu=True)
    assert torch.equal(act, act2)
    actr, _ = g.gemm(x, w, impl=1, swiglu=True)   # SIMT cross-check kernel, same fusion
    d2 = g.bf16_ulp_diff(act, actr) * ((act.float() - actr.float()).abs() > 2e-3 * ref.float().abs().mean())
    assert float(d2.max()) <= 6.0 and float((d2 > 2.01).float().mean()) < 1e-4


def test_gemm_crosscheck_kernel_agrees(g):
    gen = torch.Generator(device="cuda").manual_seed(7)
    x = (torch.randn(48, 1024, generator=gen, device="cuda") * 0.5).bfloat16()
    w = (torch.randn(640, 1024, generator=gen, device="cuda") * 0.05).bfloat16()
    y, _ = g.gemm(x, w, impl=0)
    yr, _ = g.gemm(x, w, impl=1)
    # both kernels accumulate in fp32 in different orders: <= 1 bf16 ulp, except where the result is a near-total
    # cancellation (|y| tiny relative to the summands), where 1 ulp of the OUTPUT is far below fp32 summation noise
    diff = (y.float() - yr.float()).abs()
    assert float((g.bf16_ulp_diff(y, yr) * (diff > 2e-4)).max()) <= 1.0


@pytest.mark.parametrize("T,H", [(1, 256), (5, 768), (32, 4096), (17, 8192)])
def test_rmsnorm_and_fused_add(g, T, H):
    torch.manual_seed(T + H)
    x = torch.randn(T, H).bfloat16().cuda()
    r = torch.randn(T, H).bfloat16().cuda()
    w = (1 + 0.1 * torch.randn(H)).bfloat16().cuda()
    eps = 1e-5
    out = torch.empty(T, H, dtype=torch.bfloat16, device="cuda")
    assert g.lib().tgis_k_rmsnorm(g.ptr(x), None, g.ptr(w), g.ptr(out), T, H, eps) == 0, g.kerr()
    assert torch.equal(out, g.rmsnorm_restated(x, w, eps)[0])
    rc = r.clone()
    assert g.lib().tgis_k_rmsnorm(g.ptr(x), g.ptr(rc), g.ptr(w), g.ptr(out), T, H, eps) == 0, g.kerr()
    want, z = g.rmsnorm_restated(x, w, eps, residual=r)
    assert torch.equal(z, x + r)  # bf16 add = fp32 add rounded to bf16 (vllm layernorm_kernels.cu: add in scalar_t)
    assert torch.equal(rc, z)
    assert torch.equal(out, want)


def test_silu_mul(g):
    """bf16(bf16(silu(gate)) * up), the rounding points of bf16 torch ops (vllm activation_kernels.cu)"""
    torch.manual_seed(3)
    T, F = 9, 1536
    gu = (torch.randn(T, 2 * F) * 2).bfloat16()
    ref = torch.nn.functional.silu(gu[:, :F]) * gu[:, F:]
    act = torch.empty(T, F, dtype=torch.bfloat16, device="cuda")
    guc = gu.cuda()
    assert g.lib().tgis_k_silu_mul(g.ptr(guc), g.ptr(act), T, F) == 0, g.kerr()
    assert torch.equal(act.cpu(), ref), int((act.cpu() != ref).sum())


def test_rope_and_kv_scatter_bit_exact(g):
    from oracle.llama_oracle import LlamaConfig, LlamaOracle, rope_table

    cfg = LlamaConfig(n_layers=1, hidden=256, n_q_heads=4, n_kv_heads=2, ffn=256, vocab=64, max_model_len=256)
    table = rope_table(cfg)
    torch.manual_seed(5)
    T = 37
    n_heads = cfg.n_q_heads + 2 * cfg.n_kv_heads
    qkv = torch.randn(T, n_heads, 128).bfloat16()
    positions = np.arange(3, 3 + T, dtype=np.int32)
    n_blocks = 6
    perm = np.random.RandomState(0).permutation(n_blocks * 32)[:T].astype(np.int32)  # arbitrary distinct slots
    kc = torch.zeros(n_blocks, cfg.n_kv_heads, 16, 32, 8, dtype=torch.bfloat16, device="cuda")
    vc = torch.zeros(n_blocks, cfg.n_kv_heads, 32, 16, 8, dtype=torch.bfloat16, device="cuda")
    qkv_c = qkv.cuda().clone()
    tab_c = table.cuda()
    rc = g.lib().tgis_k_rope_kv(g.ptr(qkv_c), g.i32p(positions), g.i32p(perm), g.ptr(tab_c), g.ptr(kc), g.ptr(vc), T,
                                cfg.n_q_heads, cfg.n_kv_heads)
    assert rc == 0, g.kerr()
    # oracle: every product / sum rounded to bf16 (HF apply_rotary_pos_emb on bf16 tensors)
    half = 64
    cs = table[torch.from_numpy(positions).long()]
    cos, sin = cs[:, None, :half], cs[:, None, half:]
    qk = qkv[:, : cfg.n_q_heads + cfg.n_kv_heads]
    x1, x2 = qk[..., :half], qk[..., half:]
    rot = torch.cat([x1 * cos - x2 * sin, x2 * cos + x1 * sin], dim=-1)
    got = qkv_c.cpu()
    assert torch.equal(got[:, : cfg.n_q_heads + cfg.n_kv_heads], rot)
    assert torch.equal(got[:, cfg.n_q_heads + cfg.n_kv_heads:], qkv[:, cfg.n_q_heads + cfg.n_kv_heads:])
    k_dense = g.dense_from_k_cache(kc).cpu()
    v_dense = g.dense_from_v_cache(vc).cpu()
    slots = torch.from_numpy(perm).long()
    assert torch.equal(k_dense[slots], rot[:, cfg.n_q_heads:])
    assert torch.equal(v_dense[slots], qkv[:, cfg.n_q_heads + cfg.n_kv_heads:])


@pytest.mark.parametrize("heads", [(24, 4), (32, 8)])
@pytest.mark.parametrize("T", [32, 200])
def test_qkv_gemm_with_fused_rope_epilogue_is_bit_identical(g, T, heads):
    """The qkv projection's split-tile reduction (gemm_wgmma.cu) followed in the same kernel by RoPE + scatter into the
    paged K / V layouts, against the unfused pair (GEMM -> bf16 qkv, then rope_kvwrite_kernel): qkv rows and both caches
    must be bit-identical.  32 heads = 32 weight tiles, 48 heads (the Llama-3-8B shape) = 48 tiles, each split over a
    cluster (reduction through distributed shared memory) or, where the clusters do not all fit the GPU at once, through
    the global-memory fix-up.  T = 200 (one 256-token tile over 16 k-blocks) is not split: the test skips there."""
    import ctypes as C

    (n_q, n_kv), K = heads, 1024
    n_heads = n_q + 2 * n_kv
    N = n_heads * 128
    torch.manual_seed(21)
    rows = 256
    x = torch.zeros(rows, K, dtype=torch.bfloat16, device="cuda")
    x[:T] = (torch.randn(T, K, device="cuda") * 0.5).bfloat16()
    w = (torch.randn(N, K, device="cuda") * 0.05).bfloat16()
    table = (torch.rand(512, 128, device="cuda") * 2 - 1).bfloat16()       # any cos | sin table: same one for both paths
    positions = np.random.RandomState(1).randint(0, 512, size=T).astype(np.int32)
    n_blocks = 16
    slots = np.random.RandomState(2).permutation(n_blocks * 32)[:T].astype(np.int32)
    slots[3] = -1                                                            # "do not cache" row
    kc1 = torch.zeros(n_blocks, n_kv, 16, 32, 8, dtype=torch.bfloat16, device="cuda")
    vc1 = torch.zeros_like(kc1)
    kc2, vc2 = torch.zeros_like(kc1), torch.zeros_like(kc1)
    y1 = torch.zeros(T, N, dtype=torch.bfloat16, device="cuda")
    rc = g.lib().tgis_k_gemm_rope(g.ptr(x), g.ptr(w), g.ptr(y1), T, n_q, n_kv, K, rows, g.i32p(positions), g.i32p(slots),
                                  g.ptr(table), g.ptr(kc1), g.ptr(vc1))
    assert rc in (0, 1), g.kerr()
    if rc == 1:
        pytest.skip("the launch plan does not split every tile on this device")
    y2 = torch.zeros(T, N, dtype=torch.bfloat16, device="cuda")
    ms = C.c_float(0)
    assert g.lib().tgis_k_gemm(g.ptr(x), g.ptr(w), g.ptr(y2), T, N, K, rows, 0, 1, C.byref(ms), 0) == 0, g.kerr()
    assert g.lib().tgis_k_rope_kv(g.ptr(y2), g.i32p(positions), g.i32p(slots), g.ptr(table), g.ptr(kc2), g.ptr(vc2), T,
                                  n_q, n_kv) == 0, g.kerr()
    assert torch.equal(y1, y2)
    assert torch.equal(kc1, kc2) and torch.equal(vc1, vc2)
    assert float(kc1.float().abs().sum()) > 0 and float(vc1.float().abs().sum()) > 0


def _attention_case(g, n_q, n_kv, seq_specs, seed):
    """seq_specs: list of (context_len_before, q_len).  Returns (out_gpu, float64 reference) on the CPU."""
    gen = torch.Generator().manual_seed(seed)
    T = sum(q for _, q in seq_specs)
    q_all = torch.randn(T, n_q, 128, generator=gen).bfloat16()
    qkv = torch.zeros(T, n_q + 2 * n_kv, 128, dtype=torch.bfloat16)
    qkv[:, :n_q] = q_all
    bt_stride = max((c + q + 31) // 32 for c, q in seq_specs)
    n_blocks = sum((c + q + 31) // 32 for c, q in seq_specs)
    order = np.random.RandomState(seed).permutation(n_blocks)  # scattered physical blocks
    k_dense = torch.zeros(n_blocks * 32, n_kv, 128, dtype=torch.bfloat16)
    v_dense = torch.zeros(n_blocks * 32, n_kv, 128, dtype=torch.bfloat16)
    bt = np.zeros((len(seq_specs), bt_stride), dtype=np.int32)
    seqs = np.zeros((len(seq_specs), 4), dtype=np.int32)
    ref = torch.zeros(T, n_q, 128, dtype=torch.float64)
    blk_cursor, q_start = 0, 0
    for s, (ctx, ql) in enumerate(seq_specs):
        kv_len = ctx + ql
        nb = (kv_len + 31) // 32
        blocks = order[blk_cursor: blk_cursor + nb]
        blk_cursor += nb
        bt[s, :nb] = blocks
        k = (torch.randn(kv_len, n_kv, 128, generator=gen) * 1.5).bfloat16()
        v = torch.randn(kv_len, n_kv, 128, generator=gen).bfloat16()
        for j in range(kv_len):
            slot = int(blocks[j // 32]) * 32 + j % 32
            k_dense[slot], v_dense[slot] = k[j], v[j]
        seqs[s] = (q_start, ql, kv_len, s)
        ref[q_start: q_start + ql] = g.attention_reference_f64(q_all[q_start: q_start + ql], k, v, ctx,
                                                               1.0 / math.sqrt(128))
        q_start += ql
    kc = g.k_cache_from_dense(k_dense.cuda(), n_blocks)
    vc = g.v_cache_from_dense(v_dense.cuda(), n_blocks)
    out = torch.zeros(T, n_q, 128, dtype=torch.bfloat16, device="cuda")
    qkv_c = qkv.cuda()
    rc = g.lib().tgis_k_attention(g.ptr(qkv_c), g.ptr(kc), g.ptr(vc), g.i32p(seqs.reshape(-1)), len(seq_specs),
                                  g.i32p(bt.reshape(-1)), len(seq_specs), bt_stride, g.ptr(out), n_q, n_kv,
                                  1.0 / math.sqrt(128))
    assert rc == 0, g.kerr()
    return out.cpu(), ref


@pytest.mark.parametrize("n_q,n_kv", [(4, 2), (8, 2), (6, 2), (8, 1), (2, 2)])
def test_attention_decode_split_kv(g, n_q, n_kv):
    specs = [(c, 1) for c in (0, 1, 30, 31, 32, 127, 128, 129, 255, 300, 575, 1000)]
    out, ref = _attention_case(g, n_q, n_kv, specs, seed=n_q * 10 + n_kv)
    n_bad, exact, worst = g.attention_bar(out, ref)
    assert n_bad == 0, worst
    assert exact >= 0.99, exact


@pytest.mark.parametrize("n_q,n_kv", [(4, 2), (8, 2), (6, 2), (8, 1)])
def test_attention_prefill_and_mixed(g, n_q, n_kv):
    specs = [(0, 5), (0, 16), (0, 17), (0, 50), (40, 33), (0, 1), (100, 1), (31, 70), (0, 129), (200, 2)]
    out, ref = _attention_case(g, n_q, n_kv, specs, seed=n_q * 100 + n_kv)
    n_bad, exact, worst = g.attention_bar(out, ref)
    assert n_bad == 0, worst
    assert exact >= 0.99, exact


# ----------------------------------------------------------------------------------------------------- sampler
def _rows(g, n):
    r = np.zeros(n, dtype=g.SAMPLE_ROW_DTYPE)
    r["temperature"], r["top_p"], r["rep_penalty"] = 1.0, 1.0, 1.0
    r["eos_id"], r["seq_slot"] = 2, -1
    r["logits_row"] = np.arange(n)
    return r


@pytest.mark.parametrize("V", [1024, 128256])
def test_sampler_greedy_logprobs_rank_topn(g, V):
    from oracle.sampler_oracle import SamplingCase, sample_row

    torch.manual_seed(V)
    n = 6
    logits = torch.randn(n, V) * 2
    logits[1, 77] = logits[1].max() + 1  # clear winner
    logits[2, 500] = logits[2, 9] = logits[2].max() + 0.5  # exact tie -> lowest index wins
    rows = _rows(g, n)
    rows["flags"] = g.SAMPLE_GREEDY | g.SAMPLE_LOGPROBS
    rows["n_topn"] = [1, 3, 5, 11, 2, 1]
    out = g.run_sampler(logits.cuda(), rows)
    for i in range(n):
        o = sample_row(logits[i].float(), SamplingCase(greedy=True, num_logprobs=int(rows["n_topn"][i])))
        assert out["token"][i] == o["token"]
        assert abs(out["logprob"][i] - o["logprob"]) < 1e-3
        assert out["rank"][i] == o["rank"]
        k = int(rows["n_topn"][i])
        assert out["n_topn"][i] == k
        np.testing.assert_allclose(out["topn_lps"][i][:k], o["topn_logprobs"], atol=1e-3)
        # ids must agree wherever the logprobs are not tied
        for j in range(k):
            if out["topn_ids"][i][j] != o["topn_ids"][j]:
                assert abs(out["topn_lps"][i][j] - o["topn_logprobs"][j]) < 1e-6
    assert out["token"][2] == 9


def test_sampler_greedy_processors_exact(g):
    """ExpDecay + min_tokens + repetition penalty on greedy rows (reference logits_processors.py:33-47)."""
    from oracle.sampler_oracle import SamplingCase, len_penalty_factor_m1, sample_row

    V, n = 4096, 8
    torch.manual_seed(11)
    logits = torch.randn(n, V) * 1.5
    eos = 2
    words = (V + 31) // 32
    bm = np.zeros((n, words), dtype=np.uint32)
    seen = torch.zeros(n, V, dtype=torch.bool)
    rows = _rows(g, n)
    rows["flags"] = g.SAMPLE_GREEDY | g.SAMPLE_LOGPROBS
    rows["n_topn"] = 1
    rows["eos_id"] = eos
    rows["seq_slot"] = np.arange(n)
    cases = []
    for i in range(n):
        top = torch.topk(logits[i].float(), 4).indices
        # make EOS competitive so the length penalty decides; penalise the raw argmax via repetition penalty
        logits[i, eos] = logits[i, top[1]]
        case = SamplingCase(greedy=True, num_logprobs=1, eos_token_id=eos)
        if i % 2 == 0:
            case.length_penalty = (2, 1.5)
            case.n_out = 2 + i
        if i in (1, 2, 5):
            case.repetition_penalty = 1.7
            seen[i, top[0]] = True
            seen[i, 5] = True
        if i in (3, 4):
            case.min_tokens, case.n_out = 10, (4 if i == 3 else case.n_out)
        cases.append(case)
        rows["rep_penalty"][i] = case.repetition_penalty
        rows["n_out"][i], rows["min_tokens"][i] = case.n_out, case.min_tokens
        if case.length_penalty:
            f = len_penalty_factor_m1(case.n_out, *case.length_penalty)
            if f != 0.0:
                rows["flags"][i] |= g.SAMPLE_LENPEN
                rows["len_decay_factor"][i] = f
        for t in torch.nonzero(seen[i]).flatten().tolist():
            bm[i, t // 32] |= np.uint32(1) << np.uint32(t % 32)
    bitmap = torch.from_numpy(bm.view(np.int32))
    out = g.run_sampler(logits.cuda(), rows, bitmap.cuda())
    for i in range(n):
        o = sample_row(logits[i].float(), cases[i], seen[i])
        assert out["token"][i] == o["token"], (i, out["token"][i], o["token"])
        assert abs(out["logprob"][i] - o["logprob"]) < 1e-3
        assert out["rank"][i] == o["rank"]


@pytest.mark.parametrize("V", [2048, 128256])
def test_sampler_random_sampling_paths(g, V):
    """typical-p / top-k / top-p / temperature: the sampled token must lie in the oracle's allowed set and (own
    counter-based RNG restated in numpy) equal the oracle's draw."""
    from oracle.sampler_oracle import SamplingCase, sample_row

    torch.manual_seed(V + 1)
    cases = [
        SamplingCase(greedy=False, temperature=0.7, seed=1),
        SamplingCase(greedy=False, temperature=1.0, top_k=50, seed=2),
        SamplingCase(greedy=False, temperature=1.3, top_p=0.8, seed=3),
        SamplingCase(greedy=False, temperature=0.9, top_k=200, top_p=0.5, seed=4),
        SamplingCase(greedy=False, temperature=1.0, typical_p=0.9, seed=5),
        SamplingCase(greedy=False, temperature=1.0, typical_p=0.2, top_k=40, seed=6),
        SamplingCase(greedy=False, temperature=1.0, typical_p=0.9, repetition_penalty=1.2, length_penalty=(64, 1.05),
                     n_out=100, min_tokens=128, seed=1234 << 20),
        SamplingCase(greedy=False, temperature=2.0, top_p=0.05, seed=8),
    ]
    n = len(cases)
    logits = torch.randn(n, V) * 3
    from oracle.sampler_oracle import len_penalty_factor_m1

    rows = _rows(g, n)
    words = (V + 31) // 32
    bitmap = torch.zeros(n, words, dtype=torch.int32)
    seen = torch.zeros(n, V, dtype=torch.bool)
    seen[:, 10:20] = True
    bitmap[:, 0] = sum(1 << b for b in range(10, 20))
    for i, c in enumerate(cases):
        c.num_logprobs = 2
        rows["flags"][i] = g.SAMPLE_LOGPROBS | (g.SAMPLE_TYPICAL if 0 < c.typical_p < 1 else 0)
        rows["n_topn"][i] = 2
        rows["temperature"][i], rows["top_k"][i], rows["top_p"][i] = c.temperature, c.top_k, c.top_p
        rows["typical_p"][i], rows["rep_penalty"][i] = c.typical_p, c.repetition_penalty
        rows["n_out"][i], rows["min_tokens"][i], rows["step"][i] = c.n_out, c.min_tokens, c.n_out
        rows["seed_lo"][i], rows["seed_hi"][i] = c.seed & 0xFFFFFFFF, c.seed >> 32
        rows["seq_slot"][i] = i
        if c.length_penalty:
            f = len_penalty_factor_m1(c.n_out, *c.length_penalty)
            if f != 0.0:
                rows["flags"][i] |= g.SAMPLE_LENPEN
                rows["len_decay_factor"][i] = f
    out = g.run_sampler(logits.cuda(), rows, bitmap.cuda())
    same = 0
    for i, c in enumerate(cases):
        o = sample_row(logits[i].float(), c, seen[i])
        tok = int(out["token"][i])
        assert bool(o["allowed"][tok]), (i, tok)
        same += int(tok == o["token"])
        lp = torch.log_softmax(logits[i].float(), -1)
        assert abs(out["logprob"][i] - float(lp[tok])) < 1e-3
        assert out["rank"][i] == int((lp >= lp[tok]).sum())
    assert same >= n - 1, same


def test_sampler_distribution_matches_softmax(g):
    """Exponential-race sampling (vllm topk_topp_sampler.py:395-416) is distributional: chi-square on 20k draws."""
    V, n = 64, 20000
    torch.manual_seed(0)
    base = torch.randn(V) * 1.5
    logits = base[None, :].repeat(n, 1).contiguous()
    rows = _rows(g, n)
    rows["seed_lo"] = np.arange(n) * 2654435761 % (1 << 32)
    rows["seed_hi"] = 7
    out = g.run_sampler(logits.cuda(), rows)
    p = torch.softmax(base.float(), -1).numpy()
    counts = np.bincount(out["token"], minlength=V)
    exp = p * n
    chi2 = float(((counts - exp) ** 2 / np.maximum(exp, 1e-9)).sum())
    assert chi2 < 120.0, chi2  # 63 dof: P(chi2 > 120) ~ 2e-5


@pytest.mark.parametrize("V", [1024, 128256])
def test_sampler_bf16_logits_ties_rank_and_argmax(g, V):
    """The product path's logits are bf16 (vLLM's lm_head output dtype): thousands of EXACT ties per row.  Greedy must
    pick the lowest id among equal maxima (torch.argmax), rank counts every tied entry (vllm ops/logprobs.py:27),
    logprobs come from the fp32 view of the bf16 values -- all index-exact against the oracle on the same bf16 row."""
    from oracle.sampler_oracle import SamplingCase, sample_row

    torch.manual_seed(V + 7)
    n = 6
    logits = (torch.randn(n, V) * 2).to(torch.bfloat16)
    mx = logits[2].float().max()
    logits[2, 700] = logits[2, 31] = logits[2, 900] = (mx + 0.5).to(torch.bfloat16)   # three-way tie at the top
    rows = _rows(g, n)
    rows["flags"] = g.SAMPLE_GREEDY | g.SAMPLE_LOGPROBS
    rows["n_topn"] = [1, 3, 5, 11, 2, 1]
    out = g.run_sampler(logits.cuda(), rows)
    ties = 0
    for i in range(n):
        o = sample_row(logits[i].float(), SamplingCase(greedy=True, num_logprobs=int(rows["n_topn"][i])))
        assert out["token"][i] == o["token"]
        assert abs(out["logprob"][i] - o["logprob"]) < 1e-4
        assert out["rank"][i] == o["rank"]
        ties += int(o["rank"] > 1)
        k = int(rows["n_topn"][i])
        np.testing.assert_allclose(out["topn_lps"][i][:k], o["topn_logprobs"], atol=1e-4)
        for j in range(k):   # ids agree wherever the values are not tied; tied values are listed lowest id first
            if out["topn_ids"][i][j] != o["topn_ids"][j]:
                assert abs(out["topn_lps"][i][j] - o["topn_logprobs"][j]) < 1e-6   # 2 fp32 ulps at |lp| ~ 6
    assert out["token"][2] == 31 and out["rank"][2] == 3 and ties >= 1


def test_sampler_bf16_logits_sampling_paths_match_fp32_view(g):
    """bf16 logits through typical-p / penalties / top-k / top-p / race: bit-identical to running the same kernel on the
    fp32 copy of those bf16 values (the cast is exact), and equal to the oracle's draw."""
    from oracle.sampler_oracle import SamplingCase, len_penalty_factor_m1, sample_row

    V = 128256
    torch.manual_seed(5)
    cases = [SamplingCase(greedy=False, temperature=1.0, typical_p=0.9, repetition_penalty=1.2, length_penalty=(64, 1.05),
                          n_out=100, min_tokens=128, seed=1234, num_logprobs=2),
             SamplingCase(greedy=False, temperature=0.8, top_k=40, top_p=0.9, seed=99, num_logprobs=2),
             SamplingCase(greedy=True, length_penalty=(2, 1.5), n_out=9, num_logprobs=2)]
    n = len(cases)
    lb = (torch.randn(n, V) * 3).to(torch.bfloat16)
    rows = _rows(g, n)
    words = (V + 31) // 32
    bitmap = torch.zeros(n, words, dtype=torch.int32)
    seen = torch.zeros(n, V, dtype=torch.bool)
    seen[:, 10:20] = True
    bitmap[:, 0] = sum(1 << b for b in range(10, 20))
    for i, c in enumerate(cases):
        rows["flags"][i] = g.SAMPLE_LOGPROBS | (g.SAMPLE_TYPICAL if (0 < c.typical_p < 1 and not c.greedy) else 0) | \
            (g.SAMPLE_GREEDY if c.greedy else 0)
        rows["n_topn"][i] = 2
        rows["temperature"][i], rows["top_k"][i], rows["top_p"][i] = c.temperature, c.top_k, c.top_p
        rows["typical_p"][i], rows["rep_penalty"][i] = c.typical_p, c.repetition_penalty
        rows["n_out"][i], rows["min_tokens"][i], rows["step"][i] = c.n_out, c.min_tokens, c.n_out
        rows["seed_lo"][i], rows["seed_hi"][i] = c.seed & 0xFFFFFFFF, c.seed >> 32
        rows["seq_slot"][i] = i
        if c.length_penalty:
            f = len_penalty_factor_m1(c.n_out, *c.length_penalty)
            if f != 0.0:
                rows["flags"][i] |= g.SAMPLE_LENPEN
                rows["len_decay_factor"][i] = f
    a = g.run_sampler(lb.cuda(), rows, bitmap.cuda())
    b = g.run_sampler(lb.float().cuda(), rows, bitmap.clone().cuda())
    for f in ("token", "logprob", "rank", "n_topn"):
        assert np.array_equal(a[f], b[f]), f
    for f in ("topn_ids", "topn_lps"):      # entries beyond n_topn are not written
        assert np.array_equal(a[f][:, :2], b[f][:, :2]), f
    for i, c in enumerate(cases):
        o = sample_row(lb[i].float(), c, seen[i] if c.repetition_penalty != 1.0 else None)
        assert int(a["token"][i]) == o["token"] or bool(o["allowed"][int(a["token"][i])])
