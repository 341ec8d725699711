"""-m gpu: Granite (GraniteForCausalLM = the Llama stack + four config.json scalars) through the C ABI.

Kernels: the residual multiplier in the add + RMSNorm kernel and the embedding multiplier in the gather are bit-exact
restatements of bf16 torch ops; the sampler treats the columns of a padded vocabulary (ld = round_up(V, 8) > V) as
absent in every pass, and with a logit scale sees bf16(logit * s).  Engine: granite-tiny (V = 1021, tied embeddings,
scalars 12 / 0.22 / 1/128 / 1/3) against the oracle with the bands tests/test_engine_gpu.py uses for Llama.
"""
import dataclasses

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SAMPLE_FORCED = 32   # csrc/kernels.h: the token is given (prompt logprobs); report its logprob / rank / top-n


@pytest.fixture(scope="module")
def g():
    import tgis_gpu_utils as gpu_utils

    assert torch.cuda.is_available()
    return gpu_utils


# ----------------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("T", [1, 37, 2048])
@pytest.mark.parametrize("H", [256, 4096])
def test_residual_multiplier_norm_is_bit_exact(g, T, H):
    torch.manual_seed(T * 7 + H)
    m, eps = 0.22, 1e-5
    x = (torch.randn(T, H) * 3).to(torch.bfloat16).cuda()
    r0 = (torch.randn(T, H) * 5).to(torch.bfloat16).cuda()
    w = (1 + 0.1 * torch.randn(H)).to(torch.bfloat16).cuda()
    r, out = r0.clone(), torch.empty(T, H, dtype=torch.bfloat16, device="cuda")
    assert g.lib().tgis_k_rmsnorm_mult(g.ptr(x), g.ptr(r), g.ptr(w), g.ptr(out), T, H, eps, m) == 0, g.kerr()
    # residual: bf16(r + bf16(x * m)), two roundings (bf16 torch ops)
    assert torch.equal(r, r0 + x * m)
    # the norm that follows: rmsnorm_kernel's summation order and rounding points, bit for bit
    want, z = g.rmsnorm_restated(x, w, eps, residual=r0, mult=m)
    assert torch.equal(r, z) and torch.equal(out, want)
    # m = 1 is tgis_k_rmsnorm bit for bit
    r3, out3 = r0.clone(), torch.empty_like(out)
    r4, out4 = r0.clone(), torch.empty_like(out)
    assert g.lib().tgis_k_rmsnorm_mult(g.ptr(x), g.ptr(r3), g.ptr(w), g.ptr(out3), T, H, eps, 1.0) == 0, g.kerr()
    assert g.lib().tgis_k_rmsnorm(g.ptr(x), g.ptr(r4), g.ptr(w), g.ptr(out4), T, H, eps) == 0, g.kerr()
    assert torch.equal(r3, r4) and torch.equal(out3, out4)


@pytest.mark.parametrize("mult", [12.0, 1.0, 0.3])
def test_embedding_multiplier_gather_is_bit_exact(g, mult):
    torch.manual_seed(3)
    V, H, T = 1021, 4096, 77
    table = (torch.randn(V, H) * 0.02).to(torch.bfloat16).cuda()
    tok = torch.randint(0, V, (T,), dtype=torch.int32).cuda()
    out = torch.empty(T, H, dtype=torch.bfloat16, device="cuda")
    assert g.lib().tgis_k_embed(g.ptr(tok), g.ptr(table), g.ptr(out), T, H, V, mult) == 0, g.kerr()
    want = table[tok.long()] * mult if mult != 1.0 else table[tok.long()]
    assert torch.equal(out, want)


def _rows(g, n):
    r = np.zeros(n, dtype=g.SAMPLE_ROW_DTYPE)
    r["temperature"], r["top_p"], r["rep_penalty"] = 1.0, 1.0, 1.0
    r["eos_id"], r["seq_slot"] = 2, -1
    r["logits_row"] = np.arange(n)
    return r


def _padded(logits: torch.Tensor) -> torch.Tensor:
    """[n, V] -> bf16 [n, round_up(V, 8)] on the device; the padding columns hold the largest logit of the buffer + 8, so
    that any pass which read one as a vocabulary entry would return it or count it."""
    n, V = logits.shape
    Vp = (V + 7) // 8 * 8
    buf = torch.full((n, Vp), float(logits.max()) + 8, dtype=torch.bfloat16)
    buf[:, :V] = logits.to(torch.bfloat16)
    return buf.cuda()


def _cases(V):
    from oracle.sampler_oracle import SamplingCase

    return [
        SamplingCase(greedy=True),
        SamplingCase(greedy=False, temperature=0.7, seed=1),
        SamplingCase(greedy=False, temperature=1.0, top_k=50, seed=2),
        SamplingCase(greedy=False, temperature=1.3, top_p=0.8, seed=3),
        SamplingCase(greedy=False, temperature=0.9, top_k=V + 5, top_p=0.5, seed=4),
        SamplingCase(greedy=False, temperature=1.0, typical_p=0.9, seed=5),
        SamplingCase(greedy=False, temperature=1.0, top_k=V, seed=6),
        SamplingCase(greedy=True, typical_p=0.0, repetition_penalty=1.3),
    ]


def _fill_rows(g, rows, cases, V):
    for i, c in enumerate(cases):
        c.num_logprobs = 5
        rows["flags"][i] = g.SAMPLE_LOGPROBS | (g.SAMPLE_GREEDY if c.greedy else 0) | (
            g.SAMPLE_TYPICAL if 0 < c.typical_p < 1 else 0)
        rows["n_topn"][i] = 5
        rows["temperature"][i], rows["top_k"][i], rows["top_p"][i] = c.temperature, c.top_k, c.top_p
        rows["typical_p"][i], rows["rep_penalty"][i] = c.typical_p, c.repetition_penalty
        rows["seed_lo"][i], rows["seed_hi"][i] = c.seed & 0xFFFFFFFF, c.seed >> 32
        rows["seq_slot"][i] = i


def _sample(g, buf, V, rows, bitmap=None, allow=None):
    """the sampler on a padded bf16 buffer: ld = buf.stride(0) = round_up(V, 8), vocab = V"""
    out = np.zeros(len(rows), dtype=g.SAMPLE_OUT_DTYPE)
    rc = g.lib().tgis_k_sampler_masked(g.ptr(buf), 1, buf.stride(0), V, rows.ctypes.data_as(g.C.c_void_p), len(rows),
                                       g.ptr(bitmap) if bitmap is not None else None,
                                       g.ptr(allow) if allow is not None else None, out.ctypes.data_as(g.C.c_void_p), 1,
                                       None)
    assert rc == 0, g.kerr()
    return out


def _check(out, rows_f32, cases, seen, V):
    from oracle.sampler_oracle import sample_row

    same = 0
    for i, c in enumerate(cases):
        o = sample_row(rows_f32[i], c, seen[i])
        tok = int(out["token"][i])
        assert 0 <= tok < V, (i, tok)
        if o["allowed"] is not None:
            assert bool(o["allowed"][tok]), (i, tok)
        same += int(tok == o["token"])
        lp = torch.log_softmax(rows_f32[i], -1)
        assert abs(out["logprob"][i] - float(lp[tok])) < 1e-3
        assert out["rank"][i] == int((lp >= lp[tok]).sum()) and out["rank"][i] <= V
        ids = out["topn_ids"][i][:5]
        assert all(0 <= t < V for t in ids), ids
        top = torch.topk(lp, 5)
        np.testing.assert_allclose(out["topn_lps"][i][:5], top.values.numpy(), atol=1e-3)
    assert same >= len(cases) - 1, same


@pytest.mark.parametrize("V", [1021, 49155])
@pytest.mark.parametrize("cluster,smem", [("1", "1"), ("2", "1"), ("4", "1"), ("8", "1"), ("8", "0"), ("1", "0")])
def test_sampler_padded_vocabulary(g, monkeypatch, V, cluster, smem):
    monkeypatch.setenv("TGIS_SAMPLER_CLUSTER", cluster)
    monkeypatch.setenv("TGIS_SAMPLER_SMEM", smem)
    torch.manual_seed(V)
    cases = _cases(V)
    n = len(cases)
    logits = (torch.randn(n, V) * 3).to(torch.bfloat16).float()
    logits[0, V - 1] = logits[0].max() + 1            # greedy winner in the partial last 8-group
    buf = _padded(logits)
    assert buf.stride(0) % 8 == 0 and buf.stride(0) > V
    rows = _rows(g, n)
    _fill_rows(g, rows, cases, V)
    words = (V + 31) // 32
    bitmap = torch.zeros(n, words, dtype=torch.int32)
    seen = torch.zeros(n, V, dtype=torch.bool)
    seen[:, 10:20] = True
    bitmap[:, 0] = sum(1 << b for b in range(10, 20))
    out = _sample(g, buf, V, rows, bitmap.cuda())
    assert int(out["token"][0]) == V - 1
    _check(out, logits, cases, seen, V)


@pytest.mark.parametrize("V", [1021, 49155])
def test_sampler_padded_forced_rows_and_guided_last_group(g, V):
    from oracle.sampler_oracle import SamplingCase, sample_row

    torch.manual_seed(V + 1)
    n = 4
    logits = (torch.randn(n, V) * 2).to(torch.bfloat16).float()
    buf = _padded(logits)
    rows = _rows(g, n)
    # rows 0, 1: forced (prompt logprobs) on the last token and on token 0
    for i, t in ((0, V - 1), (1, 0)):
        rows["flags"][i] = SAMPLE_FORCED | g.SAMPLE_LOGPROBS
        rows["seed_lo"][i], rows["n_topn"][i] = t, 4
    # rows 2, 3: guided; only tokens of the partial last 8-group are allowed (greedy, and a seeded draw)
    last0 = V // 8 * 8
    allowed = list(range(last0, V))
    words = (V + 31) // 32
    allow = np.zeros((n, words), dtype=np.uint32)
    for t in allowed:
        allow[2:, t >> 5] |= np.uint32(1) << np.uint32(t & 31)
    rows["flags"][2] = g.SAMPLE_GREEDY | g.SAMPLE_LOGPROBS | g.SAMPLE_MASKED
    rows["flags"][3] = g.SAMPLE_LOGPROBS | g.SAMPLE_MASKED
    rows["seed_lo"][3] = 9
    rows["n_topn"][2:] = 3
    rows["seq_slot"][2:] = [2, 3]
    out = _sample(g, buf, V, rows, allow=torch.from_numpy(allow.view(np.int32)).cuda())
    for i, t in ((0, V - 1), (1, 0)):
        lp = torch.log_softmax(logits[i], -1)
        assert int(out["token"][i]) == t
        assert abs(out["logprob"][i] - float(lp[t])) < 1e-3
        assert out["rank"][i] == int((lp >= lp[t]).sum())
        assert all(0 <= x < V for x in out["topn_ids"][i][:4])
    mask = torch.zeros(V, dtype=torch.bool)
    mask[allowed] = True
    for i, case in ((2, SamplingCase(greedy=True, num_logprobs=3)),
                    (3, SamplingCase(greedy=False, seed=9, num_logprobs=3))):
        o = sample_row(logits[i], case, None, allow=mask)
        assert int(out["token"][i]) == o["token"] and o["token"] in allowed
        assert abs(out["logprob"][i] - o["logprob"]) < 1e-3 and out["rank"][i] == o["rank"]
        assert sorted(out["topn_ids"][i][:3].tolist()) == sorted(o["topn_ids"]) or len(allowed) < 3


@pytest.mark.parametrize("scale", [1.0 / 3.0, 1.0 / 16.0])
@pytest.mark.parametrize("V", [1021, 49155])
def test_sampler_logit_scale_reports_the_scaled_row(g, V, scale):
    torch.manual_seed(int(V * scale * 48))
    cases = _cases(V)
    n = len(cases)
    logits = (torch.randn(n, V) * 6).to(torch.bfloat16).float()
    buf = _padded(logits)
    before = buf.clone()
    rows = _rows(g, n)
    _fill_rows(g, rows, cases, V)
    out = np.zeros(n, dtype=g.SAMPLE_OUT_DTYPE)
    rc = g.lib().tgis_k_sampler_scaled(g.ptr(buf), 1, buf.stride(0), V, rows.ctypes.data_as(g.C.c_void_p), n, None,
                                       None, out.ctypes.data_as(g.C.c_void_p), scale)
    assert rc == 0, g.kerr()
    assert torch.equal(buf, before)
    scaled = (logits.to(torch.bfloat16) * torch.tensor(scale, dtype=torch.float32)).to(torch.bfloat16).float()
    # (rows with repetition penalty carry no seen bitmap here: nothing is penalised)
    _check(out, scaled, cases, [None] * n, V)


# ----------------------------------------------------------------------------------------------------- engine
def _mc(cfg, **over):
    from vllm_tgis_adapter_b200.engine.core import ModelConfig

    return ModelConfig(n_layers=cfg.n_layers, hidden=cfg.hidden, n_q_heads=cfg.n_q_heads, n_kv_heads=cfg.n_kv_heads,
                       ffn=cfg.ffn, vocab=cfg.vocab, rope_theta=cfg.rope_theta, rms_eps=cfg.rms_eps,
                       max_model_len=cfg.max_model_len, tie_word_embeddings=cfg.tie_word_embeddings,
                       embedding_multiplier=cfg.embedding_multiplier, residual_multiplier=cfg.residual_multiplier,
                       attention_multiplier=cfg.attention_multiplier, logits_scaling=cfg.logits_scaling, **over)


def _run_engine(prompts, sp, seed=1, max_loras=0, adapters=None, **kw):
    from granite_oracle import CONFIGS, synthetic_weights
    from oracle.llama_oracle import rope_table
    from vllm_tgis_adapter_b200.engine.core import NativeEngine

    cfg = CONFIGS["granite-tiny"]
    weights = synthetic_weights(cfg, seed=seed)
    assert "lm_head.weight" not in weights
    eng = NativeEngine(_mc(cfg), max_loras=max_loras, max_lora_rank=16, **kw)
    eng.load_weights(weights)
    eng.load_weight("tgis.rope_cos_sin", rope_table(cfg))
    for slot, ad in (adapters or {}).items():
        eng.load_adapter(slot, ad)
    outs = eng.generate_sync(prompts, sp)
    st = eng.status()
    eng.close()
    assert st.errored == 0
    return cfg, weights, outs, st


def _tokens(outs):
    return [[(r.new_token, r.logprob, r.rank, tuple(r.topn)) for r in recs if r.new_token is not None] for recs in outs]


def _check_greedy_vs_oracle(cfg, weights, prompts, outs, n_new, lora=None):
    from granite_oracle import GraniteOracle

    ora = GraniteOracle(cfg, weights)
    flips, total, diffs = 0, 0, []
    for p, recs in zip(prompts, outs):
        toks = [r for r in recs if r.new_token is not None]
        assert len(toks) == n_new
        st = ora.new_seq()
        logits = ora.step([(st, p)], lora=[lora] if lora else None)[0]
        for r in toks:
            assert 0 <= r.new_token < cfg.vocab
            lp = torch.log_softmax(logits, -1)
            top2 = torch.topk(logits, 2).values
            margin = float(top2[0] - top2[1])
            total += 1
            diffs.append(abs(r.logprob - float(lp[r.new_token])))
            if r.new_token != int(torch.argmax(logits)):
                assert margin < 0.02, (margin, r.new_token)
                flips += 1
            elif margin > 0.02:
                assert r.rank == int((lp >= lp[r.new_token]).sum())
            logits = ora.step([(st, [r.new_token])], lora=[lora] if lora else None)[0]
    diffs = np.array(diffs)
    assert flips <= max(1, total // 25), (flips, total)
    assert float(diffs.mean()) < 4e-3 and float(np.percentile(diffs, 95)) < 1e-2 and float(diffs.max()) < 2e-2, (
        float(diffs.mean()), float(diffs.max()))


@pytest.mark.parametrize("chunk", [2048, 48])
def test_granite_tiny_greedy_matches_oracle(chunk):
    from granite_oracle import CONFIGS
    from vllm_tgis_adapter_b200.engine.core import make_sampling_params

    V = CONFIGS["granite-tiny"].vocab
    rng = np.random.RandomState(0)
    prompts = [rng.randint(3, V, size=n).tolist() for n in (5, 33, 64, 100, 17, 250)]
    prompts[0][-1] = V - 1                     # the last (partial-group) token id is a valid prompt token
    n_new = 24
    sp = make_sampling_params(greedy=True, max_tokens=n_new, min_tokens=n_new, num_logprobs=1, eos_token_id=2)
    cfg, w, outs, st = _run_engine(prompts, sp, max_num_seqs=8, max_batched_tokens=chunk, kv_cache_bytes=64 << 20)
    assert st.graph_launches > 0
    _check_greedy_vs_oracle(cfg, w, prompts, outs, n_new)


def test_granite_tiny_rejects_out_of_vocab_prompt_ids():
    from granite_oracle import CONFIGS
    from vllm_tgis_adapter_b200.engine.core import EngineError, NativeEngine, make_sampling_params

    cfg = CONFIGS["granite-tiny"]
    eng = NativeEngine(_mc(cfg), max_num_seqs=2, max_batched_tokens=64, kv_cache_bytes=16 << 20)
    try:
        with pytest.raises(EngineError, match="out of range"):
            eng.add_request("x", [5, cfg.vocab], make_sampling_params(max_tokens=2))   # 1021: padding row, not a token
    finally:
        eng.close()


@pytest.mark.parametrize("chunk", [2048, 48])
def test_granite_tiny_prompt_logprobs_match_oracle(chunk):
    from granite_oracle import GraniteOracle
    from vllm_tgis_adapter_b200.engine.core import make_sampling_params

    rng = np.random.RandomState(7)
    prompts = [rng.randint(3, 1021, size=n).tolist() for n in (100, 9, 37)]
    sp = make_sampling_params(greedy=True, max_tokens=2, num_logprobs=1, prompt_logprobs=3)
    cfg, w, outs, _ = _run_engine(prompts, sp, max_num_seqs=4, max_batched_tokens=chunk, kv_cache_bytes=32 << 20)
    ora = GraniteOracle(cfg, w)
    diffs = []
    for p, recs in zip(prompts, outs):
        prec = sorted([r for r in recs if r.prompt_pos >= 1], key=lambda r: r.prompt_pos)
        assert [r.prompt_pos for r in prec] == list(range(1, len(p)))
        logits = ora.step([(ora.new_seq(), p)], want_all_logits=True)
        lp = torch.log_softmax(logits, -1)
        for r in prec:
            i = r.prompt_pos
            assert r.token_id == p[i]
            ref = float(lp[i - 1, p[i]])
            diffs.append(abs(r.logprob - ref))
            lo = int((lp[i - 1] > ref + 0.03).sum()) + 1
            hi = int((lp[i - 1] >= ref - 0.03).sum())
            assert lo <= r.rank <= hi, (r.rank, lo, hi)
            assert len(r.topn) == 3 and all(0 <= t < cfg.vocab for t, _ in r.topn)
            top = torch.topk(lp[i - 1], 3)
            assert abs(r.topn[0][1] - float(top.values[0])) < 2e-2
    diffs = np.array(diffs)
    assert float(diffs.mean()) < 4e-3 and float(diffs.max()) < 3e-2, (float(diffs.mean()), float(diffs.max()))


def test_granite_tiny_graphs_and_batch_invariance():
    """CUDA-graph replay == plain launches, and a prompt alone == the same prompt in a crowded batch with preemption: bit
    for bit."""
    from vllm_tgis_adapter_b200.engine.core import make_sampling_params

    rng = np.random.RandomState(13)
    prompts = [rng.randint(3, 1021, size=n).tolist() for n in (70, 5, 130, 33, 64, 200)]
    sp = make_sampling_params(greedy=True, max_tokens=24, min_tokens=24, num_logprobs=2)
    kw = dict(max_num_seqs=8, max_batched_tokens=96, kv_cache_bytes=64 << 20)
    _, _, a, st_a = _run_engine(prompts, sp, use_cuda_graphs=True, **kw)
    _, _, b, st_b = _run_engine(prompts, sp, use_cuda_graphs=False, **kw)
    assert st_a.graph_launches > 0 and st_b.graph_launches == 0
    assert _tokens(a) == _tokens(b)
    sp40 = make_sampling_params(greedy=True, max_tokens=40, min_tokens=40)
    _, _, solo, _ = _run_engine(prompts[:1], sp40, max_num_seqs=1, max_batched_tokens=512, kv_cache_bytes=32 << 20)
    _, _, crowd, st = _run_engine(prompts, sp40, max_num_seqs=6, max_batched_tokens=64, kv_cache_bytes=17 * 65536)
    assert [r.new_token for r in solo[0] if r.new_token is not None] == \
        [r.new_token for r in crowd[0] if r.new_token is not None]
    assert st.preemptions > 0
    for recs in crowd:
        assert len([r for r in recs if r.new_token is not None]) == 40


def test_granite_engine_starts_on_its_checkpoint_and_64_dim_heads_refused():
    import dataclasses

    from granite_oracle import CONFIGS, synthetic_weights
    from vllm_tgis_adapter_b200.engine.core import EngineError, NativeEngine

    cfg = CONFIGS["granite-tiny"]
    eng = NativeEngine(_mc(cfg), max_num_seqs=2, max_batched_tokens=64, kv_cache_bytes=16 << 20)
    eng.load_weights(synthetic_weights(cfg, seed=1))   # start refuses a checkpoint with tensors missing
    eng.start()
    eng.close()
    with pytest.raises(EngineError, match="finite and non-negative"):
        NativeEngine(dataclasses.replace(_mc(cfg), residual_multiplier=-1.0), max_num_seqs=2, max_batched_tokens=64,
                     kv_cache_bytes=16 << 20)
    with pytest.raises(EngineError, match="head_dim"):
        NativeEngine(_mc(cfg, head_dim=64), max_num_seqs=2, max_batched_tokens=64, kv_cache_bytes=16 << 20)


def test_granite_tiny_lora_matches_oracle_and_leaves_base_requests_untouched(tmp_path):
    from test_lora_cpu import make_peft_dir

    from granite_oracle import CONFIGS
    from vllm_tgis_adapter_b200.engine.core import make_sampling_params
    from vllm_tgis_adapter_b200.engine.lora import read_adapter

    cfg = CONFIGS["granite-tiny"]
    d = make_peft_dir(tmp_path, "a", n_layers=cfg.n_layers, hidden=cfg.hidden, q_dim=cfg.q_dim, kv_dim=cfg.kv_dim,
                      ffn=cfg.ffn, r=8, alpha=16, seed=1)
    ad = read_adapter(str(d), n_layers=cfg.n_layers, max_rank=16)[1]
    rng = np.random.RandomState(7)
    prompts = [rng.randint(3, cfg.vocab, size=n).tolist() for n in (5, 33, 64, 17)]
    n_new = 16

    def sps(slots):
        return [make_sampling_params(greedy=True, max_tokens=n_new, min_tokens=n_new, num_logprobs=1, eos_token_id=2,
                                     lora_slot=s) for s in slots]

    kw = dict(max_num_seqs=8, max_batched_tokens=2048, kv_cache_bytes=64 << 20)
    _, w, base, _ = _run_engine(prompts, sps([0] * 4), **kw)
    _, _, mixed, _ = _run_engine(prompts, sps([1, 1, 0, 0]), max_loras=1, adapters={1: ad}, **kw)
    base_t, mixed_t = _tokens(base), _tokens(mixed)
    assert mixed_t[2] == base_t[2] and mixed_t[3] == base_t[3]
    assert mixed_t[0] != base_t[0]
    _check_greedy_vs_oracle(cfg, w, prompts[:2], mixed[:2], n_new, lora=ad)


def test_granite_checkpoint_loads_through_the_model_directory(tmp_path):
    """A tiny HF GraniteForCausalLM saved with save_pretrained (tied embeddings, odd vocabulary): config.json mapping,
    safetensors loading and the engine's lm_head tie; greedy tokens follow the oracle on the same weights."""
    import argparse

    from transformers import GraniteConfig as HFGraniteConfig
    from transformers import GraniteForCausalLM

    from granite_oracle import GraniteConfig
    from vllm_tgis_adapter_b200.engine.core import make_sampling_params
    from vllm_tgis_adapter_b200.engine.loader import _make_native_engine, _resolve_model

    hf_cfg = HFGraniteConfig(vocab_size=1021, hidden_size=256, intermediate_size=512, num_hidden_layers=2,
                           num_attention_heads=2, num_key_value_heads=1, rms_norm_eps=1e-5, max_position_embeddings=512,
                           tie_word_embeddings=True, embedding_multiplier=12.0, residual_multiplier=0.22,
                           attention_multiplier=1.0 / 128, logits_scaling=3.0)
    torch.manual_seed(0)
    model = GraniteForCausalLM(hf_cfg).to(torch.bfloat16)
    with torch.no_grad():
        for p in model.parameters():
            if p.dim() == 2:
                p.normal_(0, 0.02)
    model.save_pretrained(tmp_path, safe_serialization=True)
    args = argparse.Namespace(model=str(tmp_path), max_model_len=None, synthetic_weights=False, max_num_seqs=4,
                              max_num_batched_tokens=256, gpu_memory_utilization=0.05, seed=0, enable_lora=False)
    mc, path = _resolve_model(args)
    assert mc.vocab == 1021 and mc.is_granite and mc.tie_word_embeddings and mc.head_dim == 128
    eng = _make_native_engine(args, mc, path, device=0)
    prompts = [[5, 17, 1000, 3, 250, 77, 9, 640, 1020], [12, 13, 14]]
    n_new = 12
    outs = eng.generate_sync(prompts, make_sampling_params(greedy=True, max_tokens=n_new, min_tokens=n_new,
                                                           num_logprobs=1))
    eng.close()
    sd = {k: v for k, v in model.state_dict().items() if "rotary" not in k and k != "lm_head.weight"}
    cfg = GraniteConfig(n_layers=2, hidden=256, n_q_heads=2, n_kv_heads=1, ffn=512, vocab=1021,
                      rope_theta=mc.rope_theta, rms_eps=1e-5, max_model_len=mc.max_model_len,
                      embedding_multiplier=12.0, residual_multiplier=0.22, attention_multiplier=1.0 / 128,
                      logits_scaling=3.0, tie_word_embeddings=True)
    _check_greedy_vs_oracle(cfg, sd, prompts, outs, n_new)
