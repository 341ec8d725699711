"""-m gpu: Qwen3.  The RoPE + KV writer with the per-head q / k RMSNorm (rope_kvwrite_kernel<128, QKNORM>) bit for bit
against a torch restatement of its own summation order, and within 1 bf16 ulp of the oracle's fp32 norm; the engine on
the qwen3-tiny preset against tests/qwen3_oracle.py with the bars of tests/test_llama3_gpu.py (greedy, prompt logprobs,
LoRA); bit-identity under batching with preemption, CUDA graphs and prefix-cache hits; the start-up refusals; a
save_pretrained checkpoint directory; and the qwen3-0.6b preset over gRPC."""
import dataclasses
import math

import numpy as np
import pytest
import torch

from qwen3_oracle import CONFIGS, Qwen3Config, Qwen3Oracle, synthetic_weights

pytestmark = pytest.mark.gpu

_W = {}


@pytest.fixture(scope="module")
def g():
    import tgis_gpu_utils as gpu_utils

    return gpu_utils


def _cfg(**over):
    return dataclasses.replace(CONFIGS["qwen3-tiny"], **over)


def _mc(**over):
    from vllm_tgis_adapter_b200.engine.core import PRESETS

    return dataclasses.replace(PRESETS["qwen3-tiny"], **over)


def _weights():
    if "w" not in _W:
        _W["w"] = synthetic_weights(_cfg(), seed=6)
    return _W["w"]


def _engine(max_model_len=2048, weights=None, **kw):
    from oracle.llama_oracle import rope_table
    from vllm_tgis_adapter_b200.engine.core import NativeEngine

    kw.setdefault("max_num_seqs", 8)
    kw.setdefault("kv_cache_bytes", 32 << 20)
    eng = NativeEngine(_mc(max_model_len=max_model_len), **kw)
    eng.load_weights(weights or _weights())          # no lm_head.weight: tied
    eng.load_weight("tgis.rope_cos_sin", rope_table(_cfg(max_model_len=max_model_len)))
    return eng


def _sp(**kw):
    from vllm_tgis_adapter_b200.engine.core import make_sampling_params

    d = dict(greedy=True, max_tokens=16, min_tokens=16, num_logprobs=1, eos_token_id=2)
    d.update(kw)
    return make_sampling_params(**d)


def _gen(eng, prompts, sp):
    outs = eng.generate_sync(prompts, sp)
    return [[(r.new_token, r.logprob, r.rank, tuple(r.topn)) for r in recs if r.new_token is not None] for recs in outs]


def _prompt(n, seed, vocab=1021):
    return np.random.RandomState(seed).randint(3, vocab, size=n).tolist()


def _ulp(x: float) -> float:
    return 2.0 ** (math.floor(math.log2(max(abs(x), 1e-6))) - 7)


# ----------------------------------------------------------------------------------------------------- the kernel
POISON = -77.5   # a bf16 value no write produces here: every cache slot the writer must not touch keeps it


def _restate(qkv, positions, table, q_norm, k_norm, eps, n_q, n_kv):
    """rope_kvwrite_kernel<128, QKNORM> in torch, on the device: per thread c = 0..7 of a head, fp32 squares of dims
    8c..8c+7 then 64+8c..64+8c+7 added one at a time from 0; the 8 partials combined as ((s0 + s1) + (s2 + s3)) +
    ((s4 + s5) + (s6 + s7)); rs = rsqrt(ss / 128 + eps); y = bf16(bf16(x * rs) * w); then the bf16 rotation.
    Returns the q and k heads, normalised and rotated, [T, n_q + n_kv, 128] bf16."""
    T = qkv.shape[0]
    nh = n_q + n_kv
    x = qkv[:, :nh].float()
    lo, hi = x[..., :64].reshape(T, nh, 8, 8), x[..., 64:].reshape(T, nh, 8, 8)
    s = torch.zeros(T, nh, 8, dtype=torch.float32, device=qkv.device)
    for e in range(8):
        s = s + lo[..., e] * lo[..., e]
    for e in range(8):
        s = s + hi[..., e] * hi[..., e]
    s = s[..., 0::2] + s[..., 1::2]
    s = s[..., 0::2] + s[..., 1::2]
    ss = s[..., 0] + s[..., 1]
    rs = torch.rsqrt(ss / 128.0 + eps)
    w = torch.cat([q_norm[None].expand(n_q, 128), k_norm[None].expand(n_kv, 128)]).float()
    y = ((x * rs[..., None]).bfloat16().float() * w).bfloat16()
    cs = table[torch.from_numpy(positions).long().to(qkv.device)]
    cos, sin = cs[:, None, :64], cs[:, None, 64:]
    y1, y2 = y[..., :64], y[..., 64:]
    return torch.cat([y1 * cos - y2 * sin, y2 * cos + y1 * sin], dim=-1)


def _run_writer(g, qkv, positions, slots, table, q_norm, k_norm, eps, n_q, n_kv, n_blocks):
    kc = torch.full((n_blocks, n_kv, 16, 32, 8), POISON, dtype=torch.bfloat16, device="cuda")
    vc = torch.full((n_blocks, n_kv, 32, 16, 8), POISON, dtype=torch.bfloat16, device="cuda")
    out = qkv.clone()
    rc = g.lib().tgis_k_rope_kv_qknorm(g.ptr(out), g.i32p(positions), g.i32p(slots), g.ptr(table), g.ptr(kc), g.ptr(vc),
                                       qkv.shape[0], n_q, n_kv, g.ptr(q_norm), g.ptr(k_norm), eps, 1, None)
    assert rc == 0, g.kerr()
    return out, kc, vc


@pytest.mark.parametrize("heads", [(16, 8), (32, 8), (4, 2)], ids=["0.6b", "8b", "tiny"])
@pytest.mark.parametrize("T", [1, 31, 32, 257, 2048])
def test_qknorm_writer_is_bit_exact_against_its_summation_order(g, heads, T):
    n_q, n_kv = heads
    nh = n_q + 2 * n_kv
    gen = torch.Generator(device="cuda").manual_seed(T * 100 + n_q)
    # each head at its own scale (0.01 .. 30), so the norm has work to do; weights well away from 1
    scale = torch.exp(torch.empty(T, nh, 1, device="cuda").uniform_(math.log(0.01), math.log(30.0), generator=gen))
    qkv = (torch.randn(T, nh, 128, device="cuda", generator=gen) * scale).bfloat16()
    q_norm = (0.25 + 2.25 * torch.rand(128, device="cuda", generator=gen)).bfloat16()
    k_norm = (0.25 + 2.25 * torch.rand(128, device="cuda", generator=gen)).bfloat16()
    max_pos = 8192
    table = (torch.rand(max_pos, 128, device="cuda", generator=gen) * 2 - 1).bfloat16()
    rs = np.random.RandomState(T + n_q)
    positions = rs.randint(0, max_pos, size=T).astype(np.int32)
    positions[0] = max_pos - 1
    assert T == 1 or (positions > 4096).any()
    n_blocks = (T + 31) // 32 + 3
    slots = rs.permutation(n_blocks * 32)[:T].astype(np.int32)
    slots[rs.rand(T) < 0.1] = -1             # "do not cache" rows
    if T > 1:
        slots[1] = -1
    eps = 1e-6
    out, kc, vc = _run_writer(g, qkv, positions, slots, table, q_norm, k_norm, eps, n_q, n_kv, n_blocks)
    want = _restate(qkv, positions, table, q_norm, k_norm, eps, n_q, n_kv)
    assert torch.equal(out[:, :n_q + n_kv], want)
    assert torch.equal(out[:, n_q + n_kv:], qkv[:, n_q + n_kv:])          # V untouched in qkv
    k_dense, v_dense = g.dense_from_k_cache(kc), g.dense_from_v_cache(vc)
    cached = torch.from_numpy(slots[slots >= 0]).long().cuda()
    rows = torch.from_numpy(np.nonzero(slots >= 0)[0]).long().cuda()
    assert torch.equal(k_dense[cached], want[rows, n_q:])
    assert torch.equal(v_dense[cached], qkv[rows, n_q + n_kv:])
    untouched = torch.ones(n_blocks * 32, dtype=torch.bool, device="cuda")
    untouched[cached] = False
    assert bool((k_dense[untouched] == POISON).all()) and bool((v_dense[untouched] == POISON).all())
    # the plain writer on the same input differs: the norm did run
    plain = qkv.clone()
    kc2, vc2 = torch.zeros_like(kc), torch.zeros_like(vc)
    assert g.lib().tgis_k_rope_kv_qknorm(g.ptr(plain), g.i32p(positions), g.i32p(slots), g.ptr(table), g.ptr(kc2),
                                         g.ptr(vc2), T, n_q, n_kv, None, None, 0.0, 1, None) == 0, g.kerr()
    assert not torch.equal(plain[:, :n_q + n_kv], out[:, :n_q + n_kv])


def test_qknorm_agrees_with_the_oracle_fp32_norm_within_one_ulp(g):
    """with cos = 1, sin = 0 the rotation is the identity, so the writer's output is the norm itself: within 1 bf16 ulp of
    Qwen3RMSNorm as the oracle computes it (fp32 mean of squares in torch's order, torch rsqrt)"""
    n_q, n_kv, T = 16, 8, 257
    nh = n_q + 2 * n_kv
    gen = torch.Generator(device="cuda").manual_seed(3)
    scale = torch.exp(torch.empty(T, nh, 1, device="cuda").uniform_(math.log(0.01), math.log(30.0), generator=gen))
    qkv = (torch.randn(T, nh, 128, device="cuda", generator=gen) * scale).bfloat16()
    q_norm = (0.25 + 2.25 * torch.rand(128, device="cuda", generator=gen)).bfloat16()
    k_norm = (0.25 + 2.25 * torch.rand(128, device="cuda", generator=gen)).bfloat16()
    table = torch.cat([torch.ones(16, 64), torch.zeros(16, 64)], dim=-1).bfloat16().cuda()
    positions = np.arange(T, dtype=np.int32) % 16
    slots = np.full(T, -1, dtype=np.int32)
    out, _, _ = _run_writer(g, qkv, positions, slots, table, q_norm, k_norm, 1e-6, n_q, n_kv, 1)
    cfg = Qwen3Config(n_layers=1, hidden=256, n_q_heads=n_q, n_kv_heads=n_kv, ffn=256, vocab=64, rms_eps=1e-6,
                      max_model_len=16)
    w = synthetic_weights(cfg, seed=0)
    w["model.layers.0.self_attn.q_norm.weight"], w["model.layers.0.self_attn.k_norm.weight"] = q_norm.cpu(), k_norm.cpu()
    ora = Qwen3Oracle(cfg, w)
    ref = torch.cat([ora.head_norm(qkv[:, :n_q].cpu(), q_norm.cpu()),
                     ora.head_norm(qkv[:, n_q:n_q + n_kv].cpu(), k_norm.cpu())], dim=1)
    got = out[:, :n_q + n_kv].cpu()
    ulps = g.bf16_ulp_diff(got, ref)
    assert float(ulps.max()) <= 1.0
    assert float((ulps == 0).float().mean()) > 0.95


# ----------------------------------------------------------------------------------------------------- the engine
def _check_greedy(cfg, weights, prompts, outs, n_new):
    """teacher-forced on the engine's tokens: a flip only inside a 2-ulp race, logprobs within 3 bf16 ulps of the top
    logit, rank 1 outside a race, the top-n ids and values against the oracle's"""
    ora = Qwen3Oracle(cfg, weights, device="cuda")
    flips = steps = 0
    for p, recs in zip(prompts, outs):
        recs = [r for r in recs if r.new_token is not None]
        assert len(recs) == n_new
        s = ora.new_seq()
        logits = ora.step([(s, p)])[0]
        for r in recs:
            lp = torch.log_softmax(logits, -1)
            top2 = torch.topk(logits, 2).values
            u, margin = _ulp(float(top2[0])), float(top2[0] - top2[1])
            steps += 1
            if r.new_token != int(torch.argmax(logits)):
                assert margin <= 2 * u + 1e-6, (margin, u)
                flips += 1
            elif margin > 2 * u:
                assert r.rank == 1
            assert abs(r.logprob - float(lp[r.new_token])) <= 3 * u
            for tid, tlp in r.topn:
                assert abs(tlp - float(lp[tid])) <= 3 * u
                assert float(lp[tid]) >= float(torch.topk(lp, len(r.topn)).values[-1]) - 2 * u
            logits = ora.step([(s, [r.new_token])])[0]
    assert flips <= steps // 10, (flips, steps)


@pytest.mark.parametrize("chunk", [2048, 48])
def test_greedy_generation_matches_the_qwen3_oracle(chunk):
    prompts = [_prompt(n, 10 + n) for n in (5, 70, 129, 300, 700)]
    prompts[0][-1] = 1020                      # the last token id of the odd vocabulary
    n_new = 16
    eng = _engine(max_batched_tokens=chunk)
    outs = eng.generate_sync(prompts, _sp(max_tokens=n_new, min_tokens=n_new, num_logprobs=3))
    st = eng.status()
    eng.close()
    assert st.errored == 0 and st.graph_launches > 0
    _check_greedy(_cfg(), _weights(), prompts, outs, n_new)


@pytest.mark.parametrize("chunk", [2048, 48])
def test_prompt_logprobs_match_the_qwen3_oracle(chunk):
    prompts = [_prompt(n, 70 + n) for n in (100, 9, 37)]
    eng = _engine(max_batched_tokens=chunk)
    outs = eng.generate_sync(prompts, _sp(max_tokens=2, min_tokens=0, prompt_logprobs=3))
    eng.close()
    ora = Qwen3Oracle(_cfg(), _weights(), device="cuda")
    for p, recs in zip(prompts, outs):
        prec = sorted([r for r in recs if r.prompt_pos >= 1], key=lambda r: r.prompt_pos)
        assert [r.prompt_pos for r in prec] == list(range(1, len(p)))
        logits = ora.step([(ora.new_seq(), p)], want_all_logits=True)
        lp = torch.log_softmax(logits, -1)
        for r in prec:
            i = r.prompt_pos
            assert r.token_id == p[i]
            u = _ulp(float(logits[i - 1].max()))
            ref = float(lp[i - 1, p[i]])
            assert abs(r.logprob - ref) <= 3 * u, (i, r.logprob, ref)
            lo = int((lp[i - 1] > ref + 3 * u).sum()) + 1
            hi = int((lp[i - 1] >= ref - 3 * u).sum())
            assert lo <= r.rank <= hi, (r.rank, lo, hi)
            assert len(r.topn) == 3
            assert abs(r.topn[0][1] - float(lp[i - 1].max())) <= 3 * u


def test_batch_invariance_with_preemption():
    """a prompt alone vs in a crowded batch over a KV cache so small that sequences are preempted and recomputed: the same
    tokens and logprobs, bit for bit"""
    prompts = [_prompt(n, n) for n in (60, 90, 40, 75, 33, 120)]
    sp = _sp(max_tokens=40, min_tokens=40)
    solo_eng = _engine(max_model_len=512, max_num_seqs=1, max_batched_tokens=512)
    solo = _gen(solo_eng, prompts[:1], sp)
    solo_eng.close()
    # 2 layers * 2 kv heads * 32 tok * 128 dims * 2 B * 2 (K, V) = 64 KiB per block; 17 blocks = 544 tokens for 6 sequences
    crowd_eng = _engine(max_model_len=512, max_num_seqs=6, max_batched_tokens=64, kv_cache_bytes=17 * 65536)
    crowd = _gen(crowd_eng, prompts, sp)
    st = crowd_eng.status()
    crowd_eng.close()
    assert st.total_blocks == 17 and st.preemptions > 0 and st.errored == 0
    assert crowd[0] == solo[0]
    assert all(len(c) == 40 for c in crowd)


def test_cuda_graphs_on_and_off_give_identical_ids():
    prompts = [_prompt(n, 50 + n) for n in (20, 130, 260)]
    res = {}
    for graphs in (True, False):
        eng = _engine(use_cuda_graphs=graphs)
        res[graphs] = _gen(eng, prompts, _sp(max_tokens=24, min_tokens=24, num_logprobs=2))
        st = eng.status()
        eng.close()
        assert (st.graph_launches > 0) == graphs
    assert res[True] == res[False]


def test_prefix_cache_hit_takes_the_split_context_kernel_and_changes_nothing():
    """P = 1024 shared tokens + a 100-token tail; with P's prefix cached, P's prefill is a 100-row suffix over 1024 cached
    tokens (the split-context kernel).  Ids and logprobs equal a cold engine chunked at the same boundary, bit for bit."""
    P = _prompt(1124, 1)
    X = P[:1024] + _prompt(100, 2)
    cold = _engine(max_batched_tokens=1024, enable_prefix_caching=True)
    want = _gen(cold, [P], _sp())
    cold.close()
    eng = _engine(max_batched_tokens=1024, enable_prefix_caching=True)
    _gen(eng, [X], _sp())
    q0, h0, _ = eng.prefix_cache_stats()
    got = _gen(eng, [P], _sp())
    q1, h1, _ = eng.prefix_cache_stats()
    eng.close()
    assert h0 == 0 and q1 - q0 == len(P) and h1 - h0 == 1024
    assert got == want


def test_lora_follows_the_oracle_and_leaves_base_requests_untouched(tmp_path):
    """adapter deltas land on the raw q / k / v, before the per-head norm (vLLM: qkv_proj's output carries the delta)"""
    from test_lora_cpu import make_peft_dir

    from vllm_tgis_adapter_b200.engine.lora import read_adapter

    cfg = _cfg()
    d = make_peft_dir(tmp_path, "a", n_layers=cfg.n_layers, hidden=cfg.hidden, q_dim=cfg.q_dim, kv_dim=cfg.kv_dim,
                      ffn=cfg.ffn, r=8, alpha=16, seed=1)
    ad = read_adapter(str(d), n_layers=cfg.n_layers, max_rank=16)[1]
    prompts = [_prompt(n, 200 + n) for n in (5, 33, 64, 17)]
    n_new = 16

    def sps(slots):
        return [_sp(max_tokens=n_new, min_tokens=n_new, lora_slot=s) for s in slots]

    base_eng = _engine()
    base = _gen(base_eng, prompts, sps([0] * 4))
    base_eng.close()
    eng = _engine(max_loras=1, max_lora_rank=16)
    eng.load_adapter(1, ad)
    outs = eng.generate_sync(prompts, sps([1, 1, 0, 0]))
    st = eng.status()
    eng.close()
    assert st.errored == 0
    mixed = [[(r.new_token, r.logprob, r.rank, tuple(r.topn)) for r in recs if r.new_token is not None] for recs in outs]
    assert mixed[2] == base[2] and mixed[3] == base[3]
    assert mixed[0] != base[0] and mixed[1] != base[1]
    # adapter requests vs the oracle's LoRA forward, teacher-forced on the engine's tokens, at the bars of
    # tests/test_lora_gpu.py (the shrink / expand sums round in another order than torch's)
    ora = Qwen3Oracle(cfg, _weights(), device="cuda")
    flips = total = 0
    diffs = []
    for p, toks in zip(prompts[:2], mixed[:2]):
        s = ora.new_seq()
        logits = ora.step([(s, p)], lora=[ad])[0]
        for tok, lp, _, _ in toks:
            olp = torch.log_softmax(logits, -1)
            top2 = torch.topk(logits, 2).values
            total += 1
            diffs.append(abs(lp - float(olp[tok])))
            if int(torch.argmax(logits)) != tok:
                assert float(top2[0] - top2[1]) < 0.03
                flips += 1
            logits = ora.step([(s, [tok])], lora=[ad])[0]
    diffs = np.array(diffs)
    assert flips <= max(1, total // 12), (flips, total)
    assert float(diffs.mean()) < 6e-3 and float(diffs.max()) < 4e-2, (float(diffs.mean()), float(diffs.max()))


def test_start_up_refusals():
    from vllm_tgis_adapter_b200.engine.core import PRESETS, EngineError, NativeEngine

    kw = dict(max_num_seqs=2, max_batched_tokens=64, kv_cache_bytes=16 << 20)
    with pytest.raises(EngineError, match="tgis_engine_create failed: .*not OPT"):
        NativeEngine(dataclasses.replace(PRESETS["opt-tiny"], qk_norm=True), **kw)
    with pytest.raises(EngineError, match="tgis_engine_create failed: .*head_dim 128"):
        NativeEngine(_mc(head_dim=64, n_q_heads=4, hidden=256), **kw)
    with pytest.raises(EngineError, match="single GPU only"):
        NativeEngine(_mc(), tp_size=2, tp_rank=0, nccl_id=bytes(128), shm_name="/tgis_test_unused", **kw)
    # a missing vector: start fails and names the layer
    eng = NativeEngine(_mc(), **kw)
    w = dict(_weights())
    del w["model.layers.1.self_attn.k_norm.weight"]
    eng.load_weights(w)
    with pytest.raises(EngineError, match=r"layer 1 has no model\.layers\.1\.self_attn\.k_norm\.weight"):
        eng.start()
    with pytest.raises(EngineError, match="layer 1"):
        eng.run_until_idle()
    # a wrong length is an error, and does not count as loaded
    with pytest.raises(EngineError, match="shape mismatch"):
        eng.load_weight("model.layers.1.self_attn.k_norm.weight", torch.ones(64, dtype=torch.bfloat16))
    with pytest.raises(EngineError, match="layer 1"):
        eng.start()
    eng.load_weight("model.layers.1.self_attn.k_norm.weight", _weights()["model.layers.1.self_attn.k_norm.weight"])
    eng.start()
    eng.close()
    # the norm weights are not names a Llama engine knows, as before
    eng = NativeEngine(_mc(qk_norm=False), **kw)
    with pytest.raises(EngineError, match="unknown layer weight model.layers.0.self_attn.q_norm.weight"):
        eng.load_weight("model.layers.0.self_attn.q_norm.weight", torch.ones(128, dtype=torch.bfloat16))
    eng.close()


def test_hf_checkpoint_directory_loads_and_follows_the_oracle(tmp_path):
    """Qwen3ForCausalLM.save_pretrained (bf16, tied, q width != hidden, odd vocabulary) with the synthetic tokenizer saved
    beside it: the loader's config mapping, the safetensors reader and the tokenizer; greedy tokens follow the oracle"""
    import argparse

    from transformers import Qwen3Config as HFQwen3Config
    from transformers import Qwen3ForCausalLM

    from vllm_tgis_adapter_b200.engine.loader import _make_native_engine, _resolve_model
    from vllm_tgis_adapter_b200.engine.tokenizer import build_synthetic_tokenizer, load_tokenizer, synthetic_prompt

    hf_cfg = HFQwen3Config(vocab_size=1021, hidden_size=256, intermediate_size=512, num_hidden_layers=2,
                           num_attention_heads=4, num_key_value_heads=2, head_dim=128, rms_norm_eps=1e-6,
                           max_position_embeddings=1024, tie_word_embeddings=True,
                           rope_parameters={"rope_type": "default", "rope_theta": 1000000.0})
    torch.manual_seed(0)
    model = Qwen3ForCausalLM(hf_cfg).to(torch.bfloat16)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if p.dim() == 2:
                p.normal_(0, 0.02)
            elif "q_norm" in name or "k_norm" in name:
                p.uniform_(0.25, 2.5)
    model.save_pretrained(tmp_path, safe_serialization=True)
    build_synthetic_tokenizer(1021).save_pretrained(tmp_path)
    args = argparse.Namespace(model=str(tmp_path), max_model_len=None, synthetic_weights=False, max_num_seqs=4,
                              max_num_batched_tokens=256, gpu_memory_utilization=0.05, seed=0, enable_lora=False)
    mc, path = _resolve_model(args)
    assert (mc.qk_norm, mc.vocab, mc.tie_word_embeddings, mc.head_dim, mc.max_model_len) == (True, 1021, True, 128, 1024)
    tok = load_tokenizer(str(path), mc.vocab)
    prompts = [_prompt(90, 1), [12, 13, 14, 1020]]
    assert [tok(synthetic_prompt(p), add_special_tokens=False)["input_ids"] for p in prompts] == prompts
    eng = _make_native_engine(args, mc, path, device=0)
    outs = eng.generate_sync(prompts, _sp(max_tokens=12, min_tokens=12))
    eng.close()
    sd = {k: v for k, v in model.state_dict().items() if "rotary" not in k and k != "lm_head.weight"}
    cfg = Qwen3Config(n_layers=2, hidden=256, n_q_heads=4, n_kv_heads=2, ffn=512, vocab=1021, rope_theta=1000000.0,
                      rms_eps=1e-6, max_model_len=1024, tie_word_embeddings=True)
    _check_greedy(cfg, sd, prompts, outs, 12)


def test_synthetic_qwen3_06b_preset_over_grpc():
    """`--model qwen3-0.6b --synthetic-weights` through loader.build_engine and the gRPC service: Generate returns the
    requested tokens, and GenerateStream with max_new_tokens = 10 yields 11 messages (the reference's own assertion: the
    input-token message, then one per token)"""
    import argparse
    import asyncio
    import threading

    import grpc

    from vllm_tgis_adapter_b200.engine.loader import build_engine
    from vllm_tgis_adapter_b200.engine.tokenizer import synthetic_prompt
    from vllm_tgis_adapter_b200.grpc import grpc_server
    from vllm_tgis_adapter_b200.grpc.pb import generation_pb2 as pb

    args = argparse.Namespace(model="qwen3-0.6b", max_model_len=2048, synthetic_weights=True, max_num_seqs=4,
                              max_num_batched_tokens=256, gpu_memory_utilization=0.2, seed=0, enable_lora=False,
                              tensor_parallel_size=1, device=0, tokenizer=None, max_new_tokens=64,
                              output_special_tokens=False, default_include_stop_seqs=True, disable_prompt_logprobs=False,
                              adapter_cache=None, prefix_store_path=None, host="127.0.0.1", grpc_port=0, ssl_keyfile=None,
                              ssl_certfile=None, ssl_ca_certs=None)
    loop, ready, box = asyncio.new_event_loop(), threading.Event(), {}

    def run():
        asyncio.set_event_loop(loop)

        async def main():
            box["engine"] = build_engine(args)
            box["engine"].start(loop)
            box["stop"] = asyncio.Event()
            server = await grpc_server.start_grpc_server(args, box["engine"], box["stop"])
            box["port"] = server.bound_port
            ready.set()
            await box["stop"].wait()
            await server.stop(0)
            box["engine"].shutdown()

        loop.run_until_complete(main())

    th = threading.Thread(target=run, daemon=True)
    th.start()
    assert ready.wait(180)
    try:
        with grpc.insecure_channel(f"127.0.0.1:{box['port']}") as ch:
            call = ch.unary_unary("/fmaas.GenerationService/Generate",
                                  request_serializer=pb.BatchedGenerationRequest.SerializeToString,
                                  response_deserializer=pb.BatchedGenerationResponse.FromString)
            params = pb.Parameters()
            params.stopping.max_new_tokens = params.stopping.min_new_tokens = 10
            prompts = [_prompt(80, 4, 151936), _prompt(9, 5, 151936)]
            resp = call(pb.BatchedGenerationRequest(model_id="m", params=params, requests=[
                pb.GenerationRequest(text=synthetic_prompt(p)) for p in prompts]), timeout=60)
            assert [r.generated_token_count for r in resp.responses] == [10, 10]
            assert [r.input_token_count for r in resp.responses] == [80, 9]
            stream = ch.unary_stream("/fmaas.GenerationService/GenerateStream",
                                     request_serializer=pb.SingleGenerationRequest.SerializeToString,
                                     response_deserializer=pb.GenerationResponse.FromString)
            sparams = pb.Parameters()
            sparams.stopping.max_new_tokens = 10
            chunks = list(stream(pb.SingleGenerationRequest(model_id="m", params=sparams, request=pb.GenerationRequest(
                text=synthetic_prompt(prompts[0]))), timeout=60))
            assert len(chunks) == 11 and chunks[0].input_token_count == 80
    finally:
        loop.call_soon_threadsafe(box["stop"].set)
        th.join(20)
    assert not th.is_alive()
