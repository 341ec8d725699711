"""-m gpu: Qwen2 / Qwen2.5.  The RoPE + KV writer on the qkv GEMM's fp32 accumulators with the bias added before the one
rounding (rope_kvwrite_kernel<D, false, BIAS>), bit for bit against a torch restatement of its rounding points and against
opt_bias_act followed by the plain writer (the LoRA steps' sequence); the engine on the qwen2-tiny (GQA group 6, 128-dim
heads) and qwen2-tiny-hd64 (group 7, 64-dim heads) presets against tests/qwen2_oracle.py with the bars of
tests/test_qwen3_gpu.py (greedy, prompt logprobs, LoRA); a Qwen2 engine with zero biases against the Llama engine on
the same weights; bit-identity under batching with preemption, CUDA graphs and prefix-cache hits; the start-up refusals;
a save_pretrained checkpoint directory; and the qwen2.5-0.5b and qwen2.5-7b presets over gRPC."""
import dataclasses

import numpy as np
import pytest
import torch

from qwen2_oracle import CONFIGS, Qwen2Oracle, synthetic_weights
from test_qwen3_gpu import _prompt, _sp, _ulp
from tgis_gpu_utils import paged_k_cache as k_cache_from_dense, paged_v_cache as v_cache_from_dense

pytestmark = pytest.mark.gpu

PRESETS_UNDER_TEST = ["qwen2-tiny", "qwen2-tiny-hd64"]
_W = {}


@pytest.fixture(scope="module")
def g():
    import tgis_gpu_utils as gpu_utils

    return gpu_utils


def _cfg(preset="qwen2-tiny", **over):
    return dataclasses.replace(CONFIGS[preset], **over)


def _mc(preset="qwen2-tiny", **over):
    from vllm_tgis_adapter_b200.engine.core import PRESETS

    return dataclasses.replace(PRESETS[preset], **over)


def _weights(preset="qwen2-tiny"):
    if preset not in _W:
        _W[preset] = synthetic_weights(_cfg(preset), seed=8)
    return _W[preset]


def _engine(preset="qwen2-tiny", max_model_len=2048, weights=None, mc=None, **kw):
    from oracle.llama_oracle import rope_table
    from vllm_tgis_adapter_b200.engine.core import NativeEngine

    kw.setdefault("max_num_seqs", 8)
    kw.setdefault("kv_cache_bytes", 32 << 20)
    eng = NativeEngine(mc or _mc(preset, max_model_len=max_model_len), **kw)
    eng.load_weights(weights or _weights(preset))          # no lm_head.weight: tied
    eng.load_weight("tgis.rope_cos_sin", rope_table(_cfg(preset, max_model_len=max_model_len)))
    return eng


def _gen(eng, prompts, sp):
    outs = eng.generate_sync(prompts, sp)
    return [[(r.new_token, r.logprob, r.rank, tuple(r.topn)) for r in recs if r.new_token is not None] for recs in outs]


def _check_greedy(cfg, weights, prompts, outs, n_new):
    """teacher-forced on the engine's tokens: a flip only inside a 2-ulp race, logprobs within 3 bf16 ulps of the top
    logit, rank 1 outside a race, the top-n ids and values against the oracle's (the bars of tests/test_qwen3_gpu.py)"""
    ora = Qwen2Oracle(cfg, weights, device="cuda")
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


# ----------------------------------------------------------------------------------------------------- the kernel
POISON = -77.5   # a bf16 value no write produces here: every cache slot the writer must not touch keeps it


def _restate(acc, bias, positions, table, n_q, n_kv, D):
    """rope_kvwrite_kernel<D, false, BIAS> in torch: x = bf16(acc + bias) (fp32 add, one rounding), then the bf16
    rotation of the q and k heads (every product rounded, as the plain writer and the oracle's _rope do); v = x."""
    T = acc.shape[0]
    x = (acc.view(T, -1, D) + bias.float().view(1, -1, D)).bfloat16()
    half = D // 2
    cs = table[torch.from_numpy(positions).long().to(acc.device)]
    cos, sin = cs[:, None, :half], cs[:, None, half:]
    qk = x[:, :n_q + n_kv]
    x1, x2 = qk[..., :half], qk[..., half:]
    rot = torch.cat([x1 * cos - x2 * sin, x2 * cos + x1 * sin], dim=-1)
    return torch.cat([rot, x[:, n_q + n_kv:]], dim=1)


def _caches(n_blocks, n_kv, D):
    kc = torch.full((n_blocks, n_kv, D // 8, 32, 8), POISON, dtype=torch.bfloat16, device="cuda")
    vc = torch.full((n_blocks, n_kv, 32, D // 8, 8), POISON, dtype=torch.bfloat16, device="cuda")
    return kc, vc


def _writer_case(T, n_q, n_kv, D, seed):
    nh = n_q + 2 * n_kv
    gen = torch.Generator(device="cuda").manual_seed(seed)
    acc = torch.randn(T, nh * D, device="cuda", generator=gen) * 0.7
    acc[:, ::5] *= 40.0                                    # some accumulators far above the bias
    bias = torch.randn(nh * D, device="cuda", generator=gen) * 0.5
    bias[(n_q * D)::13] = 24.0                             # k / v biases far above the projection's scale
    bias = bias.bfloat16()
    max_pos = 8192
    table = (torch.rand(max_pos, D, device="cuda", generator=gen) * 2 - 1).bfloat16()
    rs = np.random.RandomState(seed)
    positions = rs.randint(0, max_pos, size=T).astype(np.int32)
    positions[0] = max_pos - 1
    n_blocks = (T + 31) // 32 + 3
    slots = rs.permutation(n_blocks * 32)[:T].astype(np.int32)
    slots[rs.rand(T) < 0.1] = -1             # "do not cache" rows
    if T > 1:
        slots[1] = -1
    return acc, bias, table, positions, slots, n_blocks


WRITER_HEADS = [(128, 6, 1), (128, 28, 4), (64, 14, 2), (64, 7, 1)]   # tiny, 7B, 0.5B, tiny-hd64


@pytest.mark.parametrize("D,n_q,n_kv", WRITER_HEADS, ids=["tiny", "7b", "0.5b", "tiny-hd64"])
@pytest.mark.parametrize("T", [1, 31, 32, 257, 2048])
def test_bias_writer_is_bit_exact_against_its_rounding_points(g, D, n_q, n_kv, T):
    acc, bias, table, positions, slots, n_blocks = _writer_case(T, n_q, n_kv, D, seed=T * 100 + n_q + D)
    assert T == 1 or (positions > 4096).any()
    nh = n_q + 2 * n_kv
    qkv = torch.full((T, nh, D), POISON, dtype=torch.bfloat16, device="cuda")
    kc, vc = _caches(n_blocks, n_kv, D)
    rc = g.lib().tgis_k_rope_kv_bias(D, g.ptr(acc), g.ptr(bias), g.ptr(qkv), g.i32p(positions), g.i32p(slots),
                                     g.ptr(table), g.ptr(kc), g.ptr(vc), T, n_q, n_kv, 1, None)
    assert rc == 0, g.kerr()
    want = _restate(acc, bias, positions, table, n_q, n_kv, D)
    assert torch.equal(qkv, want)
    k_pool = torch.full((n_blocks * 32, n_kv, D), POISON, dtype=torch.bfloat16, device="cuda")
    v_pool = k_pool.clone()
    live = torch.from_numpy(slots >= 0).cuda()
    sl = torch.from_numpy(slots).long().cuda()[live]
    k_pool[sl] = want[live][:, n_q:n_q + n_kv]
    v_pool[sl] = want[live][:, n_q + n_kv:]
    assert torch.equal(kc, k_cache_from_dense(k_pool, n_blocks)) and torch.equal(vc, v_cache_from_dense(v_pool, n_blocks))
    # the rounding point matters on these inputs: rounding acc to bf16 before the bias add gives other bits
    twice = _restate(acc.bfloat16().float(), bias, positions, table, n_q, n_kv, D)
    assert not torch.equal(twice, want)


@pytest.mark.parametrize("D,n_q,n_kv", WRITER_HEADS, ids=["tiny", "7b", "0.5b", "tiny-hd64"])
@pytest.mark.parametrize("T", [1, 257, 2048])
def test_bias_writer_equals_bias_kernel_then_plain_writer(g, D, n_q, n_kv, T):
    """the fused writer against the two-kernel sequence of the engine's LoRA steps: opt_bias_act (relu 0) into qkv, then
    the plain writer in place -- qkv and both caches bit for bit"""
    acc, bias, table, positions, slots, n_blocks = _writer_case(T, n_q, n_kv, D, seed=T + 7 * n_q + D)
    nh = n_q + 2 * n_kv
    fused = torch.full((T, nh, D), POISON, dtype=torch.bfloat16, device="cuda")
    kc1, vc1 = _caches(n_blocks, n_kv, D)
    assert g.lib().tgis_k_rope_kv_bias(D, g.ptr(acc), g.ptr(bias), g.ptr(fused), g.i32p(positions), g.i32p(slots),
                                       g.ptr(table), g.ptr(kc1), g.ptr(vc1), T, n_q, n_kv, 3, None) == 0, g.kerr()
    two = torch.full((T, nh, D), POISON, dtype=torch.bfloat16, device="cuda")
    kc2, vc2 = _caches(n_blocks, n_kv, D)
    assert g.lib().tgis_k_opt_bias_act(g.ptr(acc), g.ptr(bias), g.ptr(two), T, nh * D, 0) == 0, g.kerr()
    assert g.lib().tgis_k_rope_kv_hd(D, g.ptr(two), g.i32p(positions), g.i32p(slots), g.ptr(table), g.ptr(kc2),
                                     g.ptr(vc2), T, n_q, n_kv) == 0, g.kerr()
    assert torch.equal(fused, two) and torch.equal(kc1, kc2) and torch.equal(vc1, vc2)


# ----------------------------------------------------------------------------------------------------- the engine
@pytest.mark.parametrize("preset", PRESETS_UNDER_TEST)
@pytest.mark.parametrize("chunk", [2048, 48])
def test_greedy_generation_matches_the_qwen2_oracle(preset, chunk):
    prompts = [_prompt(n, 10 + n) for n in (5, 70, 129, 300, 700)]
    prompts[0][-1] = 1020                      # the last token id of the odd vocabulary
    n_new = 16
    eng = _engine(preset, max_batched_tokens=chunk)
    outs = eng.generate_sync(prompts, _sp(max_tokens=n_new, min_tokens=n_new, num_logprobs=3))
    st = eng.status()
    eng.close()
    assert st.errored == 0 and st.graph_launches > 0
    _check_greedy(_cfg(preset), _weights(preset), prompts, outs, n_new)


@pytest.mark.parametrize("preset", PRESETS_UNDER_TEST)
@pytest.mark.parametrize("chunk", [2048, 48])
def test_prompt_logprobs_match_the_qwen2_oracle(preset, chunk):
    prompts = [_prompt(n, 70 + n) for n in (100, 9, 37)]
    eng = _engine(preset, max_batched_tokens=chunk)
    outs = eng.generate_sync(prompts, _sp(max_tokens=2, min_tokens=0, prompt_logprobs=3))
    eng.close()
    ora = Qwen2Oracle(_cfg(preset), _weights(preset), device="cuda")
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


@pytest.mark.parametrize("preset", PRESETS_UNDER_TEST)
def test_zero_biases_give_the_llama_engine_bit_for_bit(preset):
    """the bias path is the Llama path plus the bias: bf16(acc + 0) = bf16(acc), so a Qwen2 engine with all-zero biases
    gives the Llama engine's tokens and logprobs (which takes the GEMM-fused RoPE epilogue at decode)"""
    w = {k: (torch.zeros_like(v) if k.endswith("_proj.bias") else v) for k, v in _weights(preset).items()}
    prompts = [_prompt(n, 300 + n) for n in (5, 70, 129, 300)]
    sp = _sp(max_tokens=24, min_tokens=24, num_logprobs=3)
    res = {}
    for bias in (True, False):
        ww = w if bias else {k: v for k, v in w.items() if not k.endswith("_proj.bias")}
        eng = _engine(preset, weights=ww, mc=_mc(preset, qkv_bias=bias))
        res[bias] = _gen(eng, prompts, sp)
        eng.close()
    assert res[True] == res[False]


def test_batch_invariance_with_preemption():
    """a prompt alone vs in a crowded batch over a KV cache so small that sequences are preempted and recomputed: the same
    tokens and logprobs, bit for bit"""
    prompts = [_prompt(n, n) for n in (60, 90, 40, 75, 33, 120)]
    sp = _sp(max_tokens=40, min_tokens=40)
    solo_eng = _engine(max_model_len=512, max_num_seqs=1, max_batched_tokens=512)
    solo = _gen(solo_eng, prompts[:1], sp)
    solo_eng.close()
    # 2 layers * 1 kv head * 32 tok * 128 dims * 2 B * 2 (K, V) = 32 KiB per block; 17 blocks = 544 tokens for 6 sequences
    crowd_eng = _engine(max_model_len=512, max_num_seqs=6, max_batched_tokens=64, kv_cache_bytes=17 * 32768)
    crowd = _gen(crowd_eng, prompts, sp)
    st = crowd_eng.status()
    crowd_eng.close()
    assert st.total_blocks == 17 and st.preemptions > 0 and st.errored == 0
    assert crowd[0] == solo[0]
    assert all(len(c) == 40 for c in crowd)


@pytest.mark.parametrize("preset", PRESETS_UNDER_TEST)
def test_cuda_graphs_on_and_off_give_identical_ids(preset):
    prompts = [_prompt(n, 50 + n) for n in (20, 130, 260)]
    res = {}
    for graphs in (True, False):
        eng = _engine(preset, use_cuda_graphs=graphs)
        res[graphs] = _gen(eng, prompts, _sp(max_tokens=24, min_tokens=24, num_logprobs=2))
        st = eng.status()
        eng.close()
        assert (st.graph_launches > 0) == graphs
    assert res[True] == res[False]


@pytest.mark.parametrize("preset", PRESETS_UNDER_TEST)
def test_prefix_cache_hit_takes_the_split_context_kernel_and_changes_nothing(preset):
    """P = 1024 shared tokens + a 100-token tail; with P's prefix cached, P's prefill is a 100-row suffix over 1024 cached
    tokens (the split-context kernel).  Ids and logprobs equal a cold engine chunked at the same boundary, bit for bit."""
    P = _prompt(1124, 1)
    X = P[:1024] + _prompt(100, 2)
    cold = _engine(preset, max_batched_tokens=1024, enable_prefix_caching=True)
    want = _gen(cold, [P], _sp())
    cold.close()
    eng = _engine(preset, max_batched_tokens=1024, enable_prefix_caching=True)
    _gen(eng, [X], _sp())
    q0, h0, _ = eng.prefix_cache_stats()
    got = _gen(eng, [P], _sp())
    q1, h1, _ = eng.prefix_cache_stats()
    eng.close()
    assert h0 == 0 and q1 - q0 == len(P) and h1 - h0 == 1024
    assert got == want


def test_lora_follows_the_oracle_and_leaves_base_requests_untouched(tmp_path):
    """adapter deltas land on the biased q / k / v, before RoPE (vLLM: qkv_proj's biased output carries the delta)"""
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
    ora = Qwen2Oracle(cfg, _weights(), device="cuda")
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
    with pytest.raises(EngineError, match="tgis_engine_create failed: .*OPT"):
        NativeEngine(dataclasses.replace(PRESETS["opt-tiny"], qkv_bias=True), **kw)
    with pytest.raises(EngineError, match=r"Qwen2\) is supported on a single GPU only"):
        NativeEngine(_mc(), tp_size=2, tp_rank=0, nccl_id=bytes(128), shm_name="/tgis_test_unused", **kw)
    with pytest.raises(EngineError, match="head_dim 64.*LoRA"):
        NativeEngine(_mc("qwen2-tiny-hd64"), max_loras=1, **kw)
    with pytest.raises(EngineError, match="tgis_engine_create failed: .*q/k norm"):
        NativeEngine(_mc(qk_norm=True), **kw)
    # a missing vector: start fails and names the layer and the tensor
    eng = NativeEngine(_mc(), **kw)
    w = dict(_weights())
    del w["model.layers.1.self_attn.k_proj.bias"]
    eng.load_weights(w)
    with pytest.raises(EngineError, match=r"layer 1 has no model\.layers\.1\.self_attn\.k_proj\.bias"):
        eng.start()
    with pytest.raises(EngineError, match="layer 1"):
        eng.run_until_idle()
    # a wrong length is an error, and does not count as loaded
    with pytest.raises(EngineError, match="shape mismatch"):
        eng.load_weight("model.layers.1.self_attn.k_proj.bias", torch.ones(64, dtype=torch.bfloat16))
    with pytest.raises(EngineError, match="layer 1"):
        eng.start()
    eng.load_weight("model.layers.1.self_attn.k_proj.bias", _weights()["model.layers.1.self_attn.k_proj.bias"])
    eng.start()
    eng.close()
    # the bias names are not names a Llama engine knows, as before
    eng = NativeEngine(_mc(qkv_bias=False), **kw)
    with pytest.raises(EngineError, match="unknown layer weight model.layers.0.self_attn.q_proj.bias"):
        eng.load_weight("model.layers.0.self_attn.q_proj.bias", torch.ones(768, dtype=torch.bfloat16))
    eng.close()


def test_hf_checkpoint_directory_loads_and_follows_the_oracle(tmp_path):
    """Qwen2ForCausalLM.save_pretrained (bf16, tied, GQA group 6, odd vocabulary, random biases) with the synthetic
    tokenizer saved beside it: the loader's config mapping, the safetensors reader and the tokenizer; greedy tokens
    follow the oracle"""
    import argparse

    from transformers import Qwen2Config as HFQwen2Config
    from transformers import Qwen2ForCausalLM

    from vllm_tgis_adapter_b200.engine.loader import _make_native_engine, _resolve_model
    from vllm_tgis_adapter_b200.engine.tokenizer import build_synthetic_tokenizer, load_tokenizer, synthetic_prompt

    hf_cfg = HFQwen2Config(vocab_size=1021, hidden_size=768, intermediate_size=1024, num_hidden_layers=2,
                           num_attention_heads=6, num_key_value_heads=1, rms_norm_eps=1e-6,
                           max_position_embeddings=1024, tie_word_embeddings=True,
                           rope_parameters={"rope_type": "default", "rope_theta": 1000000.0})
    torch.manual_seed(0)
    model = Qwen2ForCausalLM(hf_cfg).to(torch.bfloat16)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if p.dim() == 2:
                p.normal_(0, 0.02)
            elif name.endswith("_proj.bias"):
                p.normal_(0, 1.0)
    model.save_pretrained(tmp_path, safe_serialization=True)
    build_synthetic_tokenizer(1021).save_pretrained(tmp_path)
    args = argparse.Namespace(model=str(tmp_path), max_model_len=None, synthetic_weights=False, max_num_seqs=4,
                              max_num_batched_tokens=256, gpu_memory_utilization=0.05, seed=0, enable_lora=False)
    mc, path = _resolve_model(args)
    assert (mc.qkv_bias, mc.vocab, mc.tie_word_embeddings, mc.head_dim, mc.max_model_len) == (True, 1021, True, 128, 1024)
    tok = load_tokenizer(str(path), mc.vocab)
    prompts = [_prompt(90, 1), [12, 13, 14, 1020]]
    assert [tok(synthetic_prompt(p), add_special_tokens=False)["input_ids"] for p in prompts] == prompts
    eng = _make_native_engine(args, mc, path, device=0)
    outs = eng.generate_sync(prompts, _sp(max_tokens=12, min_tokens=12))
    eng.close()
    sd = {k: v for k, v in model.state_dict().items() if "rotary" not in k and k != "lm_head.weight"}
    cfg = _cfg(max_model_len=1024)
    _check_greedy(cfg, sd, prompts, outs, 12)


@pytest.mark.parametrize("preset", ["qwen2.5-0.5b", "qwen2.5-7b"])
def test_synthetic_qwen25_preset_over_grpc(preset):
    """`--model <preset> --synthetic-weights` through loader.build_engine and the gRPC service: Generate returns the
    requested tokens, and GenerateStream with max_new_tokens = 10 yields 11 messages (the input-token message, then one
    per token)"""
    import argparse
    import asyncio
    import threading

    import grpc

    from vllm_tgis_adapter_b200.engine.loader import build_engine
    from vllm_tgis_adapter_b200.engine.tokenizer import synthetic_prompt
    from vllm_tgis_adapter_b200.grpc import grpc_server
    from vllm_tgis_adapter_b200.grpc.pb import generation_pb2 as pb

    args = argparse.Namespace(model=preset, max_model_len=2048, synthetic_weights=True, max_num_seqs=4,
                              max_num_batched_tokens=256, gpu_memory_utilization=0.3, seed=0, enable_lora=False,
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
    assert ready.wait(300)
    vocab = 151936 if preset == "qwen2.5-0.5b" else 152064
    try:
        with grpc.insecure_channel(f"127.0.0.1:{box['port']}") as ch:
            call = ch.unary_unary("/fmaas.GenerationService/Generate",
                                  request_serializer=pb.BatchedGenerationRequest.SerializeToString,
                                  response_deserializer=pb.BatchedGenerationResponse.FromString)
            params = pb.Parameters()
            params.stopping.max_new_tokens = params.stopping.min_new_tokens = 10
            prompts = [_prompt(80, 4, vocab), _prompt(9, 5, vocab)]
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
