"""-m gpu: GPTBigCode (TGIS_ARCH_GPT_BIGCODE) on the engine: the GELU-tanh mode of opt_bias_act bit for bit against torch
CUDA (and ReLU / identity as before); both tiny presets and a 48-head multi-query engine against tests/gpt_bigcode_oracle.py
(greedy tokens, logprobs, ranks, top-n and prompt logprobs at chunks 48 and 2048); bit-identity under batching with
preemption, CUDA graphs and a prefix-cache hit; a save_pretrained checkpoint directory; the starcoderbase-1b preset over
gRPC; and the start-up refusals."""
import dataclasses
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from gpt_bigcode_oracle import CONFIGS, GPTBigCodeConfig, GPTBigCodeOracle, synthetic_weights

pytestmark = pytest.mark.gpu

_W = {}
# a 48-query-head multi-query stack (StarCoder-15B's group, head octets 6 x 8) small enough for the oracle
G48 = GPTBigCodeConfig(n_layers=2, hidden=48 * 128, n_heads=48, n_kv_heads=1, ffn=2048, vocab=1021)


@pytest.fixture(scope="module")
def g():
    import tgis_gpu_utils as gpu_utils

    return gpu_utils


def _cfg(name):
    return G48 if name == "g48" else CONFIGS[name]


def _weights(name):
    if name not in _W:
        _W[name] = synthetic_weights(_cfg(name), seed=9)
    return _W[name]


def _mc(name, **over):
    from vllm_tgis_adapter_b200.engine.core import PRESETS, ModelConfig

    if name == "g48":
        c = G48
        mc = ModelConfig(n_layers=c.n_layers, hidden=c.hidden, n_q_heads=c.n_heads, n_kv_heads=c.n_kv_heads, ffn=c.ffn,
                         vocab=c.vocab, rms_eps=c.ln_eps, max_model_len=2048, arch="gpt_bigcode",
                         tie_word_embeddings=True)
    else:
        mc = PRESETS[name]
    return dataclasses.replace(mc, **over)


def _engine(name, weights=None, max_model_len=2048, **kw):
    from vllm_tgis_adapter_b200.engine.core import NativeEngine

    kw.setdefault("max_num_seqs", 8)
    kw.setdefault("kv_cache_bytes", 32 << 20)
    eng = NativeEngine(_mc(name, max_model_len=max_model_len), **kw)
    eng.load_weights(weights or _weights(name))   # no lm_head.weight: tied
    return eng


def _sp(**kw):
    from vllm_tgis_adapter_b200.engine.core import make_sampling_params

    kw.setdefault("greedy", True)
    kw.setdefault("eos_token_id", 2)
    return make_sampling_params(**kw)


def _gen(eng, prompts, sp):
    outs = eng.generate_sync(prompts, sp)
    return [[(r.new_token, r.logprob, r.rank, tuple(r.topn)) for r in recs if r.new_token is not None] for recs in outs]


def _ulp(x):
    return 2.0 ** (math.floor(math.log2(max(abs(x), 1e-30))) - 7)


def _prompts(vocab, lens, seed):
    rng = np.random.RandomState(seed)
    return [rng.randint(3, vocab, size=n).tolist() for n in lens]


# ----------------------------------------------------------------------------------------------------- the kernel
@pytest.mark.parametrize("T,N", [(1, 2048), (37, 8192), (300, 24576)])
def test_gelu_tanh_mode_is_bit_exact_against_torch_cuda(g, T, N):
    """out = bf16(gelu_tanh(bf16(acc + b))) bit for bit against torch CUDA's F.gelu(approximate="tanh") on the bf16
    projection; ReLU (1) and identity (0) give the bits they gave before; another mode is refused"""
    gen = torch.Generator(device="cuda").manual_seed(T + N)
    acc = torch.randn(T, N, device="cuda", generator=gen) * 3.0
    acc[:, ::7] *= 30.0
    bias = (torch.randn(N, device="cuda", generator=gen) * 0.5).bfloat16()
    out = torch.empty(T, N, dtype=torch.bfloat16, device="cuda")
    y = (acc + bias.float()).bfloat16()
    want = {0: y, 1: torch.relu(acc + bias.float()).bfloat16(), 2: F.gelu(y, approximate="tanh")}
    assert want[2].dtype == torch.bfloat16
    for act, ref in want.items():
        out.fill_(7.0)
        assert g.lib().tgis_k_opt_bias_act(g.ptr(acc), g.ptr(bias), g.ptr(out), T, N, act) == 0, g.kerr()
        assert torch.equal(out, ref), (act, int((out != ref).sum()))
    assert g.lib().tgis_k_opt_bias_act(g.ptr(acc), g.ptr(bias), g.ptr(out), T, N, 3) != 0


# ----------------------------------------------------------------------------------------------------- the engine
def _check_greedy(cfg, weights, prompts, outs, n_new):
    """teacher-forced on the engine's tokens: a flip only inside a 2-ulp race, logprobs within 3 bf16 ulps of the top
    logit, rank 1 outside a race, the top-n ids and values against the oracle's"""
    ora = GPTBigCodeOracle(cfg, weights, device="cuda")
    flips = steps = 0
    for p, recs in zip(prompts, outs):
        assert len(recs) == n_new
        s = ora.new_seq()
        logits = ora.step([(s, p)])[0]
        for tok, lp_e, rank, topn in recs:
            lp = torch.log_softmax(logits, -1)
            top2 = torch.topk(logits, 2).values
            u, margin = _ulp(float(top2[0])), float(top2[0] - top2[1])
            steps += 1
            if tok != int(torch.argmax(logits)):
                assert margin <= 2 * u + 1e-6, (margin, u)
                flips += 1
            elif margin > 2 * u:
                assert rank == 1
            assert abs(lp_e - float(lp[tok])) <= 3 * u
            for tid, tlp in topn:
                assert abs(tlp - float(lp[tid])) <= 3 * u
            logits = ora.step([(s, [tok])])[0]
    assert flips <= steps // 10, (flips, steps)


@pytest.mark.parametrize("chunk", [48, 2048])
@pytest.mark.parametrize("name", ["gpt-bigcode-tiny", "gpt-bigcode-tiny-mha", "g48"])
def test_greedy_generation_matches_the_oracle(name, chunk):
    prompts = _prompts(1021, (5, 40, 130, 300, 17), seed=3)
    eng = _engine(name, max_batched_tokens=chunk)
    outs = _gen(eng, prompts, _sp(max_tokens=16, min_tokens=16, num_logprobs=3))
    st = eng.status()
    eng.close()
    assert st.errored == 0
    _check_greedy(_cfg(name), _weights(name), prompts, outs, 16)


@pytest.mark.parametrize("chunk", [48, 2048])
@pytest.mark.parametrize("name", ["gpt-bigcode-tiny", "gpt-bigcode-tiny-mha", "g48"])
def test_prompt_logprobs_match_the_oracle(name, chunk):
    prompts = _prompts(1021, (150, 9, 37), seed=5)
    eng = _engine(name, max_batched_tokens=chunk)
    outs = eng.generate_sync(prompts, _sp(max_tokens=2, num_logprobs=1, prompt_logprobs=2))
    eng.close()
    ora = GPTBigCodeOracle(_cfg(name), _weights(name), device="cuda")
    for p, recs in zip(prompts, outs):
        prec = sorted([r for r in recs if r.prompt_pos >= 1], key=lambda r: r.prompt_pos)
        assert [r.prompt_pos for r in prec] == list(range(1, len(p)))
        logits = ora.step([(ora.new_seq(), p)], want_all_logits=True)
        lp = torch.log_softmax(logits, -1)
        for r in prec:
            u = _ulp(float(logits[r.prompt_pos - 1].abs().max()))
            assert r.token_id == p[r.prompt_pos]
            assert abs(r.logprob - float(lp[r.prompt_pos - 1, r.token_id])) <= 3 * u


def test_batch_invariance_with_preemption_and_cuda_graphs():
    """a prompt alone vs in a crowded batch over a KV cache so small that sequences are preempted and recomputed, and
    CUDA graphs on vs off: the same tokens and logprobs, bit for bit"""
    name = "gpt-bigcode-tiny"
    prompts = _prompts(1021, (60, 90, 40, 75, 33, 120), seed=11)
    sp = _sp(max_tokens=40, min_tokens=40, num_logprobs=2)
    solo_eng = _engine(name, max_model_len=512, max_num_seqs=1, max_batched_tokens=512)
    solo = _gen(solo_eng, prompts[:1], sp)
    solo_eng.close()
    # 2 layers * 1 kv head * 32 tok * 128 dims * 2 B * 2 (K, V) = 32 KiB per block; 17 blocks = 544 tokens for 6 sequences
    crowd_eng = _engine(name, max_model_len=512, max_num_seqs=6, max_batched_tokens=64, kv_cache_bytes=17 * 32768)
    crowd = _gen(crowd_eng, prompts, sp)
    st = crowd_eng.status()
    crowd_eng.close()
    assert st.total_blocks == 17 and st.preemptions > 0 and st.errored == 0
    assert crowd[0] == solo[0] and all(len(c) == 40 for c in crowd)
    res = {}
    for graphs in (True, False):
        eng = _engine(name, use_cuda_graphs=graphs)
        res[graphs] = _gen(eng, prompts[:3], _sp(max_tokens=24, min_tokens=24, num_logprobs=2))
        st = eng.status()
        eng.close()
        assert (st.graph_launches > 0) == graphs
    assert res[True] == res[False]


@pytest.mark.parametrize("name", ["gpt-bigcode-tiny", "g48"])
def test_prefix_cache_hit_takes_the_split_context_kernel_and_changes_nothing(name):
    """P = 1100 shared tokens + a 100-token tail; with P's prefix cached (1088 tokens, 34 blocks), P's prefill is a short
    suffix over > 1024 cached tokens (the split-context kernel on head chunks).  Ids and logprobs equal a cold engine
    chunked at the same boundary, bit for bit."""
    P = _prompts(1021, (1188,), seed=1)[0]
    X = P[:1088] + _prompts(1021, (100,), seed=2)[0]
    cold = _engine(name, max_batched_tokens=1088, enable_prefix_caching=True)
    want = _gen(cold, [P], _sp(num_logprobs=2))
    cold.close()
    eng = _engine(name, max_batched_tokens=1088, enable_prefix_caching=True)
    _gen(eng, [X], _sp())
    q0, h0, _ = eng.prefix_cache_stats()
    got = _gen(eng, [P], _sp(num_logprobs=2))
    q1, h1, _ = eng.prefix_cache_stats()
    eng.close()
    assert h0 == 0 and q1 - q0 == len(P) and h1 - h0 == 1088
    assert got == want


def test_hf_checkpoint_directory_loads_and_follows_the_oracle(tmp_path):
    """GPTBigCodeForCausalLM.save_pretrained of the tiny stacks (multi-query and multi-head: c_attn's row orders differ)
    -> config.json mapping + safetensors loading -> the same tokens as the weights loaded directly"""
    import sys
    from pathlib import Path

    from transformers import GPTBigCodeForCausalLM

    sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "scripts"))
    from gen_gpt_bigcode_golden import hf_config
    from vllm_tgis_adapter_b200.engine.core import NativeEngine
    from vllm_tgis_adapter_b200.engine.loader import load_safetensors_dir, model_config_from_hf

    for name in ("gpt-bigcode-tiny", "gpt-bigcode-tiny-mha"):
        cfg = dataclasses.replace(_cfg(name), max_model_len=2048)
        d = tmp_path / name
        model = GPTBigCodeForCausalLM(hf_config(cfg)).to(torch.bfloat16)
        model.load_state_dict(_weights(name), strict=False)
        model.tie_weights()
        model.save_pretrained(d, safe_serialization=True)
        mc = model_config_from_hf(d, None)
        assert mc == _mc(name)
        prompts = _prompts(1021, (70, 9), seed=17)
        sp = _sp(max_tokens=12, min_tokens=12, num_logprobs=1)
        eng = NativeEngine(mc, max_num_seqs=4, kv_cache_bytes=32 << 20)
        load_safetensors_dir(eng, d)
        from_dir = _gen(eng, prompts, sp)
        eng.close()
        eng = _engine(name)
        direct = _gen(eng, prompts, sp)
        eng.close()
        assert from_dir == direct, name


def test_start_up_refusals():
    from vllm_tgis_adapter_b200.engine.core import EngineError, NativeEngine

    kw = dict(max_num_seqs=2, kv_cache_bytes=8 << 20)
    bad = [(dict(n_q_heads=65, hidden=65 * 128), "at most 64 query heads"),
           (dict(n_kv_heads=2), "n_kv_heads must be 1"),
           (dict(head_dim=64, hidden=12 * 64), "head_dim must be 128"),
           (dict(hidden=1024), "hidden must be n_q_heads"),
           (dict(sliding_window=40), "sliding-window")]
    for over, msg in bad:
        with pytest.raises(EngineError, match=msg):
            NativeEngine(_mc("gpt-bigcode-tiny", **over), **kw)
    # groups above 8 stay refused for the Llama stack (OPT has n_kv_heads = n_q_heads)
    with pytest.raises(EngineError, match="GQA group size must be 1 to 8"):
        NativeEngine(dataclasses.replace(_mc("gpt-bigcode-tiny"), arch="llama"), **kw)
    # a checkpoint with a tensor missing does not start
    eng = NativeEngine(_mc("gpt-bigcode-tiny"), **kw)
    eng.load_weights({k: v for k, v in _weights("gpt-bigcode-tiny").items() if k != "transformer.h.1.mlp.c_fc.bias"})
    with pytest.raises(EngineError, match="GPTBigCode checkpoint incomplete: 27 of 28"):
        eng.start()
    eng.close()
    # wpe shorter than max_model_len is refused
    eng = NativeEngine(_mc("gpt-bigcode-tiny"), **kw)
    with pytest.raises(EngineError, match="shape mismatch for transformer.wpe.weight"):
        eng.load_weight("transformer.wpe.weight", torch.zeros(100, 1536, dtype=torch.bfloat16))
    eng.close()


def test_starcoderbase_1b_preset_over_grpc():
    """`--model starcoderbase-1b --synthetic-weights` through loader.build_engine and the gRPC service"""
    import argparse
    import asyncio
    import threading

    import grpc

    from vllm_tgis_adapter_b200.engine.loader import build_engine
    from vllm_tgis_adapter_b200.engine.tokenizer import synthetic_prompt
    from vllm_tgis_adapter_b200.grpc import grpc_server
    from vllm_tgis_adapter_b200.grpc.pb import generation_pb2 as pb

    args = argparse.Namespace(model="starcoderbase-1b", max_model_len=2048, synthetic_weights=True, max_num_seqs=4,
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
    assert ready.wait(300), "server did not come up"
    try:
        with grpc.insecure_channel(f"127.0.0.1:{box['port']}") as ch:
            call = ch.unary_unary("/fmaas.GenerationService/Generate",
                                  request_serializer=pb.BatchedGenerationRequest.SerializeToString,
                                  response_deserializer=pb.BatchedGenerationResponse.FromString)
            params = pb.Parameters()
            params.stopping.max_new_tokens = params.stopping.min_new_tokens = 10
            prompts = _prompts(49152, (80, 9), seed=19)
            resp = call(pb.BatchedGenerationRequest(model_id="m", params=params, requests=[
                pb.GenerationRequest(text=synthetic_prompt(p)) for p in prompts]), timeout=120)
            assert [r.generated_token_count for r in resp.responses] == [10, 10]
            assert [r.input_token_count for r in resp.responses] == [80, 9]
    finally:
        loop.call_soon_threadsafe(box["stop"].set)
        th.join(60)
    assert not th.is_alive()
