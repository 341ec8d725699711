"""-m gpu: the engine end to end on a Llama-3.2-style stack (preset llama-tiny-hd64: native 64-dim heads, tied
embeddings, rope_type llama3 scaling with original_max_position_embeddings 64, so every prompt here runs past it), against
tests/llama3_oracle.py with the ulp bars of tests/test_parity_gpu.py; batch invariance with preemption, prefix caching and
CUDA graphs on 64-dim heads; the KV block count at half the head size; and the start-up refusals."""
import dataclasses
import math

import numpy as np
import pytest
import torch

from llama3_oracle import CONFIGS, Llama3Oracle, rope_table, synthetic_weights

pytestmark = pytest.mark.gpu

_W = {}


def _cfg(**over):
    return dataclasses.replace(CONFIGS["llama-tiny-hd64"], **over)


def _mc(**over):
    from vllm_tgis_adapter_b200.engine.core import PRESETS

    return dataclasses.replace(PRESETS["llama-tiny-hd64"], **over)


def _weights():
    if "w" not in _W:
        _W["w"] = synthetic_weights(_cfg(), seed=6)
    return _W["w"]


def _engine(max_model_len=2048, table=True, **kw):
    from vllm_tgis_adapter_b200.engine.core import NativeEngine

    kw.setdefault("max_num_seqs", 8)
    kw.setdefault("kv_cache_bytes", 32 << 20)
    eng = NativeEngine(_mc(max_model_len=max_model_len), **kw)
    eng.load_weights(_weights())          # no lm_head.weight: tied
    if table:
        eng.load_weight("tgis.rope_cos_sin", rope_table(_cfg(max_model_len=max_model_len)))
    return eng


def _sp(**kw):
    from vllm_tgis_adapter_b200.engine.core import make_sampling_params

    d = dict(greedy=True, max_tokens=16, min_tokens=16, num_logprobs=1, eos_token_id=2)
    d.update(kw)
    return make_sampling_params(**d)


def _gen(eng, prompts, sp):
    outs = eng.generate_sync(prompts, sp)
    return [[(r.new_token, r.logprob) for r in recs if r.new_token is not None] for recs in outs]


def _prompt(n, seed):
    return np.random.RandomState(seed).randint(3, 1024, size=n).tolist()


def _ulp(x: float) -> float:
    return 2.0 ** (math.floor(math.log2(max(abs(x), 1e-6))) - 7)


@pytest.mark.parametrize("chunk", [2048, 48])
def test_greedy_generation_matches_the_llama3_oracle(chunk):
    """tokens and logprobs against the oracle, teacher-forced on the engine's tokens: a flip only inside a 2-ulp race,
    logprobs within 3 bf16 ulps of the top logit; whole-prompt and chunked prefill (48 tokens per step); prompts of 5 to
    700 tokens, all but the first past original_max_position_embeddings = 64 after a few steps"""
    cfg = _cfg()
    prompts = [_prompt(n, 10 + n) for n in (5, 70, 129, 300, 700)]
    n_new = 16
    eng = _engine(max_batched_tokens=chunk)
    outs = eng.generate_sync(prompts, _sp(max_tokens=n_new, min_tokens=n_new))
    st = eng.status()
    eng.close()
    assert st.errored == 0 and st.graph_launches > 0
    ora = Llama3Oracle(cfg, _weights(), device="cuda")
    flips = steps = 0
    max_ulps = 0.0
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
            max_ulps = max(max_ulps, abs(r.logprob - float(lp[r.new_token])) / u)
            logits = ora.step([(s, [r.new_token])])[0]
    print(f"chunk {chunk}: {flips} flips in {steps} steps, max logprob diff {max_ulps:.2f} ulp")
    assert flips <= steps // 10 and max_ulps <= 3.0, (flips, steps, max_ulps)


def test_batch_invariance_and_preemption_at_64_dim_heads():
    """a prompt alone vs in a crowded batch over a KV cache so small that sequences are preempted and recomputed: the
    same tokens and logprobs, bit for bit (fixed 128-token splits, split-order merge, deterministic GEMM schedule)"""
    prompts = [_prompt(n, n) for n in (60, 90, 40, 75, 33, 120)]
    sp = _sp(max_tokens=40, min_tokens=40)
    solo_eng = _engine(max_model_len=512, max_num_seqs=1, max_batched_tokens=512)
    solo = _gen(solo_eng, prompts[:1], sp)
    solo_eng.close()
    # 2 layers * 2 kv heads * 32 tok * 64 dims * 2 B * 2 (K, V) = 32 KiB per block; 17 blocks = 544 tokens for 6 sequences
    crowd_eng = _engine(max_model_len=512, max_num_seqs=6, max_batched_tokens=64, kv_cache_bytes=17 * 32768)
    crowd = _gen(crowd_eng, prompts, sp)
    st = crowd_eng.status()
    crowd_eng.close()
    assert st.total_blocks == 17 and st.preemptions > 0 and st.errored == 0
    assert [t for t, _ in crowd[0]] == [t for t, _ in solo[0]]
    assert all(len(c) == 40 for c in crowd)


def test_prefix_cache_hit_takes_the_split_context_kernel_and_changes_nothing():
    """P = 1024 shared tokens + a 100-token tail.  With caching on and the prefix already served, P's prefill is a
    100-row suffix over 1024 cached tokens: the split-context kernel's shape (q_len <= 128 over >= 1024).  Ids and
    logprobs equal a cold engine whose prefill is chunked at the same boundary, bit for bit; with caching off (the
    suffix on the ordinary prefill kernel) the ids are the same."""
    P = _prompt(1124, 1)
    X = P[:1024] + _prompt(100, 2)
    cold = _engine(max_batched_tokens=1024, enable_prefix_caching=True)
    want = _gen(cold, [P], _sp())
    cold.close()
    off = _engine(max_batched_tokens=1024)
    assert [[t for t, _ in r] for r in _gen(off, [P], _sp())] == [[t for t, _ in r] for r in want]
    off.close()
    eng = _engine(max_batched_tokens=1024, enable_prefix_caching=True)
    _gen(eng, [X], _sp())
    q0, h0, _ = eng.prefix_cache_stats()
    got = _gen(eng, [P], _sp())
    q1, h1, _ = eng.prefix_cache_stats()
    eng.close()
    assert h0 == 0 and q1 - q0 == len(P) and h1 - h0 == 1024   # the suffix: 100 rows over 1024 cached tokens
    assert got == want


def test_cuda_graphs_on_and_off_give_identical_ids():
    prompts = [_prompt(n, 50 + n) for n in (20, 130, 260)]
    res = {}
    for graphs in (True, False):
        eng = _engine(use_cuda_graphs=graphs)
        res[graphs] = _gen(eng, prompts, _sp(max_tokens=24, min_tokens=24))
        st = eng.status()
        eng.close()
        assert (st.graph_launches > 0) == graphs
    assert res[True] == res[False]


def test_half_the_head_size_is_twice_the_kv_blocks():
    """same cache bytes, same dims except head_dim 64 vs 128: twice the blocks"""
    from vllm_tgis_adapter_b200.engine.core import NativeEngine

    blocks = {}
    for hd in (64, 128):
        mc = _mc(head_dim=hd, rope_scaling_factor=0.0, max_model_len=512)
        eng = NativeEngine(mc, max_num_seqs=64, max_batched_tokens=256, kv_cache_bytes=24 << 20)
        blocks[hd] = eng.status().total_blocks
        eng.close()
    assert abs(blocks[64] - 2 * blocks[128]) <= 1 and blocks[128] > 100, blocks


def test_start_up_refusals():
    from vllm_tgis_adapter_b200.engine.core import EngineError, NativeEngine

    kw = dict(max_num_seqs=2, max_batched_tokens=64, kv_cache_bytes=16 << 20)
    with pytest.raises(EngineError, match="head_dim 64.*single GPU"):
        NativeEngine(_mc(), tp_size=2, tp_rank=0, nccl_id=bytes(128), shm_name="/tgis_test_unused", **kw)
    with pytest.raises(EngineError, match="head_dim 64.*LoRA"):
        NativeEngine(_mc(), max_loras=1, **kw)
    with pytest.raises(EngineError, match="head_dim"):
        NativeEngine(_mc(embedding_multiplier=12.0), **kw)
    with pytest.raises(EngineError, match="GQA group size must be 1, 2, 4 or 8"):
        NativeEngine(_mc(n_q_heads=6, n_kv_heads=2, hidden=384), **kw)
    # the C ABI refuses Granite scalars on a 64-dim engine too (NativeEngine checks first)
    eng = NativeEngine(_mc(rope_scaling_factor=0.0), **kw)
    from vllm_tgis_adapter_b200.engine import _lib

    assert eng.lib.tgis_engine_set_model_scalars(eng._h, 12.0, 0.22, 0.0, 1.0) != 0
    assert "head_dim" in _lib.last_error(eng.lib)
    assert eng.lib.tgis_engine_set_model_scalars(eng._h, 1.0, 1.0, 0.0, 1.0) == 0   # the Llama defaults are fine
    eng.close()
    # a model whose rotary table is scaled must be given it: the built-in table is the unscaled one.  NativeEngine loads the
    # table of a scaled config itself; through the C ABI alone the requirement stands until the table arrives
    eng = NativeEngine(_mc(rope_scaling_factor=0.0), **kw)
    eng.load_weights(_weights())
    assert eng.lib.tgis_engine_require_rope_table(eng._h) == 0
    with pytest.raises(EngineError, match="rope_cos_sin"):
        eng.start()
    with pytest.raises(EngineError, match="rope_cos_sin"):
        eng.run_until_idle()
    eng.load_weight("tgis.rope_cos_sin", rope_table(_cfg()))
    eng.start()
    eng.close()
    eng = _engine(table=False)     # scaled preset: NativeEngine brought the table
    assert _gen(eng, [[5, 6, 7]], _sp(max_tokens=2, min_tokens=2))[0]
    eng.close()


def _check_greedy(cfg, weights, prompts, outs, n_new):
    ora = Llama3Oracle(cfg, weights, device="cuda")
    for p, recs in zip(prompts, outs):
        recs = [r for r in recs if r.new_token is not None]
        assert len(recs) == n_new
        s = ora.new_seq()
        logits = ora.step([(s, p)])[0]
        for r in recs:
            lp = torch.log_softmax(logits, -1)
            top2 = torch.topk(logits, 2).values
            u = _ulp(float(top2[0]))
            if r.new_token != int(torch.argmax(logits)):
                assert float(top2[0] - top2[1]) <= 2 * u + 1e-6
            assert abs(r.logprob - float(lp[r.new_token])) <= 3 * u
            logits = ora.step([(s, [r.new_token])])[0]


@pytest.mark.parametrize("style", ["llama-3.1", "llama-3.2"])
def test_hf_checkpoint_directory_loads_and_follows_the_oracle(tmp_path, style):
    """config.json + model.safetensors as a Llama-3.1 checkpoint has them (legacy `rope_scaling`, 128-dim heads, its own
    lm_head) and as Llama-3.2-1B has them (`rope_parameters`, head_dim 64, tied: no lm_head.weight in the file), through the
    loader's config mapping and safetensors reader; greedy tokens and logprobs follow the oracle on the same weights."""
    import argparse
    import json

    from safetensors.torch import save_file

    from llama3_oracle import Llama3Config
    from vllm_tgis_adapter_b200.engine.loader import _make_native_engine, _resolve_model

    hd, tied = (128, False) if style == "llama-3.1" else (64, True)
    cfg = Llama3Config(n_layers=2, hidden=256, n_q_heads=4, n_kv_heads=2, ffn=512, vocab=1024, head_dim=hd,
                       rope_theta=500000.0, max_model_len=1024, rope_factor=8.0, rope_original_max_pos=64,
                       tie_word_embeddings=tied)
    weights = synthetic_weights(cfg, seed=9)
    rope = {"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
            "original_max_position_embeddings": 64}
    hf = {"architectures": ["LlamaForCausalLM"], "model_type": "llama", "hidden_size": 256, "num_attention_heads": 4,
          "num_key_value_heads": 2, "num_hidden_layers": 2, "intermediate_size": 512, "vocab_size": 1024,
          "head_dim": hd, "max_position_embeddings": 1024, "rms_norm_eps": 1e-5, "tie_word_embeddings": tied}
    if style == "llama-3.1":
        hf.update(rope_theta=500000.0, rope_scaling=rope)
    else:
        hf.update(rope_parameters={**rope, "rope_theta": 500000.0})
    (tmp_path / "config.json").write_text(json.dumps(hf))
    save_file({k: v.contiguous() for k, v in weights.items()}, str(tmp_path / "model.safetensors"))
    args = argparse.Namespace(model=str(tmp_path), max_model_len=None, synthetic_weights=False, max_num_seqs=4,
                              max_num_batched_tokens=256, gpu_memory_utilization=0.05, seed=0, enable_lora=False)
    mc, path = _resolve_model(args)
    assert (mc.head_dim, mc.tie_word_embeddings, mc.rope_scaled, mc.max_model_len) == (hd, tied, True, 1024)
    assert ("lm_head.weight" in weights) != tied
    eng = _make_native_engine(args, mc, path, device=0)
    prompts = [_prompt(90, 1), [12, 13, 14]]
    outs = eng.generate_sync(prompts, _sp(max_tokens=12, min_tokens=12))
    eng.close()
    _check_greedy(cfg, weights, prompts, outs, 12)


def test_synthetic_llama32_preset_generates_over_grpc():
    """`--model llama-tiny-hd64 --synthetic-weights` through loader.build_engine and the gRPC service: Generate returns the
    requested tokens (the llama3.2-1b preset takes the same path at full size)."""
    import argparse
    import asyncio
    import threading

    import grpc

    from vllm_tgis_adapter_b200.engine.loader import build_engine
    from vllm_tgis_adapter_b200.engine.tokenizer import synthetic_prompt
    from vllm_tgis_adapter_b200.grpc import grpc_server
    from vllm_tgis_adapter_b200.grpc.pb import generation_pb2 as pb

    args = argparse.Namespace(model="llama-tiny-hd64", max_model_len=None, synthetic_weights=True, max_num_seqs=4,
                              max_num_batched_tokens=256, gpu_memory_utilization=0.05, seed=0, enable_lora=False,
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
    assert ready.wait(120)
    try:
        with grpc.insecure_channel(f"127.0.0.1:{box['port']}") as ch:
            call = ch.unary_unary("/fmaas.GenerationService/Generate",
                                  request_serializer=pb.BatchedGenerationRequest.SerializeToString,
                                  response_deserializer=pb.BatchedGenerationResponse.FromString)
            params = pb.Parameters()
            params.stopping.max_new_tokens = params.stopping.min_new_tokens = 10
            prompts = [_prompt(80, 4), _prompt(9, 5)]
            resp = call(pb.BatchedGenerationRequest(model_id="m", params=params, requests=[
                pb.GenerationRequest(text=synthetic_prompt(p)) for p in prompts]), timeout=60)
        assert [r.generated_token_count for r in resp.responses] == [10, 10]
        assert [r.input_token_count for r in resp.responses] == [80, 9]
    finally:
        loop.call_soon_threadsafe(box["stop"].set)
        th.join(20)
    assert not th.is_alive()
