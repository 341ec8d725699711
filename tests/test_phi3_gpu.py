"""-m gpu: Phi-3.  The engine on the phi3-tiny preset (96-dim heads, GQA group 1, odd vocabulary) against
tests/phi3_oracle.py in both LongRoPE regimes and with a window, with the bars of tests/test_mistral_gpu.py; bit-identity
under batching with preemption, with CUDA graphs on and off and on a prefix-cache hit; 4/3 the KV blocks of a 128-dim
engine at equal bytes; the start-up refusals; a save_pretrained checkpoint with fused tensors; the phi3-mini-4k preset
over gRPC; and a phi3-medium-4k-shaped engine (128-dim heads, group 4)."""
import dataclasses
import math

import numpy as np
import pytest
import torch

from phi3_oracle import Phi3Config, Phi3Oracle, fuse, synthetic_weights

pytestmark = pytest.mark.gpu

ORIG, MAX_POS = 64, 512
_G = torch.Generator().manual_seed(5)
LONG = tuple((1.0 + torch.rand(48, generator=_G) * 7.0).tolist())
SHORT = tuple((1.0 + torch.rand(48, generator=_G) * 0.5).tolist())
_W = {}
EOS = 2


def _cfg(max_model_len, longrope=True, window=None):
    extra = dict(long_factor=LONG, short_factor=SHORT, original_max_pos=ORIG, max_position_embeddings=MAX_POS) \
        if longrope else {}
    return Phi3Config(n_layers=2, hidden=384, n_q_heads=4, n_kv_heads=4, ffn=512, vocab=1021, head_dim=96,
                      rope_theta=10000.0, rms_eps=1e-5, max_model_len=max_model_len, sliding_window=window, **extra)


def _mc(max_model_len, longrope=True, **over):
    from vllm_tgis_adapter_b200.engine.core import PRESETS

    extra = dict(rope_long_factor=LONG, rope_short_factor=SHORT, rope_original_max_pos=ORIG,
                 rope_max_position_embeddings=MAX_POS) if longrope else {}
    return dataclasses.replace(PRESETS["phi3-tiny"], max_model_len=max_model_len, **extra, **over)


def _weights():
    if "w" not in _W:
        _W["w"] = synthetic_weights(_cfg(512), seed=9)
    return _W["w"]


def _engine(model, **kw):
    from vllm_tgis_adapter_b200.engine.core import NativeEngine

    kw.setdefault("max_num_seqs", 8)
    kw.setdefault("kv_cache_bytes", 32 << 20)
    eng = NativeEngine(model, **kw)
    eng.load_weights(_weights())   # the LongRoPE table is loaded by NativeEngine itself
    return eng


def _sp(**kw):
    from vllm_tgis_adapter_b200.engine.core import make_sampling_params

    d = dict(greedy=True, max_tokens=16, min_tokens=16, num_logprobs=1, eos_token_id=EOS)
    d.update(kw)
    return make_sampling_params(**d)


def _gen(eng, prompts, sp):
    outs = eng.generate_sync(prompts, sp)
    return [[(r.new_token, r.logprob, r.rank, tuple(r.topn)) for r in recs if r.new_token is not None] for recs in outs]


def _prompt(n, seed, vocab=1021):
    return np.random.RandomState(seed).randint(3, vocab, size=n).tolist()


def _ulp(x: float) -> float:
    return 2.0 ** (math.floor(math.log2(max(abs(x), 1e-6))) - 7)


def _check_greedy(ora, prompts, outs, n_new):
    """teacher-forced on the engine's tokens (tests/test_mistral_gpu.py's bars): a flip only inside a 2-ulp race,
    logprobs and top-n within 3 bf16 ulps of the oracle's"""
    flips = steps = 0
    for p, recs in zip(prompts, outs):
        recs = [r for r in recs if r.new_token is not None]
        assert len(recs) == n_new
        s = ora.new_seq()
        logits = ora.step([(s, p)])[0]
        for r in recs:
            lp = torch.log_softmax(logits, -1)
            allowed = logits.clone()
            allowed[EOS] = float("-inf")
            top2 = torch.topk(allowed, 2).values
            u, margin = _ulp(float(top2[0])), float(top2[0] - top2[1])
            steps += 1
            if r.new_token != int(torch.argmax(allowed)):
                assert margin <= 2 * u + 1e-6, (margin, u)
                flips += 1
            assert abs(r.logprob - float(lp[r.new_token])) <= 3 * u
            for tid, tlp in r.topn:
                assert abs(tlp - float(lp[tid])) <= 3 * u
            logits = ora.step([(s, [r.new_token])])[0]
    assert flips <= steps // 10, (flips, steps)


@pytest.mark.parametrize("max_model_len,window", [(64, None), (512, None), (512, 40)])
def test_greedy_generation_matches_the_phi3_oracle(max_model_len, window):
    """short regime (max_model_len = original: short factors), long regime (long factors for every position, also for
    prompts shorter than the original length, as vLLM does), and long with a window of 40"""
    n_new = 12
    lens = (5, 30, 50) if max_model_len == 64 else (5, 50, 129, 300)
    prompts = [_prompt(n, 10 + n) for n in lens]
    prompts[0][-1] = 1020
    eng = _engine(_mc(max_model_len, sliding_window=window), max_batched_tokens=256)
    outs = eng.generate_sync(prompts, _sp(max_tokens=n_new, min_tokens=n_new, num_logprobs=3))
    st = eng.status()
    eng.close()
    assert st.errored == 0
    ora = Phi3Oracle(_cfg(max_model_len, window=window), _weights(), device="cuda")
    _check_greedy(ora, prompts, outs, n_new)


def test_the_regimes_and_the_window_change_the_oracle_on_these_prompts():
    p = _prompt(50, 60)
    outs = []
    for regime, window in (("short", None), ("long", None), ("long", 40)):
        o = Phi3Oracle(_cfg(512, window=window), _weights(), regime=regime, device="cuda")
        outs.append(o.step([(o.new_seq(), p)])[0])
    assert float((outs[0] - outs[1]).abs().max()) > 0.05 and float((outs[1] - outs[2]).abs().max()) > 0.05


def test_batch_invariance_with_preemption():
    prompts = [_prompt(n, n) for n in (60, 90, 40, 75, 33, 120)]
    sp = _sp(max_tokens=40, min_tokens=40)
    solo_eng = _engine(_mc(512), max_num_seqs=1, max_batched_tokens=512)
    solo = _gen(solo_eng, prompts[:1], sp)
    solo_eng.close()
    # 2 layers * 4 kv heads * 32 tok * 96 dims * 2 B * 2 (K, V) = 96 KiB per block; 17 blocks = 544 tokens
    crowd_eng = _engine(_mc(512), max_num_seqs=6, max_batched_tokens=64, kv_cache_bytes=17 * 98304)
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
        eng = _engine(_mc(512, sliding_window=40), use_cuda_graphs=graphs)
        res[graphs] = _gen(eng, prompts, _sp(max_tokens=24, min_tokens=24, num_logprobs=2))
        st = eng.status()
        eng.close()
        assert (st.graph_launches > 0) == graphs
    assert res[True] == res[False]


def test_prefix_cache_hit_changes_nothing():
    """1024 shared tokens + a 100-token tail: the hit runs the split-context kernel at 96-dim heads; ids and logprobs equal
    a cold engine chunked at the same boundary, bit for bit"""
    P = _prompt(1124, 1)
    X = P[:1024] + _prompt(100, 2)
    mc = _mc(2048, sliding_window=None)
    cold = _engine(mc, max_batched_tokens=1024, enable_prefix_caching=True)
    want = _gen(cold, [P], _sp())
    cold.close()
    eng = _engine(mc, max_batched_tokens=1024, enable_prefix_caching=True)
    _gen(eng, [X], _sp())
    q0, h0, _ = eng.prefix_cache_stats()
    got = _gen(eng, [P], _sp())
    q1, h1, _ = eng.prefix_cache_stats()
    eng.close()
    assert h0 == 0 and q1 - q0 == len(P) and h1 - h0 == 1024
    assert got == want


def test_kv_blocks_follow_the_head_dim():
    """the same cache bytes hold 4/3 the blocks of a 128-dim engine with the same kv heads"""
    from vllm_tgis_adapter_b200.engine.core import ModelConfig, NativeEngine

    kw = dict(max_num_seqs=2, max_batched_tokens=64, kv_cache_bytes=12 * 131072)
    e96 = NativeEngine(_mc(256, longrope=False), **kw)
    e128 = NativeEngine(ModelConfig(n_layers=2, hidden=512, n_q_heads=4, n_kv_heads=4, ffn=512, vocab=1021,
                                    max_model_len=256), **kw)
    b96, b128 = e96.status().total_blocks, e128.status().total_blocks
    e96.close()
    e128.close()
    assert (b96, b128) == (16, 12)


def test_start_up_refusals():
    import ctypes as C

    from vllm_tgis_adapter_b200.engine.core import EngineError, NativeEngine, engine_config

    kw = dict(max_num_seqs=2, max_batched_tokens=64, kv_cache_bytes=16 << 20)
    with pytest.raises(EngineError, match="head_dim 96: GQA group size must be 1, 2, 4 or 8"):
        NativeEngine(_mc(512, n_q_heads=6, n_kv_heads=2, hidden=576), **kw)
    with pytest.raises(EngineError, match="head_dim 96: LoRA"):
        NativeEngine(_mc(512), max_loras=2, **kw)
    with pytest.raises(EngineError, match="single GPU only"):
        NativeEngine(_mc(512), tp_size=2, tp_rank=0, nccl_id=bytes(128), shm_name="/tgis_test_unused", **kw)
    with pytest.raises(EngineError, match="q/k norm .*head_dim 128"):
        NativeEngine(_mc(512, longrope=False, qk_norm=True), **kw)
    with pytest.raises(EngineError, match="head_dim 128 or 64"):
        NativeEngine(_mc(512, longrope=False, qkv_bias=True), **kw)
    with pytest.raises(EngineError, match="96-dim heads"):
        NativeEngine(_mc(512, longrope=False, embedding_multiplier=12.0), **kw)
    NativeEngine(_mc(512, longrope=False, sliding_window=40), **kw).close()
    # a LongRoPE engine refuses to start without its table.  NativeEngine loads it itself, so the wrapper is reused
    # around an engine created from the raw config.
    cfg = engine_config(_mc(512, longrope=False), **kw)
    cfg.rope_table_from_host = 1
    eng = NativeEngine(_mc(512, longrope=False), **kw)
    eng.close()
    assert eng.lib.tgis_engine_create(C.byref(cfg), C.byref(eng._h)) == 0
    eng.load_weights(_weights())
    with pytest.raises(Exception, match="rope"):
        eng.start()
    eng.close()


def test_hf_checkpoint_directory_with_fused_tensors_loads_and_follows_the_oracle(tmp_path):
    """Phi3ForCausalLM.save_pretrained (bf16, 96-dim heads, LongRoPE, fused qkv_proj / gate_up_proj) with the synthetic
    tokenizer saved beside it: the loader's config mapping, the split of the fused tensors and the LongRoPE table"""
    import argparse

    from transformers import Phi3Config as HFPhi3Config
    from transformers import Phi3ForCausalLM

    from vllm_tgis_adapter_b200.engine.loader import _make_native_engine, _resolve_model
    from vllm_tgis_adapter_b200.engine.tokenizer import build_synthetic_tokenizer

    hf_cfg = HFPhi3Config(vocab_size=1021, hidden_size=384, intermediate_size=512, num_hidden_layers=2,
                          num_attention_heads=4, num_key_value_heads=4, rms_norm_eps=1e-5,
                          max_position_embeddings=MAX_POS, original_max_position_embeddings=ORIG,
                          tie_word_embeddings=False, sliding_window=None, pad_token_id=0,
                          rope_scaling={"rope_type": "longrope", "rope_theta": 10000.0, "long_factor": list(LONG),
                                        "short_factor": list(SHORT)})
    torch.manual_seed(0)
    model = Phi3ForCausalLM(hf_cfg).to(torch.bfloat16)
    with torch.no_grad():
        for _, p in model.named_parameters():
            if p.dim() == 2:
                p.normal_(0, 0.02)
    model.save_pretrained(tmp_path, safe_serialization=True)
    build_synthetic_tokenizer(1021).save_pretrained(tmp_path)
    args = argparse.Namespace(model=str(tmp_path), max_model_len=None, synthetic_weights=False, max_num_seqs=4,
                              max_num_batched_tokens=256, gpu_memory_utilization=0.05, seed=0, enable_lora=False)
    mc, path = _resolve_model(args)
    assert (mc.head_dim, mc.max_model_len, mc.rope_original_max_pos, mc.fused_projections) == (96, MAX_POS, ORIG, True)
    prompts = [_prompt(90, 1), [12, 13, 14, 1020]]
    eng = _make_native_engine(args, mc, path, device=0)
    outs = eng.generate_sync(prompts, _sp(max_tokens=24, min_tokens=24))
    eng.close()
    sd = {k: v for k, v in model.state_dict().items() if "rotary" not in k}
    from vllm_tgis_adapter_b200.engine.loader import split_fused

    sep = {n: t for k, v in sd.items() for n, t in split_fused(k, v, mc)}
    assert fuse(sep).keys() == sd.keys()
    ora = Phi3Oracle(_cfg(MAX_POS), sep, regime="long", device="cuda")
    _check_greedy(ora, prompts, outs, 24)


def test_phi3_medium_4k_shaped_engine_builds():
    """128-dim heads, GQA group 4, fused synthetic weights through the loader's split (two layers)"""
    import argparse

    from vllm_tgis_adapter_b200.engine.core import PRESETS
    from vllm_tgis_adapter_b200.engine.loader import _make_native_engine

    mc = dataclasses.replace(PRESETS["phi3-medium-4k"], n_layers=2)
    args = argparse.Namespace(max_num_seqs=2, max_num_batched_tokens=256, gpu_memory_utilization=0.3, seed=0,
                              enable_lora=False)
    eng = _make_native_engine(args, mc, None, device=0)
    outs = eng.generate_sync([_prompt(40, 3, 32064)], _sp(max_tokens=4, min_tokens=4))
    st = eng.status()
    eng.close()
    assert st.errored == 0 and len([r for r in outs[0] if r.new_token is not None]) == 4


def test_synthetic_phi3_mini_4k_preset_over_grpc():
    """`--model phi3-mini-4k --synthetic-weights` (96-dim heads) through loader.build_engine and the gRPC
    service: Generate returns the requested tokens, GenerateStream with max_new_tokens = 10 yields 11 messages"""
    import argparse
    import asyncio
    import threading

    import grpc

    from vllm_tgis_adapter_b200.engine.loader import build_engine
    from vllm_tgis_adapter_b200.engine.tokenizer import synthetic_prompt
    from vllm_tgis_adapter_b200.grpc import grpc_server
    from vllm_tgis_adapter_b200.grpc.pb import generation_pb2 as pb

    args = argparse.Namespace(model="phi3-mini-4k", max_model_len=4096, synthetic_weights=True, max_num_seqs=4,
                              max_num_batched_tokens=512, gpu_memory_utilization=0.35, seed=0, enable_lora=False,
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
    try:
        with grpc.insecure_channel(f"127.0.0.1:{box['port']}") as ch:
            call = ch.unary_unary("/fmaas.GenerationService/Generate",
                                  request_serializer=pb.BatchedGenerationRequest.SerializeToString,
                                  response_deserializer=pb.BatchedGenerationResponse.FromString)
            params = pb.Parameters()
            params.stopping.max_new_tokens = params.stopping.min_new_tokens = 10
            prompts = [_prompt(2100, 4, 32064), _prompt(9, 5, 32064)]
            resp = call(pb.BatchedGenerationRequest(model_id="m", params=params, requests=[
                pb.GenerationRequest(text=synthetic_prompt(p)) for p in prompts]), timeout=120)
            assert [r.generated_token_count for r in resp.responses] == [10, 10]
            assert [r.input_token_count for r in resp.responses] == [2100, 9]
            stream = ch.unary_stream("/fmaas.GenerationService/GenerateStream",
                                     request_serializer=pb.SingleGenerationRequest.SerializeToString,
                                     response_deserializer=pb.GenerationResponse.FromString)
            sparams = pb.Parameters()
            sparams.stopping.max_new_tokens = 10
            chunks = list(stream(pb.SingleGenerationRequest(model_id="m", params=sparams, request=pb.GenerationRequest(
                text=synthetic_prompt(prompts[1]))), timeout=120))
            assert len(chunks) == 11 and chunks[0].input_token_count == 9
    finally:
        loop.call_soon_threadsafe(box["stop"].set)
        th.join(30)
