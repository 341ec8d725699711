"""-m gpu: Mistral.  The engine on the mistral-tiny preset (window 40, GQA group 4, q width != hidden, odd vocabulary)
against tests/mistral_oracle.py with the bars of tests/test_qwen3_gpu.py: greedy tokens, logprobs, ranks and top-n,
prompt logprobs at chunks of 48 and 2048, generation running past twice the window; bit-identity under batching with
preemption, with CUDA graphs on and off and on a prefix-cache hit; the start-up refusals; a save_pretrained checkpoint
directory; and the mistral-7b-v0.1 preset over gRPC."""
import dataclasses
import math

import numpy as np
import pytest
import torch

from mistral_oracle import CONFIGS, MistralConfig, MistralOracle, synthetic_weights

pytestmark = pytest.mark.gpu

_W = {}


def _cfg(**over):
    return dataclasses.replace(CONFIGS["mistral-tiny"], **over)


def _mc(**over):
    from vllm_tgis_adapter_b200.engine.core import PRESETS

    return dataclasses.replace(PRESETS["mistral-tiny"], **over)


def _weights():
    if "w" not in _W:
        _W["w"] = synthetic_weights(_cfg(), seed=8)
    return _W["w"]


def _engine(max_model_len=2048, weights=None, model=None, **kw):
    from oracle.llama_oracle import rope_table
    from vllm_tgis_adapter_b200.engine.core import NativeEngine

    kw.setdefault("max_num_seqs", 8)
    kw.setdefault("kv_cache_bytes", 32 << 20)
    eng = NativeEngine(model or _mc(max_model_len=max_model_len), **kw)
    eng.load_weights(weights or _weights())
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


EOS = 2


def _check_greedy(cfg, weights, prompts, outs, n_new):
    """teacher-forced on the engine's tokens: a flip only inside a 2-ulp race, logprobs within 3 bf16 ulps of the top
    logit, rank 1 outside a race, the top-n ids and values against the oracle's.  Every request asks for min_tokens =
    max_tokens, so the engine never picks EOS: the greedy choice is the argmax over the other tokens, while logprobs and
    ranks are those of the whole distribution."""
    ora = MistralOracle(cfg, weights, device="cuda")
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
            elif margin > 2 * u and abs(float(logits[EOS] - logits[r.new_token])) > 2 * u:
                assert r.rank == 1 + int(logits[EOS] > logits[r.new_token])
            assert abs(r.logprob - float(lp[r.new_token])) <= 3 * u
            for tid, tlp in r.topn:
                assert abs(tlp - float(lp[tid])) <= 3 * u
                assert float(lp[tid]) >= float(torch.topk(lp, len(r.topn)).values[-1]) - 2 * u
            logits = ora.step([(s, [r.new_token])])[0]
    assert flips <= steps // 10, (flips, steps)


def test_the_oracle_without_the_window_differs_on_these_prompts():
    """the engine checks below would pass for an engine that ignored the window only if the window changed nothing"""
    p = _prompt(300, 310)
    a = MistralOracle(_cfg(), _weights(), device="cuda")
    b = MistralOracle(_cfg(), _weights(), window=None, device="cuda")
    la, lb = a.step([(a.new_seq(), p)])[0], b.step([(b.new_seq(), p)])[0]
    assert float((la - lb).abs().max()) > 0.05


@pytest.mark.parametrize("chunk", [2048, 48])
def test_greedy_generation_matches_the_mistral_oracle(chunk):
    prompts = [_prompt(n, 10 + n) for n in (5, 70, 129, 300, 700)]
    prompts[0][-1] = 1020                      # the last token id of the odd vocabulary
    n_new = 16
    eng = _engine(max_batched_tokens=chunk)
    outs = eng.generate_sync(prompts, _sp(max_tokens=n_new, min_tokens=n_new, num_logprobs=3))
    st = eng.status()
    eng.close()
    assert st.errored == 0 and st.graph_launches > 0
    _check_greedy(_cfg(), _weights(), prompts, outs, n_new)


def test_generation_past_twice_the_window_matches_the_oracle():
    """short prompts whose decode steps alone cross W, 2W and later split boundaries (positions up to 205)"""
    prompts = [_prompt(n, 400 + n) for n in (3, 39, 41, 77)]
    n_new = 128
    eng = _engine()
    outs = eng.generate_sync(prompts, _sp(max_tokens=n_new, min_tokens=n_new, num_logprobs=2))
    eng.close()
    _check_greedy(_cfg(), _weights(), prompts, outs, n_new)


@pytest.mark.parametrize("chunk", [2048, 48])
def test_prompt_logprobs_match_the_mistral_oracle(chunk):
    prompts = [_prompt(n, 70 + n) for n in (100, 9, 37, 260)]
    eng = _engine(max_batched_tokens=chunk)
    outs = eng.generate_sync(prompts, _sp(max_tokens=2, min_tokens=0, prompt_logprobs=3))
    eng.close()
    ora = MistralOracle(_cfg(), _weights(), device="cuda")
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
    # 2 layers * 1 kv head * 32 tok * 128 dims * 2 B * 2 (K, V) = 32 KiB per block; 17 blocks = 544 tokens for 6 sequences
    crowd_eng = _engine(max_model_len=512, max_num_seqs=6, max_batched_tokens=64, kv_cache_bytes=17 * 32768)
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
    tokens (the split-context kernel, where the window leaves most of the 8 ranks no visible block).  Ids and logprobs
    equal a cold engine chunked at the same boundary, bit for bit."""
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
    _check_greedy(_cfg(), _weights(), [P], [[_Rec(*t) for t in got[0]]], 16)


@dataclasses.dataclass
class _Rec:
    new_token: int
    logprob: float
    rank: int
    topn: tuple


def test_start_up_refusals():
    from vllm_tgis_adapter_b200.engine.core import PRESETS, EngineError, NativeEngine

    kw = dict(max_num_seqs=2, max_batched_tokens=64, kv_cache_bytes=16 << 20)
    with pytest.raises(EngineError, match="tgis_engine_create failed: .*not OPT"):
        NativeEngine(dataclasses.replace(PRESETS["opt-tiny"], sliding_window=40), **kw)
    with pytest.raises(EngineError, match="single GPU only"):
        NativeEngine(_mc(), tp_size=2, tp_rank=0, nccl_id=bytes(128), shm_name="/tgis_test_unused", **kw)
    with pytest.raises(EngineError, match=">= 0"):
        NativeEngine(_mc(sliding_window=-1), **kw)
    for window in (40, 0):
        eng = NativeEngine(_mc(sliding_window=window), **kw)
        eng.load_weights(_weights())
        eng.start()
        eng.close()


def test_window_zero_through_the_setter_equals_no_window():
    prompts = [_prompt(n, 90 + n) for n in (50, 170)]
    a = _engine(model=_mc(sliding_window=None))
    b = _engine(model=_mc(sliding_window=0))
    ra, rb = _gen(a, prompts, _sp()), _gen(b, prompts, _sp())
    a.close()
    b.close()
    assert ra == rb


def test_hf_checkpoint_directory_loads_and_follows_the_oracle(tmp_path):
    """MistralForCausalLM.save_pretrained (bf16, window 40, q width != hidden, odd vocabulary) with the synthetic tokenizer
    saved beside it: the loader's config mapping, the safetensors reader and the tokenizer; greedy tokens follow the
    oracle past the window"""
    import argparse

    from transformers import MistralConfig as HFMistralConfig
    from transformers import MistralForCausalLM

    from vllm_tgis_adapter_b200.engine.loader import _make_native_engine, _resolve_model
    from vllm_tgis_adapter_b200.engine.tokenizer import build_synthetic_tokenizer, load_tokenizer, synthetic_prompt

    hf_cfg = HFMistralConfig(vocab_size=1021, hidden_size=256, intermediate_size=512, num_hidden_layers=2,
                             num_attention_heads=4, num_key_value_heads=1, head_dim=128, rms_norm_eps=1e-5,
                             max_position_embeddings=1024, tie_word_embeddings=False, sliding_window=40,
                             rope_parameters={"rope_type": "default", "rope_theta": 10000.0})
    torch.manual_seed(0)
    model = MistralForCausalLM(hf_cfg).to(torch.bfloat16)
    with torch.no_grad():
        for _, p in model.named_parameters():
            if p.dim() == 2:
                p.normal_(0, 0.02)
    model.save_pretrained(tmp_path, safe_serialization=True)
    build_synthetic_tokenizer(1021).save_pretrained(tmp_path)
    args = argparse.Namespace(model=str(tmp_path), max_model_len=None, synthetic_weights=False, max_num_seqs=4,
                              max_num_batched_tokens=256, gpu_memory_utilization=0.05, seed=0, enable_lora=False)
    mc, path = _resolve_model(args)
    assert (mc.sliding_window, mc.vocab, mc.tie_word_embeddings, mc.head_dim, mc.max_model_len) == (40, 1021, False,
                                                                                                     128, 1024)
    tok = load_tokenizer(str(path), mc.vocab)
    prompts = [_prompt(90, 1), [12, 13, 14, 1020]]
    assert [tok(synthetic_prompt(p), add_special_tokens=False)["input_ids"] for p in prompts] == prompts
    eng = _make_native_engine(args, mc, path, device=0)
    outs = eng.generate_sync(prompts, _sp(max_tokens=48, min_tokens=48))
    eng.close()
    sd = {k: v for k, v in model.state_dict().items() if "rotary" not in k}
    cfg = MistralConfig(n_layers=2, hidden=256, n_q_heads=4, n_kv_heads=1, ffn=512, vocab=1021, rope_theta=10000.0,
                        rms_eps=1e-5, max_model_len=1024, sliding_window=40)
    _check_greedy(cfg, sd, prompts, outs, 48)


def test_synthetic_mistral_7b_v01_preset_over_grpc():
    """`--model mistral-7b-v0.1 --synthetic-weights` (window 4096) through loader.build_engine and the gRPC service: Generate
    returns the requested tokens, and GenerateStream with max_new_tokens = 10 yields 11 messages"""
    import argparse
    import asyncio
    import threading

    import grpc

    from vllm_tgis_adapter_b200.engine.loader import build_engine
    from vllm_tgis_adapter_b200.engine.tokenizer import synthetic_prompt
    from vllm_tgis_adapter_b200.grpc import grpc_server
    from vllm_tgis_adapter_b200.grpc.pb import generation_pb2 as pb

    args = argparse.Namespace(model="mistral-7b-v0.1", max_model_len=8192, synthetic_weights=True, max_num_seqs=4,
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
            prompts = [_prompt(4200, 4, 32000), _prompt(9, 5, 32000)]   # the first one longer than the window
            resp = call(pb.BatchedGenerationRequest(model_id="m", params=params, requests=[
                pb.GenerationRequest(text=synthetic_prompt(p)) for p in prompts]), timeout=120)
            assert [r.generated_token_count for r in resp.responses] == [10, 10]
            assert [r.input_token_count for r in resp.responses] == [4200, 9]
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
