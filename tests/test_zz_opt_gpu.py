"""-m gpu parity of the OPT model family (SURVEY.md §8 f-4; the reference's own test model is facebook/opt-125m:
/root/reference/tests/conftest.py:79-91 leaves --model at vLLM's default, tests/test_hub.py:17 names it).

Kernel level: csrc/opt.cu against the arithmetic of oracle/opt_oracle.py (torch.nn.LayerNorm / F.linear(x, W, b) / ReLU
rounding points).  Engine level, through the C ABI: greedy tokens, logprobs, ranks and prompt logprobs against the CPU
oracle (pinned to transformers' OPTForCausalLM by tests/test_opt_oracle_cpu.py), incl. chunked prefill, 64-dim heads on
the 128-dim attention tiles and the facebook/opt-125m dims.  gRPC level: BASELINE configs[0] — one greedy request
through `Generate` on the opt-125m architecture.

(The file name sorts last on purpose: the newest model family runs after the established suite.)"""
import ctypes as C
import dataclasses

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _lib():
    from vllm_tgis_adapter_b200.engine import _lib as L

    return L.load_library()


def _p(t):
    return C.c_void_p(t.data_ptr())


# ---------------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("T,H", [(1, 256), (37, 768), (2048, 768), (300, 4096), (5, 8192)])
@pytest.mark.parametrize("add", [False, True])
def test_opt_layernorm_kernel_matches_torch_layernorm(T, H, add):
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(T * 7 + H)
    resid = (torch.randn(T, H, generator=g, device="cuda") * 1.5).to(torch.bfloat16)
    w = (1 + 0.1 * torch.randn(H, generator=g, device="cuda")).to(torch.bfloat16)
    b = (0.05 * torch.randn(H, generator=g, device="cuda")).to(torch.bfloat16)
    acc = torch.randn(T, H, generator=g, device="cuda", dtype=torch.float32)
    ab = (0.05 * torch.randn(H, generator=g, device="cuda")).to(torch.bfloat16)
    out = torch.empty_like(resid)
    r_in = resid.clone()
    if add:
        y = (acc + ab.float()).to(torch.bfloat16)
        h = r_in + y                                   # bf16 add: one rounding
    else:
        h = r_in
    ref = torch.nn.functional.layer_norm(h.float(), (H,), w.float(), b.float(), 1e-5).to(torch.bfloat16)
    rc = lib.tgis_k_opt_layernorm(_p(acc) if add else None, _p(ab) if add else None, _p(resid), _p(w), _p(b), _p(out),
                                  T, H, C.c_float(1e-5))
    assert rc == 0, lib.tgis_k_last_error()
    assert torch.equal(resid, h)                       # residual stream: bit-exact
    d = (out.float() - ref.float()).abs()
    # fp32 reductions in a different order than torch's: a result may land on the other side of a bf16 rounding tie
    # (ulp of the larger of the two: a pair that straddles a power of two is one ulp of the upper binade apart)
    ulp = 2.0 ** (torch.floor(torch.log2(torch.maximum(ref.float().abs(), out.float().abs()).clamp_min(1e-30))) - 7)
    # ... and an output next to zero is a cancellation of two terms of size ~|b|: there the fp32 noise of the terms (not
    # the bf16 grid of the tiny result) bounds the difference
    assert bool(((d <= ulp) | (d <= 1e-6)).all()), float((d / ulp).max())
    assert float((d == 0).float().mean()) > 0.98


@pytest.mark.parametrize("T,N,relu", [(1, 768, 0), (33, 3072, 1), (257, 4608, 0), (2048, 3072, 1)])
def test_opt_bias_act_kernel_is_exact(T, N, relu):
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(N + T)
    acc = torch.randn(T, N, generator=g, device="cuda", dtype=torch.float32)
    bias = (0.1 * torch.randn(N, generator=g, device="cuda")).to(torch.bfloat16)
    out = torch.empty(T, N, device="cuda", dtype=torch.bfloat16)
    rc = lib.tgis_k_opt_bias_act(_p(acc), _p(bias), _p(out), T, N, relu)
    assert rc == 0, lib.tgis_k_last_error()
    ref = acc + bias.float()
    if relu:
        ref = torch.relu(ref)
    assert torch.equal(out, ref.to(torch.bfloat16))


def test_opt_embed_kernel_is_exact():
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(3)
    V, H, P = 1000, 768, 130
    tab = torch.randn(V, H, generator=g, device="cuda").to(torch.bfloat16)
    ptab = torch.randn(P + 2, H, generator=g, device="cuda").to(torch.bfloat16)
    tok = torch.randint(0, V, (77,), generator=g, device="cuda", dtype=torch.int32)
    pos = torch.randint(0, P, (77,), generator=g, device="cuda", dtype=torch.int32)
    out = torch.empty(77, H, device="cuda", dtype=torch.bfloat16)
    rc = lib.tgis_k_opt_embed(_p(tok), _p(pos), _p(tab), _p(ptab), _p(out), 77, H, V, P + 2, 2)
    assert rc == 0, lib.tgis_k_last_error()
    assert torch.equal(out, tab[tok.long()] + ptab[pos.long() + 2])


# ---------------------------------------------------------------------------------------------------- engine
def _record(name, stats):
    """Parity statistics kept as evidence of a GPU run."""
    import json
    import os

    os.makedirs("gpurun_out", exist_ok=True)
    path = "gpurun_out/parity_stats_opt.json"
    allstats = json.load(open(path)) if os.path.exists(path) else {}
    allstats[name] = stats
    with open(path, "w") as f:
        json.dump(allstats, f, indent=1)


def _opt_cfg(name):
    from oracle.opt_oracle import OPT_CONFIGS

    if name == "opt-125m-2l":
        return dataclasses.replace(OPT_CONFIGS["opt-125m"], n_layers=2, max_model_len=512)
    return OPT_CONFIGS[name]


def _run_opt_engine(cfg, weights, prompts, sp, **eng_kw):
    from vllm_tgis_adapter_b200.engine.core import ModelConfig, NativeEngine

    mc = ModelConfig(n_layers=cfg.n_layers, hidden=cfg.hidden, n_q_heads=cfg.n_heads, n_kv_heads=cfg.n_heads, ffn=cfg.ffn,
                     vocab=cfg.vocab, head_dim=cfg.head_dim, rms_eps=cfg.ln_eps, max_model_len=cfg.max_model_len,
                     arch="opt")
    eng = NativeEngine(mc, **eng_kw)
    eng.load_weights(weights)
    outs = eng.generate_sync(prompts, sp)
    st = eng.status()
    eng.close()
    return outs, st


def _follow(ora, prompt, toks):
    """Teacher-forced oracle pass: per step (oracle argmax, logprob of the forced token, top-2 margin, rank of forced)."""
    st = ora.new_seq()
    logits = ora.step([(st, prompt)])[0]
    recs = []
    for t in toks:
        lp = torch.log_softmax(logits, -1)
        top2 = torch.topk(logits, 2).values
        recs.append((int(torch.argmax(logits)), float(lp[t]), float(top2[0] - top2[1]), int((lp >= lp[t]).sum()),
                     float(logits.abs().max())))
        logits = ora.step([(st, [t])])[0]
    return recs


@pytest.mark.parametrize("name,chunk,device", [("opt-tiny", 2048, "cpu"), ("opt-tiny", 48, "cpu"),
                                               ("opt-125m-2l", 256, "cuda")])
def test_opt_greedy_generation_matches_oracle(name, chunk, device):
    from oracle.opt_oracle import OPTOracle, synthetic_opt_weights
    from vllm_tgis_adapter_b200.engine.core import make_sampling_params

    cfg = _opt_cfg(name)
    weights = synthetic_opt_weights(cfg, seed=41)
    rng = np.random.RandomState(5)
    prompts = [rng.randint(3, cfg.vocab, size=n).tolist() for n in (5, 33, 64, 100, 17, 250)]
    n_new = 20
    sp = make_sampling_params(greedy=True, max_tokens=n_new, min_tokens=n_new, num_logprobs=1, eos_token_id=2)
    outs, st = _run_opt_engine(cfg, weights, prompts, sp, max_num_seqs=8, max_batched_tokens=chunk,
                               kv_cache_bytes=64 << 20)
    assert st.errored == 0 and st.kernel_launches > 0
    ora = OPTOracle(cfg, weights, device=device)
    flips = total = 0
    diffs = []
    for p, recs in zip(prompts, outs):
        toks = [r.new_token for r in recs if r.new_token is not None]
        assert len(toks) == n_new and recs[-1].finish_reason == 1
        for (otok, olp, margin, orank, amax), r in zip(_follow(ora, p, toks), recs):
            ulp = 2.0 ** (np.floor(np.log2(amax)) - 7)      # bf16 resolution of this row's largest logits
            total += 1
            diffs.append(abs(r.logprob - olp) / ulp)
            if r.new_token != otok:
                assert margin <= 2 * ulp, (margin, ulp, r.new_token, otok)   # only a near-tie of the oracle may flip
                flips += 1
            elif margin > 2 * ulp:
                assert r.rank == orank == 1
    diffs = np.array(diffs)
    _record(f"opt_greedy_{name}_{chunk}", {"steps": total, "token_flips": flips, "logprob_absdiff_ulps_max": float(diffs.max()),
                                            "logprob_absdiff_ulps_mean": float(diffs.mean()),
                                            "frac_identical": float((diffs == 0).mean())})
    assert flips <= max(1, total // 20), (flips, total)
    # same envelope as the Llama engine tests, in bf16 ulps of the logits: two independent stacks differ by whole ulps of
    # single logits wherever an upstream bf16 rounding lands on the other side of a tie (DESIGN.md section 5)
    assert float(diffs.mean()) < 0.6 and float(diffs.max()) <= 3.0, (float(diffs.mean()), float(diffs.max()))


def test_opt_prompt_logprobs_match_oracle_across_chunks():
    from oracle.opt_oracle import OPTOracle, synthetic_opt_weights
    from vllm_tgis_adapter_b200.engine.core import make_sampling_params

    cfg = _opt_cfg("opt-tiny")
    weights = synthetic_opt_weights(cfg, seed=43)
    rng = np.random.RandomState(7)
    prompts = [rng.randint(3, cfg.vocab, size=n).tolist() for n in (100, 9, 37)]
    sp = make_sampling_params(greedy=True, max_tokens=2, num_logprobs=1, prompt_logprobs=3)
    outs, st = _run_opt_engine(cfg, weights, prompts, sp, max_num_seqs=4, max_batched_tokens=48, kv_cache_bytes=32 << 20)
    assert st.errored == 0
    ora = OPTOracle(cfg, weights)
    diffs = []
    for p, recs in zip(prompts, outs):
        prec = sorted([r for r in recs if r.prompt_pos >= 1], key=lambda r: r.prompt_pos)
        assert [r.prompt_pos for r in prec] == list(range(1, len(p)))
        lp = torch.log_softmax(ora.step([(ora.new_seq(), p)], want_all_logits=True), -1)
        for r in prec:
            i = r.prompt_pos
            assert r.token_id == p[i]
            ref = float(lp[i - 1, p[i]])
            diffs.append(abs(r.logprob - ref))
            lo = int((lp[i - 1] > ref + 0.03).sum()) + 1
            hi = int((lp[i - 1] >= ref - 0.03).sum())
            assert lo <= r.rank <= hi, (r.rank, lo, hi)
            assert len(r.topn) == 3
    diffs = np.array(diffs)
    assert float(diffs.mean()) < 4e-3 and float(diffs.max()) < 3e-2, (float(diffs.mean()), float(diffs.max()))


def test_opt_cuda_graph_replay_equals_plain_launches(monkeypatch):
    """Decode steps of the OPT stack are captured into CUDA graphs like the Llama ones: same tokens and logprobs, bit for
    bit, with and without replay."""
    from oracle.opt_oracle import synthetic_opt_weights
    from vllm_tgis_adapter_b200.engine.core import make_sampling_params

    cfg = _opt_cfg("opt-tiny")
    weights = synthetic_opt_weights(cfg, seed=44)
    rng = np.random.RandomState(11)
    prompts = [rng.randint(3, cfg.vocab, size=n).tolist() for n in (70, 5, 130, 33)]
    sp = make_sampling_params(greedy=True, max_tokens=16, min_tokens=16, num_logprobs=2)
    res = []
    for graphs in (True, False):
        outs, st = _run_opt_engine(cfg, weights, prompts, sp, max_num_seqs=4, max_batched_tokens=256,
                                   kv_cache_bytes=32 << 20, use_cuda_graphs=graphs)
        assert st.errored == 0
        assert (st.graph_launches > 0) == graphs
        res.append([[(r.new_token, r.logprob, r.rank) for r in recs] for recs in outs])
    assert res[0] == res[1]


def test_opt_engine_refuses_what_it_does_not_implement():
    from vllm_tgis_adapter_b200.engine.core import EngineError, ModelConfig, NativeEngine

    base = dict(n_layers=1, hidden=256, n_q_heads=4, n_kv_heads=4, ffn=512, vocab=1024, head_dim=64, max_model_len=128,
                arch="opt")
    with pytest.raises(EngineError, match="LoRA"):
        NativeEngine(ModelConfig(**base), max_num_seqs=2, max_batched_tokens=64, kv_cache_bytes=8 << 20, max_loras=1)
    with pytest.raises(EngineError, match="n_kv_heads"):
        NativeEngine(ModelConfig(**{**base, "n_kv_heads": 2}), max_num_seqs=2, max_batched_tokens=64, kv_cache_bytes=8 << 20)
    with pytest.raises(EngineError, match="head_dim"):
        NativeEngine(ModelConfig(**{**base, "head_dim": 32, "n_q_heads": 8, "n_kv_heads": 8}), max_num_seqs=2,
                     max_batched_tokens=64, kv_cache_bytes=8 << 20)
    # a checkpoint with tensors missing must fail at start-up, not serve zeros
    from oracle.opt_oracle import OPTConfig, synthetic_opt_weights

    w = synthetic_opt_weights(OPTConfig(n_layers=1, hidden=256, n_heads=4, ffn=512, vocab=1024, max_positions=128,
                                        max_model_len=128), seed=1)
    eng = NativeEngine(ModelConfig(**base), max_num_seqs=2, max_batched_tokens=64, kv_cache_bytes=8 << 20)
    for k, v in w.items():
        if not k.endswith("fc2.bias"):
            eng.load_weight(k, v)
    with pytest.raises(EngineError, match="incomplete"):
        eng.start()
    eng.close()


@pytest.mark.parametrize("name,top_logit", [("opt-tiny", 1.0), ("opt-125m", 2.0)])
def test_opt_engine_matches_vllm_fixture(name, top_logit):
    """Engine (C ABI) vs what vLLM 0.22.0's own OPT implementation produced on a GPU for the same seeded checkpoint and
    requests (tests/golden/vllm_<name>.json from scripts/vllm_crosscheck.py check --configs opt-tiny opt-125m): vLLM's
    greedy continuations scored by the engine's prompt-logprob pass (every step compared, teacher-forced), vLLM's prompt
    logprobs, and the free-running greedy prefix.  In bf16 ulps of the logits, like the Llama fixtures."""
    import json
    import math
    from pathlib import Path

    from oracle.opt_oracle import OPT_CONFIGS, synthetic_opt_weights
    from vllm_tgis_adapter_b200.engine.core import ModelConfig, NativeEngine, make_sampling_params

    path = Path(__file__).resolve().parent / "golden" / f"vllm_{name}.json"
    if not path.exists():
        pytest.skip(f"{path.name} not generated yet (scripts/vllm_crosscheck.py check on the GPU box)")
    fx = json.loads(path.read_text())
    cfg = dataclasses.replace(OPT_CONFIGS[name], max_model_len=1024) if name == "opt-125m" else OPT_CONFIGS[name]
    weights = synthetic_opt_weights(cfg, seed=fx["meta"]["weights_seed"])
    u = 2.0 ** (math.floor(math.log2(top_logit)) - 7)
    rng = np.random.RandomState(0)
    greedy = [rng.randint(3, cfg.vocab, size=n).tolist() for n in (5, 33, 64, 100, 17, 250)]
    rng = np.random.RandomState(7)
    plp = [rng.randint(3, cfg.vocab, size=96).tolist() for _ in range(4)]
    mc = ModelConfig(n_layers=cfg.n_layers, hidden=cfg.hidden, n_q_heads=cfg.n_heads, n_kv_heads=cfg.n_heads, ffn=cfg.ffn,
                     vocab=cfg.vocab, head_dim=cfg.head_dim, rms_eps=cfg.ln_eps, max_model_len=cfg.max_model_len,
                     arch="opt")
    eng = NativeEngine(mc, max_num_seqs=16, max_batched_tokens=2048, kv_cache_bytes=1 << 30)
    eng.load_weights(weights)
    # free-running greedy: identical to vLLM's tokens up to the first near-tie
    n_new = len(fx["greedy"][0]["tokens"])
    sp = make_sampling_params(greedy=True, max_tokens=n_new, min_tokens=n_new, num_logprobs=3, eos_token_id=2)
    outs = eng.generate_sync(greedy, sp)
    compared = 0
    for recs, v in zip(outs, fx["greedy"]):
        recs = [r for r in recs if r.new_token is not None]
        for r, vt, vs in zip(recs, v["tokens"], v["steps"]):
            top = sorted(vs["top"], key=lambda t: -t[1])
            if r.new_token != vt:
                assert top[0][1] - top[1][1] <= 2 * u + 1e-6
                break
            compared += 1
    # teacher-forced on vLLM's continuations
    seqs = [p + v["tokens"] for p, v in zip(greedy, fx["greedy"])]
    sp = make_sampling_params(greedy=True, max_tokens=1, num_logprobs=1, prompt_logprobs=1, eos_token_id=2)
    outs = eng.generate_sync(seqs, sp)
    tf, argmax_bad = [], 0
    for p, v, recs in zip(greedy, fx["greedy"], outs):
        pos = {r.prompt_pos: r for r in recs if r.prompt_pos >= 1}
        for k, (vt, vs) in enumerate(zip(v["tokens"], v["steps"])):
            r = pos[len(p) + k]
            tf.append(abs(r.logprob - vs["logprob"]))
            top = sorted(vs["top"], key=lambda t: -t[1])
            if top[0][1] - top[1][1] > 2 * u:
                argmax_bad += int(r.topn[0][0] != vt)
    sp = make_sampling_params(greedy=True, max_tokens=1, num_logprobs=2, prompt_logprobs=2, eos_token_id=2)
    outs = eng.generate_sync(plp, sp)
    pd = []
    for p, recs, v in zip(plp, outs, fx["plp"]):
        pos = {r.prompt_pos: r for r in recs if r.prompt_pos >= 1}
        for i, vp in zip(range(1, len(p)), v["positions"]):
            pd.append(abs(pos[i].logprob - vp["logprob"]))
    eng.close()
    tf, pd = np.array(tf), np.array(pd)
    _record(f"opt_vllm_fixture_{name}", {"free_running_steps_identical": compared, "teacher_forced_steps": int(tf.size),
                                         "tf_absdiff_ulps_max": float(tf.max() / u), "tf_absdiff_ulps_mean": float(tf.mean() / u),
                                         "tf_argmax_mismatch_off_ties": argmax_bad, "prompt_positions": int(pd.size),
                                         "plp_absdiff_ulps_max": float(pd.max() / u), "plp_absdiff_ulps_mean": float(pd.mean() / u)})
    assert tf.size == sum(len(v["tokens"]) for v in fx["greedy"]) and argmax_bad == 0
    assert float(tf.max()) <= 3 * u + 1e-4 and float(tf.mean()) <= 0.6 * u, (float(tf.max()), float(tf.mean()), u)
    assert float(pd.max()) <= 4 * u + 1e-4 and float(pd.mean()) <= 0.6 * u, (float(pd.max()), float(pd.mean()), u)
    assert compared >= 0.5 * sum(len(v["tokens"]) for v in fx["greedy"]), compared


# ---------------------------------------------------------------------------------------------------- gRPC (configs[0])
def test_cfg0_opt_125m_single_greedy_generate_matches_oracle():
    """BASELINE.json configs[0] on the architecture it names: facebook/opt-125m's dims (12 layers, hidden 768, 12 x 64-dim
    heads, ffn 3072, vocab 50272, learned positions, biases, LayerNorm, ReLU; seeded random weights -- the hub checkpoint
    is not obtainable offline), ONE greedy request through `Generate` -- the reference's fixture path
    (/root/reference/tests/test_grpc_server.py:42-49: text, token count, stop reason) -- token by token against the oracle."""
    from oracle.opt_oracle import OPTOracle
    from test_server_gpu import LiveServer
    from vllm_tgis_adapter_b200.engine.tokenizer import synthetic_prompt
    from vllm_tgis_adapter_b200.grpc.pb import generation_pb2 as pb

    srv = LiveServer("opt-125m", seed=47)
    try:
        rs = np.random.RandomState(47)
        prompt = rs.randint(3, srv.cfg.vocab, size=64).tolist()
        params = pb.Parameters()
        params.stopping.max_new_tokens = 20
        params.stopping.min_new_tokens = 20
        params.response.generated_tokens = True
        params.response.token_logprobs = True
        call = srv.channel.unary_unary("/fmaas.GenerationService/Generate",
                                       request_serializer=pb.BatchedGenerationRequest.SerializeToString,
                                       response_deserializer=pb.BatchedGenerationResponse.FromString)
        resp = call(pb.BatchedGenerationRequest(model_id="m", requests=[pb.GenerationRequest(text=synthetic_prompt(prompt))],
                                                params=params), timeout=120)
        assert len(resp.responses) == 1
        r = resp.responses[0]
        assert r.text and r.generated_token_count == 20 and r.input_token_count == 64
        assert r.stop_reason == pb.StopReason.MAX_TOKENS
        toks = [int(ti.text[1:]) for ti in r.tokens]
        ora = OPTOracle(srv.cfg, srv.weights, device="cuda")
        n_same = 0
        for (otok, olp, margin, _, amax), ti, tok in zip(_follow(ora, prompt, toks), r.tokens, toks):
            ulp = 2.0 ** (np.floor(np.log2(amax)) - 7)
            if tok != otok:
                assert margin <= 2 * ulp, (margin, ulp)
            else:
                n_same += 1
            assert abs(ti.logprob - olp) <= 3 * ulp
        assert n_same >= 16
    finally:
        srv.close()
