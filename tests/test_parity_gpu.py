"""-m gpu parity at BASELINE shapes, and against the reference's real engine (vLLM 0.22.0) through committed fixtures.

  * a 2-layer stack with Llama-3-8B dims (hidden 4096, 32/8 heads, ffn 14336, V 128256): engine vs oracle at
    B = 32 x 512-token prompts, greedy (BASELINE configs[1] shape), and at B = 64 with the configs[2] parameter set
    (repetition penalty + ExpDecay length penalty + typical-p sampling, seeded -> compared through the Philox restatement);
  * mixed prompt lengths 64..512 with a KV cache too small for them (forced preemption + recompute) -- configs[3] shape;
  * a real `tgis_engine_abort` mid-generation on the threaded engine (reference call sites grpc_server.py:292,388);
  * engine vs tests/golden/vllm_<cfg>.json: token ids / logprobs / ranks that vLLM itself produced on a GPU
    for the same synthetic checkpoints and request sets (scripts/vllm_crosscheck.py).

The oracle is evaluated with torch ops on the CUDA device here (same code as on the CPU; oracle/llama_oracle.py
`device=`): the 8B-dim shapes are minutes of CPU time.  Tolerances are stated in bf16 ulps of the logits: the logits ARE
bf16 numbers (vLLM's lm_head rounds to the model dtype), so a logit that lands on the other side of a rounding boundary
moves a logprob by one ulp (0.0156 at |x| in [2,4), 0.031 in [4,8)) -- the reference's own batch-composition noise has
exactly this size (DESIGN.md section 5).
"""
import dataclasses
import json
import math
import os
import time
from pathlib import Path

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLD = Path(__file__).parent / "golden"


def _record_stats(name, stats):
    os.makedirs("gpurun_out", exist_ok=True)
    path = "gpurun_out/parity_stats.json"
    allstats = {}
    if os.path.exists(path):
        with open(path) as f:
            allstats = json.load(f)
    allstats[name] = stats
    with open(path, "w") as f:
        json.dump(allstats, f, indent=1)


def _cfg(name):
    from oracle.llama_oracle import CONFIGS

    if name == "8b2l":
        return dataclasses.replace(CONFIGS["llama3-8b"], n_layers=2, max_model_len=1024)
    return CONFIGS[name]


_WEIGHTS = {}


def _weights(name, seed=1, device="cuda"):
    from oracle.llama_oracle import synthetic_weights

    key = (name, seed, device)
    if key not in _WEIGHTS:
        _WEIGHTS.clear()   # one big set at a time
        # drawn on the CPU generator (the fixtures' checkpoints were) and moved: identical bits everywhere
        w = synthetic_weights(_cfg(name), seed=seed)
        _WEIGHTS[key] = {k: v.to(device) for k, v in w.items()}
    return _WEIGHTS[key]


def _engine(name, weights, **kw):
    from oracle.llama_oracle import rope_table
    from vllm_tgis_adapter_b200.engine.core import ModelConfig, NativeEngine

    cfg = _cfg(name)
    mc = ModelConfig(n_layers=cfg.n_layers, hidden=cfg.hidden, n_q_heads=cfg.n_q_heads, n_kv_heads=cfg.n_kv_heads,
                     ffn=cfg.ffn, vocab=cfg.vocab, rope_theta=cfg.rope_theta, rms_eps=cfg.rms_eps,
                     max_model_len=cfg.max_model_len)
    eng = NativeEngine(mc, **kw)
    eng.load_weights(weights)
    eng.load_weight("tgis.rope_cos_sin", rope_table(cfg))
    return eng


def _ulp(x: float) -> float:
    """bf16 ulp at magnitude x"""
    return 2.0 ** (math.floor(math.log2(max(abs(x), 1e-6))) - 7)


# =========================================================================================== 8B dims, B=32, ctx 512
def test_8b_dims_stack_b32_ctx512_greedy_matches_oracle():
    from oracle.llama_oracle import LlamaOracle
    from vllm_tgis_adapter_b200.engine.core import make_sampling_params

    cfg = _cfg("8b2l")
    w = _weights("8b2l")
    rng = np.random.RandomState(3)
    B, P, n_new = 32, 512, 16
    prompts = [rng.randint(1000, cfg.vocab - 1000, size=P).tolist() for _ in range(B)]
    eng = _engine("8b2l", w, max_num_seqs=B, max_batched_tokens=2048, kv_cache_bytes=512 << 20)
    sp = make_sampling_params(greedy=True, max_tokens=n_new, min_tokens=n_new, num_logprobs=1, eos_token_id=2)
    outs = eng.generate_sync(prompts, sp)
    st = eng.status()
    eng.close()
    assert st.errored == 0 and st.graph_launches > 0
    toks = [[r.new_token for r in recs if r.new_token is not None] for recs in outs]
    assert all(len(t) == n_new for t in toks)

    ora = LlamaOracle(cfg, w, device="cuda")
    sts = [ora.new_seq() for _ in range(B)]
    logits = ora.step(list(zip(sts, prompts)))          # [B, V], teacher-forced on the engine's tokens below
    diffs, flips, rank_bad, steps, max_ulps = [], 0, 0, 0, 0.0
    for k in range(n_new):
        lp = torch.log_softmax(logits, -1)
        top2 = torch.topk(logits, 2, dim=-1).values
        for b in range(B):
            rec = [r for r in outs[b] if r.new_token is not None][k]
            u = _ulp(float(top2[b, 0]))
            margin = float(top2[b, 0] - top2[b, 1])
            otok = int(torch.argmax(logits[b]))
            d = abs(rec.logprob - float(lp[b, rec.new_token]))
            diffs.append(d)
            max_ulps = max(max_ulps, d / u)
            steps += 1
            if rec.new_token != otok:
                assert margin <= 2 * u + 1e-6, (b, k, margin, u)     # only a <= 2-ulp race may flip
                flips += 1
            elif margin > 2 * u:
                rank_bad += int(rec.rank != 1)
        logits = ora.step([(sts[b], [toks[b][k]]) for b in range(B)])
    diffs = np.array(diffs)
    _record_stats("8b2l_b32_ctx512_greedy_vs_oracle", {
        "steps": steps, "token_flips": flips, "logprob_absdiff_mean": float(diffs.mean()),
        "logprob_absdiff_p95": float(np.percentile(diffs, 95)), "logprob_absdiff_max": float(diffs.max()),
        "max_diff_in_logit_ulps": max_ulps, "frac_below_1e-3": float((diffs < 1e-3).mean()),
        "frac_exact": float((diffs == 0).mean())})
    assert rank_bad == 0
    assert flips <= steps // 10, (flips, steps)
    assert max_ulps <= 3.0, max_ulps
    assert float(diffs.mean()) < 0.5 * _ulp(4.0), float(diffs.mean())


# =========================================================================================== 8B dims, B=64, configs[2]
def test_8b_dims_stack_b64_cfg3_sampling_matches_oracle():
    from oracle import sampler_oracle as so
    from oracle.llama_oracle import LlamaOracle
    from vllm_tgis_adapter_b200.engine.core import make_sampling_params

    cfg = _cfg("8b2l")
    w = _weights("8b2l")
    rng = np.random.RandomState(4)
    B, P, n_new = 64, 48, 10
    prompts = [rng.randint(1000, cfg.vocab - 1000, size=P).tolist() for _ in range(B)]
    start, decay, rep, typ, min_new = 2, 1.3, 1.2, 0.9, 4
    eng = _engine("8b2l", w, max_num_seqs=B, max_batched_tokens=2048, kv_cache_bytes=256 << 20)
    sp = make_sampling_params(greedy=False, temperature=1.0, typical_p=typ, repetition_penalty=rep,
                              length_penalty=(start, decay), seed=1234, max_tokens=n_new, min_tokens=min_new,
                              eos_token_id=2, num_logprobs=1)
    outs = eng.generate_sync(prompts, sp)
    st = eng.status()
    eng.close()
    assert st.errored == 0
    toks = [[r.new_token for r in recs if r.new_token is not None] for recs in outs]
    assert all(min_new <= len(t) <= n_new for t in toks)
    ora = LlamaOracle(cfg, w, device="cuda")
    sts = [ora.new_seq() for _ in range(B)]
    logits = ora.step(list(zip(sts, prompts)))
    alive = list(range(B))
    same, total, lp_diffs, not_allowed = 0, 0, [], 0
    t0 = time.time()
    for k in range(n_new):
        rows = logits.float().cpu()
        for j, b in enumerate(alive):
            if k >= len(toks[b]):
                continue
            seen = torch.zeros(cfg.vocab, dtype=torch.bool)
            seen[torch.tensor(prompts[b] + toks[b][:k])] = True
            case = so.SamplingCase(greedy=False, temperature=1.0, typical_p=typ, repetition_penalty=rep,
                                   length_penalty=(start, decay), eos_token_id=2, min_tokens=min_new, n_out=k,
                                   num_logprobs=1, seed=1234)
            res = so.sample_row(rows[j], case, seen)
            rec = [r for r in outs[b] if r.new_token is not None][k]
            total += 1
            same += int(res["token"] == rec.new_token)
            if res["token"] != rec.new_token:
                not_allowed += int(not bool(res["allowed"][rec.new_token]))
            lp_diffs.append(abs(float(torch.log_softmax(rows[j], -1)[rec.new_token]) - rec.logprob))
        alive = [b for b in alive if k + 1 < len(toks[b])]
        if not alive:
            break
        logits = ora.step([(sts[b], [toks[b][k]]) for b in alive])
    lp_diffs = np.array(lp_diffs)
    _record_stats("8b2l_b64_cfg3_vs_oracle", {"rows": total, "same_token": same, "mismatch_outside_kept_set": not_allowed,
                                              "logprob_absdiff_mean": float(lp_diffs.mean()),
                                              "logprob_absdiff_max": float(lp_diffs.max()),
                                              "oracle_seconds": time.time() - t0})
    # identical logits would give identical tokens (kernel-level test); here the two stacks' bf16 logits differ by an ulp
    # in a fraction of the 128k entries, which can move the typical-p boundary or the winner of a close exponential race
    assert same >= 0.9 * total, (same, total)
    assert not_allowed <= max(1, total // 100), not_allowed
    assert float(lp_diffs.max()) <= 3.0 * _ulp(4.0)


# =========================================================================================== mixed lengths + preemption
def test_8b_dims_mixed_lengths_with_forced_preemption():
    """BASELINE configs[3] shape (mixed prompt lengths, continuous batching) on the 8B-dim stack with a KV cache that cannot
    hold all sequences: evicted sequences are recomputed (vLLM V1 policy) and every request still delivers its tokens;
    the token ids equal those of a roomy-cache run except where a recomputed prefix (prefill-shaped GEMM partition instead
    of the decode-shaped one) flips a bf16 near-tie."""
    from vllm_tgis_adapter_b200.engine.core import make_sampling_params

    cfg = _cfg("8b2l")
    w = _weights("8b2l")
    rng = np.random.RandomState(5)
    lens = rng.randint(64, 513, size=16)
    prompts = [rng.randint(1000, cfg.vocab - 1000, size=int(n)).tolist() for n in lens]
    n_new = 24
    sp = make_sampling_params(greedy=True, max_tokens=n_new, min_tokens=n_new, eos_token_id=2)
    eng = _engine("8b2l", w, max_num_seqs=16, max_batched_tokens=512, kv_cache_bytes=256 << 20)
    roomy = [[r.new_token for r in recs if r.new_token is not None] for recs in eng.generate_sync(prompts, sp)]
    st_r = eng.status()
    eng.close()
    assert st_r.preemptions == 0
    # one 32-token block = 2 layers * 8 kv heads * 32 * 128 * 2 B * 2 = 256 KiB; total need ~ sum(len + 24) / 32 blocks
    need = int(sum((n + n_new + 31) // 32 for n in lens))
    tight_blocks = max(int(0.45 * need), (512 + n_new) // 32 + 2)
    eng = _engine("8b2l", w, max_num_seqs=16, max_batched_tokens=512, kv_cache_bytes=int(tight_blocks * 262144 * 1.02))
    tight = [[r.new_token for r in recs if r.new_token is not None] for recs in eng.generate_sync(prompts, sp)]
    st_t = eng.status()
    eng.close()
    assert st_t.errored == 0 and st_t.preemptions > 0, st_t.preemptions
    assert all(len(t) == n_new for t in tight) and all(len(t) == n_new for t in roomy)
    prefix = sum(next((k for k, (x, y) in enumerate(zip(a, b)) if x != y), n_new) for a, b in zip(roomy, tight))
    _record_stats("8b2l_preemption", {"preemptions": int(st_t.preemptions), "matching_prefix_tokens": prefix,
                                      "total": n_new * len(prompts),
                                      "identical_requests": sum(int(a == b) for a, b in zip(roomy, tight))})
    # measured: 11 of 16 requests identical, 83 % matching prefix with ONE preemption -- on this synthetic checkpoint a
    # quarter of the greedy steps have a top-2 margin of <= 1 bf16 ulp of the logits (N(0, 1.3) logits over a 128k
    # vocabulary), so any change of summation order flips a token within a few steps (vLLM against itself, batched vs
    # one request at a time, diverges the same way)
    assert prefix >= 0.6 * n_new * len(prompts), prefix


# =========================================================================================== abort on the real engine
def test_abort_mid_generation_frees_the_sequence():
    """tgis_engine_abort on the threaded engine (reference: `await engine.abort(request_id)`, grpc_server.py:292,388):
    the request ends with an ABORT record, its KV blocks return to the pool, other requests are unaffected."""
    from vllm_tgis_adapter_b200.engine import _lib
    from vllm_tgis_adapter_b200.engine.core import make_sampling_params

    w = _weights("tiny", seed=3)
    eng = _engine("tiny", w, max_num_seqs=4, max_batched_tokens=256, kv_cache_bytes=16 << 20)
    total_blocks = eng.status().total_blocks
    eng.start()
    sp_long = make_sampling_params(greedy=True, max_tokens=400, min_tokens=400, eos_token_id=2)
    sp_short = make_sampling_params(greedy=True, max_tokens=30, min_tokens=30, eos_token_id=2)
    eng.add_request("victim", list(range(10, 50)), sp_long)
    eng.add_request("bystander", list(range(60, 90)), sp_short)
    got = {"victim": [], "bystander": []}
    finish = {}
    aborted_at = None
    deadline = time.time() + 60
    while time.time() < deadline and len(finish) < 2:
        for o in eng.poll(50):
            if o.new_token is not None:
                got[o.request_id].append(o.new_token)
            if o.finish_reason != _lib.FINISH_NONE:
                finish[o.request_id] = o.finish_reason
        if aborted_at is None and len(got["victim"]) >= 5:
            aborted_at = len(got["victim"])
            eng.abort("victim")
            eng.abort("no-such-request")     # idempotent / unknown ids are ignored
    assert finish.get("victim") == _lib.FINISH_ABORT, finish
    assert finish.get("bystander") == _lib.FINISH_LENGTH and len(got["bystander"]) == 30
    assert aborted_at is not None and aborted_at <= len(got["victim"]) < 400
    deadline = time.time() + 5       # the records are emitted inside the step; its bookkeeping ends a moment later
    while time.time() < deadline:
        st = eng.status()
        if st.n_running == 0 and st.free_blocks == total_blocks:
            break
        time.sleep(0.01)
    assert st.n_running == 0 and st.free_blocks == total_blocks, (st.free_blocks, total_blocks)
    # the engine keeps serving afterwards
    eng.add_request("after", list(range(100, 120)), sp_short)
    n_after, done = 0, False
    deadline = time.time() + 30
    while time.time() < deadline and not done:
        for o in eng.poll(50):
            n_after += int(o.new_token is not None)
            done = done or o.finish_reason != _lib.FINISH_NONE
    assert done and n_after == 30
    eng.close()


# =========================================================================================== vLLM fixtures
def _request_sets(vocab):
    rng = np.random.RandomState(0)
    greedy = [rng.randint(3, vocab, size=n).tolist() for n in (5, 33, 64, 100, 17, 250)]
    rng = np.random.RandomState(7)
    plp = [rng.randint(3, vocab, size=96).tolist() for _ in range(4)]
    rng = np.random.RandomState(11)
    lenpen = [rng.randint(3, vocab, size=n).tolist() for n in (12, 40, 77)]
    return greedy, plp, lenpen


# logit magnitude class of each synthetic checkpoint -> bf16 ulp of its top logits
_TOP_LOGIT = {"tiny": 1.0, "small": 2.0, "8b2l": 4.0}


@pytest.mark.parametrize("name", ["tiny", "small", "8b2l"])
def test_engine_matches_vllm_fixture(name):
    """Engine vs what vLLM 0.22.0 produced on a GPU for the same checkpoint and requests (tests/golden/vllm_<name>.json,
    scripts/vllm_crosscheck.py).  Greedy token ids must agree up to the first step where vLLM's own top-2 logprob
    margin is within 2 bf16 ulps; logprobs within 3 ulps of the logits, ranks equal off ties."""
    from vllm_tgis_adapter_b200.engine.core import make_sampling_params

    path = GOLD / f"vllm_{name}.json"
    if not path.exists():
        pytest.skip(f"{path.name} not generated yet (scripts/vllm_crosscheck.py check on the GPU box)")
    fx = json.loads(path.read_text())
    assert fx["meta"]["weights_seed"] == 1
    cfg = _cfg(name)
    w = _weights(name)
    greedy, plp, lenpen = _request_sets(cfg.vocab)
    u = _ulp(_TOP_LOGIT[name])
    eng = _engine(name, w, max_num_seqs=16, max_batched_tokens=2048, kv_cache_bytes=256 << 20)
    n_new = len(fx["greedy"][0]["tokens"])
    sp = make_sampling_params(greedy=True, max_tokens=n_new, min_tokens=n_new, num_logprobs=3, eos_token_id=2)
    outs = eng.generate_sync(greedy, sp)
    diffs, flips, rank_bad, compared = [], 0, 0, 0
    for recs, v in zip(outs, fx["greedy"]):
        recs = [r for r in recs if r.new_token is not None]
        for k, (r, vt, vs) in enumerate(zip(recs, v["tokens"], v["steps"])):
            top = sorted(vs["top"], key=lambda t: -t[1])
            margin = top[0][1] - top[1][1] if len(top) > 1 else 1.0
            if r.new_token != vt:
                assert margin <= 2 * u + 1e-6, (name, k, margin, u)
                flips += 1
                break   # the continuations are different sequences from here on
            diffs.append(abs(r.logprob - vs["logprob"]))
            compared += 1
            if margin > 2 * u:
                rank_bad += int(r.rank != vs["rank"])
    # prompt logprobs: teacher-forced by construction
    sp = make_sampling_params(greedy=True, max_tokens=1, num_logprobs=2, prompt_logprobs=2, eos_token_id=2)
    outs = eng.generate_sync(plp, sp)
    pdiffs, prank_close = [], 0
    for p, recs, v in zip(plp, outs, fx["plp"]):
        pos = {r.prompt_pos: r for r in recs if r.prompt_pos >= 1}
        for i, vp in zip(range(1, len(p)), v["positions"]):
            pdiffs.append(abs(pos[i].logprob - vp["logprob"]))
            # a 1-ulp move of the token's own logit shifts its rank by the number of entries inside that ulp
            prank_close += int(abs(pos[i].rank - vp["rank"]) <= max(3, vp["rank"] // 20))
    # decode tokens teacher-forced: vLLM's own continuations scored by the engine (prompt-logprob pass over prompt +
    # vLLM's tokens), so every one of vLLM's steps is compared even after the free-running sequences part ways
    seqs = [p + v["tokens"] for p, v in zip(greedy, fx["greedy"])]
    sp = make_sampling_params(greedy=True, max_tokens=1, num_logprobs=1, prompt_logprobs=1, eos_token_id=2)
    outs = eng.generate_sync(seqs, sp)
    tf_diffs, tf_argmax_bad = [], 0
    for p, v, recs in zip(greedy, fx["greedy"], outs):
        pos = {r.prompt_pos: r for r in recs if r.prompt_pos >= 1}
        for k, (vt, vs) in enumerate(zip(v["tokens"], v["steps"])):
            r = pos[len(p) + k]
            tf_diffs.append(abs(r.logprob - vs["logprob"]))
            top = sorted(vs["top"], key=lambda t: -t[1])
            margin = top[0][1] - top[1][1] if len(top) > 1 else 1.0
            if margin > 2 * u:      # a clear winner for vLLM must be the engine's top-1 as well
                tf_argmax_bad += int(r.topn[0][0] != vt)
    tf_diffs = np.array(tf_diffs)
    # ExpDecay length penalty through vLLM's processor hook
    lp_rows = []
    if "lenpen" in fx:
        sp = make_sampling_params(greedy=True, max_tokens=48, num_logprobs=1, eos_token_id=2, length_penalty=(6, 1.35))
        outs = eng.generate_sync(lenpen, sp)
        for recs, v in zip(outs, fx["lenpen"]):
            t = [r.new_token for r in recs if r.new_token is not None]
            lp_rows.append((t, v["tokens"]))
    eng.close()
    diffs, pdiffs = np.array(diffs), np.array(pdiffs)
    _record_stats(f"vllm_fixture_{name}", {
        "decode_steps_compared": compared, "first_divergences": flips,
        "decode_logprob_absdiff_mean": float(diffs.mean()), "decode_logprob_absdiff_max": float(diffs.max()),
        "decode_rank_mismatch_off_ties": rank_bad,
        "prompt_positions": int(pdiffs.size), "prompt_logprob_absdiff_mean": float(pdiffs.mean()),
        "prompt_logprob_absdiff_max": float(pdiffs.max()), "prompt_rank_close": prank_close,
        "teacher_forced_steps": int(tf_diffs.size), "teacher_forced_logprob_absdiff_mean": float(tf_diffs.mean()),
        "teacher_forced_logprob_absdiff_max": float(tf_diffs.max()), "teacher_forced_argmax_mismatch_off_ties": tf_argmax_bad,
        "lenpen_equal": [a == b for a, b in lp_rows], "ulp": u})
    # free-running prefixes: short on the 8B-dim checkpoint (a quarter of its greedy steps are <= 1-ulp races, and vLLM
    # against itself diverges the same way); the teacher-forced leg covers all of vLLM's steps
    assert compared >= (0.25 if name == "8b2l" else 0.6) * sum(len(v["tokens"]) for v in fx["greedy"]), compared
    assert tf_diffs.size == sum(len(v["tokens"]) for v in fx["greedy"]) and tf_argmax_bad == 0
    assert float(tf_diffs.max()) <= 3 * u and float(tf_diffs.mean()) <= 0.6 * u, (float(tf_diffs.max()), float(tf_diffs.mean()))
    assert rank_bad == 0
    assert float(diffs.max()) <= 3 * u and float(diffs.mean()) <= 0.6 * u, (float(diffs.max()), float(diffs.mean()), u)
    assert float(pdiffs.max()) <= 4 * u and float(pdiffs.mean()) <= 0.6 * u, (float(pdiffs.max()), float(pdiffs.mean()))
    assert prank_close >= 0.95 * pdiffs.size, (prank_close, pdiffs.size)
    for a, b in lp_rows:
        # same EOS step (or both ran to max_tokens), identical ids up to a possible near-tie flip
        assert (a[-1] == 2) == (b[-1] == 2)
        k = next((i for i, (x, y) in enumerate(zip(a, b)) if x != y), min(len(a), len(b)))
        assert k >= min(len(a), len(b)) // 2 or a == b
