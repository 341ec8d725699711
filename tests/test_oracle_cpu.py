"""Pin the CPU oracle against golden vectors produced by the reference's own code (oracle/gen_golden.py):
the reference's logits_processors.py, transformers' TypicalLogitsWarper / LlamaForCausalLM and vLLM 0.22's sampler ops.
Runs on the GPU-less box and on the GPU box (no access to /root/reference needed)."""
import json
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import sampler_oracle as so
from oracle.llama_oracle import CONFIGS, LlamaOracle, synthetic_weights

GOLD = Path(__file__).resolve().parent / "golden"


@pytest.fixture(scope="module")
def fx():
    return json.loads((GOLD / "sampler_reference.json").read_text())


def t32(x):
    return torch.tensor(x, dtype=torch.float32)


def test_exp_decay_matches_reference_processor(fx):
    for c in fx["exp_decay"]:
        logits = t32(c["logits"])
        so.exp_decay_length_penalty(logits, c["n_out"], c["start"], c["decay"], c["eos"])
        assert float(logits[c["eos"]]) == c["eos_out"], c       # bit-exact fp32
        # and the host->kernel factor reproduces it with two rounded fp32 ops (what csrc/sampler.cu does)
        x = np.float32(c["logits"][c["eos"]])
        f = np.float32(so.len_penalty_factor_m1(c["n_out"], c["start"], c["decay"]))
        y = np.float32(x + np.float32(np.abs(x) * f)) if f != 0 else x
        assert float(y) == c["eos_out"]


def test_typical_mask_matches_reference_processor(fx):
    for c in fx["typical"]:
        logits = t32(c["logits"])
        keep = so.typical_keep_mask(logits, c["mass"])
        assert torch.nonzero(~keep).flatten().tolist() == c["removed"]


def test_repetition_penalty_matches_vllm(fx):
    for c in fx["rep_penalty"]:
        logits = t32(c["logits"])
        seen = torch.zeros(fx["vocab"], dtype=torch.bool)
        seen[c["seen"]] = True
        so.apply_repetition_penalty(logits, seen, c["penalty"])
        # vLLM's torch path multiplies by 1/penalty where its CUDA op (the one that runs on GPU, and the one restated
        # here) divides: identical up to 1 fp32 ulp on positive seen logits
        np.testing.assert_allclose(logits.numpy(), np.array(c["out"], dtype=np.float32), rtol=2e-7, atol=0)


def test_topk_topp_matches_vllm(fx):
    for c in fx["topk_topp"]:
        out = so.topk_topp_mask(t32(c["logits"]), c["k"] or 0, c["p"] if c["p"] is not None else 1.0)
        assert torch.nonzero(torch.isfinite(out)).flatten().tolist() == c["kept"], (c["k"], c["p"])


def test_logprobs_rank_topn_match_vllm(fx):
    V = fx["vocab"]
    for c in fx["logprobs"]:
        logits = t32(c["logits"]).view(2, V)
        for row in range(2):
            lp = torch.log_softmax(logits[row], -1)
            tok = c["tokens"][row]
            assert int((lp >= lp[tok]).sum()) == c["ranks"][row]
            top = torch.topk(lp, c["n"])
            assert c["ids"][row][0] == tok and c["ids"][row][1:] == top.indices.tolist()
            np.testing.assert_allclose([float(lp[tok])] + top.values.tolist(), c["lps"][row], atol=1e-6)
            res = so.sample_row(logits[row], so.SamplingCase(greedy=True, num_logprobs=c["n"]))
            if row == 0:
                assert res["token"] == tok and res["rank"] == c["ranks"][0]


def test_philox_reference_vector():
    """Known-answer test of Philox4x32-10 (Random123 kat: counter 0, key 0 -> 6627e8d5 e169c58d bc57ac4c 9b00dbd8)."""
    u = so.philox_uniform(1, 0, 0)
    assert abs(float(u[0]) - ((0x6627e8d5 >> 8) + 0.5) / 16777216.0) < 1e-9


def test_llama_oracle_matches_hf_fixture_fp32():
    g = json.loads((GOLD / "llama_tiny_hf_fp32.json").read_text())
    cfg = CONFIGS[g["config"]]
    w = synthetic_weights(cfg, seed=g["weights_seed"], dtype=torch.float32)
    ora = LlamaOracle(cfg, w, dtype=torch.float32)
    st = ora.new_seq()
    logits = ora.step([(st, g["prompt"])], want_all_logits=True)
    assert logits.argmax(-1).tolist() == g["argmax_per_pos"]
    np.testing.assert_allclose(torch.logsumexp(logits, -1).numpy(), np.array(g["logsumexp_per_pos"]), atol=2e-4)
    np.testing.assert_allclose(logits[-1, :32].numpy(), np.array(g["last_logits_head"]), atol=2e-4)


def test_llama_oracle_bf16_rounding_points_match_hf_bf16_fixture():
    """The oracle in bf16 vs transformers' LlamaForCausalLM run in bf16 (tests/golden/llama_hf_bf16.json): same rounding
    points => logits agree to a few bf16 ulps (the two differ only in fp32 summation order inside the matmuls), and
    greedy argmax agrees wherever HF's own top-2 margin exceeds that."""
    g = json.loads((GOLD / "llama_hf_bf16.json").read_text())
    for case in g["cases"]:
        cfg = CONFIGS[case["config"]]
        w = synthetic_weights(cfg, seed=case["weights_seed"])
        ora = LlamaOracle(cfg, w)
        logits = ora.step([(ora.new_seq(), case["prompt"])], want_all_logits=True)
        # every value is a bf16 number (the sampler's fp32 view of model-dtype logits)
        assert torch.equal(logits, logits.to(torch.bfloat16).float())
        last = torch.tensor(case["last_logits"])
        d = (logits[-1] - last).abs()
        # measured: max |diff| = 1-2 bf16 ulps at the row's magnitude, mean ~0.3 ulp, 20-26 % of the logits bit-identical
        # (HF's CPU matmuls and the oracle's sum the same fp32 products in different orders; upstream bf16 roundings
        # that land on the other side of a tie move a logit by one ulp)
        ulp_row = 2.0 ** (torch.floor(torch.log2(last.abs().max())).item() - 7)
        assert float(d.max()) <= 2.0 * ulp_row, (float(d.max()), ulp_row)
        assert float(d.mean()) < 0.5 * ulp_row
        assert float((d == 0).float().mean()) > 0.15
        mid = torch.tensor(case["mid_logits_head"])
        dm = (logits[len(case["prompt"]) // 2, :256] - mid).abs()
        assert float(dm.max()) < 0.05
        np.testing.assert_allclose(torch.logsumexp(logits, -1).numpy(), np.array(case["logsumexp_per_pos"]), atol=1e-2)
        am = logits.argmax(-1).tolist()
        for pos, (a, b, m) in enumerate(zip(am, case["argmax_per_pos"], case["top2_margin_per_pos"])):
            if m > 0.04:
                assert a == b, (case["config"], pos, a, b, m)


def test_llama_oracle_incremental_equals_prefill_and_bf16_is_close():
    cfg = CONFIGS["tiny"]
    w = synthetic_weights(cfg, seed=4)
    prompt = list(range(40, 75))
    ora32 = LlamaOracle(cfg, {k: v.float() for k, v in w.items()}, dtype=torch.float32)
    full = ora32.step([(ora32.new_seq(), prompt)], want_all_logits=True)
    st = ora32.new_seq()
    ora32.step([(st, prompt[:20])])
    inc = [ora32.step([(st, [t])])[0] for t in prompt[20:]]
    np.testing.assert_allclose(torch.stack(inc).numpy(), full[20:].numpy(), atol=2e-5)
    ora16 = LlamaOracle(cfg, w)
    l16 = ora16.step([(ora16.new_seq(), prompt)], want_all_logits=True)
    assert float((l16 - full).abs().max()) < 0.05         # bf16 rounding points only


def test_check_stop_order():
    kw = dict(eos=2, min_tokens=0, max_tokens=5, max_model_len=100)
    assert so.check_stop(1, 2, 10, **kw) == ("stop", None)
    assert so.check_stop(1, 9, 10, stop_token_ids=(9,), **kw) == ("stop", 9)
    assert so.check_stop(5, 7, 10, **kw) == ("length", None)
    assert so.check_stop(1, 2, 10, eos=2, min_tokens=3, max_tokens=5, max_model_len=100) == (None, None)
    assert so.check_stop(2, 7, 100, **kw) == ("length", None)


@pytest.mark.parametrize("name,top_logit", [("tiny", 1.0), ("small", 2.0)])
def test_llama_oracle_matches_vllm_fixture(name, top_logit):
    """The oracle against what the reference's REAL engine path produced: vLLM 0.22.0 on a GPU running the same seeded
    checkpoint and requests (tests/golden/vllm_<name>.json, written by scripts/vllm_crosscheck.py on the GPU box).
    Teacher-forced on vLLM's tokens: logprobs within 2 bf16 ulps of the logits (mean < 0.6 ulp), greedy argmax equal
    wherever vLLM's own top-2 margin exceeds 2 ulps, prompt-token ranks within the tie band.  (vLLM against itself --
    one batch vs one request at a time -- differs by up to 1 ulp on the 8B-dim stack.)"""
    import math

    fx = json.loads((GOLD / f"vllm_{name}.json").read_text())
    cfg = CONFIGS[name]
    w = synthetic_weights(cfg, seed=fx["meta"]["weights_seed"])
    ora = LlamaOracle(cfg, w)
    u = 2.0 ** (math.floor(math.log2(top_logit)) - 7)
    rng = np.random.RandomState(0)
    greedy = [rng.randint(3, cfg.vocab, size=n).tolist() for n in (5, 33, 64, 100, 17, 250)]
    rng = np.random.RandomState(7)
    plp = [rng.randint(3, cfg.vocab, size=96).tolist() for _ in range(4)]
    diffs, flips_ok, steps = [], 0, 0
    for p, v in zip(greedy, fx["greedy"]):
        st = ora.new_seq()
        logits = ora.step([(st, p)])[0]
        for tok, vs in zip(v["tokens"], v["steps"]):
            lp = torch.log_softmax(logits, -1)
            top = sorted(vs["top"], key=lambda t: -t[1])
            margin = top[0][1] - top[1][1]
            diffs.append(abs(float(lp[tok]) - vs["logprob"]))
            steps += 1
            if int(torch.argmax(logits)) != tok:
                assert margin <= 2 * u + 1e-6, (name, margin)
                flips_ok += 1
            elif margin > 2 * u:
                assert int((lp >= lp[tok]).sum()) == vs["rank"]
            logits = ora.step([(st, [tok])])[0]
    diffs = np.array(diffs)
    assert float(diffs.max()) <= 2 * u + 1e-4 and float(diffs.mean()) <= 0.6 * u, (float(diffs.max()), float(diffs.mean()))
    assert flips_ok <= steps // 10
    pd, close, n = [], 0, 0
    for p, v in zip(plp, fx["plp"]):
        lp = torch.log_softmax(ora.step([(ora.new_seq(), p)], want_all_logits=True), -1)
        for i, vp in zip(range(1, len(p)), v["positions"]):
            row = lp[i - 1]
            pd.append(abs(float(row[p[i]]) - vp["logprob"]))
            # rank band: entries within 1.5 ulp of the token's logprob may fall on either side
            lo = int((row > row[p[i]] + 1.5 * u).sum()) + 1
            hi = int((row >= row[p[i]] - 1.5 * u).sum())
            close += int(lo <= vp["rank"] <= hi)
            n += 1
    pd = np.array(pd)
    assert float(pd.max()) <= 2 * u + 1e-4 and float(pd.mean()) <= 0.6 * u, (float(pd.max()), float(pd.mean()))
    assert close >= 0.99 * n, (close, n)
