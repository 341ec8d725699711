"""Pin the OPT oracle (oracle/opt_oracle.py) against transformers' OPTForCausalLM run in this container
(oracle/gen_opt_golden.py -> tests/golden/opt_hf_{fp32,bf16}.json).  The reference's OPT fixture is facebook/opt-125m
(/root/reference/tests/conftest.py:79-91 (no --model: vLLM's default, facebook/opt-125m) and tests/test_hub.py:17); the fixtures carry seeded random weights of that architecture."""
import dataclasses
import json
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle.opt_oracle import OPT_CONFIGS, OPTOracle, synthetic_opt_weights

GOLD = Path(__file__).resolve().parent / "golden"


def case_cfg(name):
    if name == "opt-125m-2l":
        return dataclasses.replace(OPT_CONFIGS["opt-125m"], n_layers=2)
    return OPT_CONFIGS[name]


def test_opt_oracle_matches_hf_fp32_fixture_prefill_and_cached_decode():
    g = json.loads((GOLD / "opt_hf_fp32.json").read_text())
    for c in g["cases"]:
        cfg = case_cfg(c["config"])
        ora = OPTOracle(cfg, synthetic_opt_weights(cfg, seed=c["weights_seed"]), dtype=torch.float32)
        st = ora.new_seq()
        logits = ora.step([(st, c["prompt"])], want_all_logits=True)
        assert logits.argmax(-1).tolist() == c["argmax_per_pos"]
        np.testing.assert_allclose(torch.logsumexp(logits, -1).numpy(), np.array(c["logsumexp_per_pos"]), atol=2e-5)
        np.testing.assert_allclose(logits[-1, :512].numpy(), np.array(c["last_logits_head"]), atol=2e-5)
        np.testing.assert_allclose(logits[len(c["prompt"]) // 2, :256].numpy(), np.array(c["mid_logits_head"]), atol=2e-5)
        # HF's KV-cache decode: one position per call, teacher-forced on HF's own greedy tokens
        for i, tok in enumerate(c["decode_tokens"]):
            row = ora.step([(st, [tok])])[0]
            np.testing.assert_allclose(row[:128].numpy(), np.array(c["decode_logits_head"][i]), atol=2e-5)
            assert abs(float(torch.logsumexp(row, -1)) - c["decode_logsumexp"][i]) < 2e-5
            if i + 1 < len(c["decode_tokens"]):
                assert int(row.argmax()) == c["decode_tokens"][i + 1]


def test_opt_oracle_bf16_rounding_points_match_hf_bf16_fixture():
    """Same rounding points as HF's bf16 run => logits within 2 bf16 ulps of the row's magnitude (fp32 summation order
    inside the matmuls differs), a good share bit-identical, argmax equal off ties."""
    g = json.loads((GOLD / "opt_hf_bf16.json").read_text())
    for c in g["cases"]:
        cfg = case_cfg(c["config"])
        ora = OPTOracle(cfg, synthetic_opt_weights(cfg, seed=c["weights_seed"]))
        st = ora.new_seq()
        logits = ora.step([(st, c["prompt"])], want_all_logits=True)
        assert torch.equal(logits, logits.to(torch.bfloat16).float())
        last = torch.tensor(c["last_logits_head"])
        ulp = 2.0 ** (torch.floor(torch.log2(logits[-1].abs().max())).item() - 7)
        d = (logits[-1, :512] - last).abs()
        assert float(d.max()) <= 2.0 * ulp, (float(d.max()), ulp)
        assert float(d.mean()) < 0.5 * ulp
        assert float((d == 0).float().mean()) > 0.15
        np.testing.assert_allclose(torch.logsumexp(logits, -1).numpy(), np.array(c["logsumexp_per_pos"]), atol=5e-3)
        for pos, (a, b, m) in enumerate(zip(logits.argmax(-1).tolist(), c["argmax_per_pos"], c["top2_margin_per_pos"])):
            if m > 2.0 * ulp:
                assert a == b, (c["config"], pos, a, b, m)
        for i, tok in enumerate(c["decode_tokens"]):
            row = ora.step([(st, [tok])])[0]
            dd = (row[:128] - torch.tensor(c["decode_logits_head"][i])).abs()
            assert float(dd.max()) <= 2.0 * ulp
            assert abs(float(torch.logsumexp(row, -1)) - c["decode_logsumexp"][i]) < 5e-3


def test_opt_oracle_incremental_equals_prefill():
    cfg = OPT_CONFIGS["opt-tiny"]
    w = synthetic_opt_weights(cfg, seed=5)
    prompt = list(range(40, 75))
    a = OPTOracle(cfg, w, dtype=torch.float32)
    full = a.step([(a.new_seq(), prompt)], want_all_logits=True)
    b = OPTOracle(cfg, w, dtype=torch.float32)
    st = b.new_seq()
    rows = [b.step([(st, prompt[:20])])[0]]
    for t in prompt[20:]:
        rows.append(b.step([(st, [t])])[0])
    np.testing.assert_allclose(torch.stack(rows).numpy(), full[19:].numpy(), atol=1e-5)
    # two sequences in one flat batch do not see each other
    c = OPTOracle(cfg, w, dtype=torch.float32)
    two = c.step([(c.new_seq(), prompt), (c.new_seq(), prompt[:11])])
    np.testing.assert_allclose(two[0].numpy(), full[-1].numpy(), atol=1e-5)
    np.testing.assert_allclose(two[1].numpy(), full[10].numpy(), atol=1e-5)


def test_loader_maps_opt_config_json_and_refuses_unsupported_variants(tmp_path):
    """Host side of the OPT family (engine/loader.py): facebook/opt-125m's config.json keys -> ModelConfig(arch="opt");
    the variants that need modules the engine does not have (opt-350m: post-LayerNorm, project_in/out) fail at start-up
    like an unsupported architecture does in the reference's engine, not at request time."""
    import pytest

    from vllm_tgis_adapter_b200.engine.core import PRESETS
    from vllm_tgis_adapter_b200.engine.loader import model_config_from_hf

    opt125m = {"architectures": ["OPTForCausalLM"], "model_type": "opt", "hidden_size": 768, "num_hidden_layers": 12,
               "num_attention_heads": 12, "ffn_dim": 3072, "vocab_size": 50272, "max_position_embeddings": 2048,
               "word_embed_proj_dim": 768, "do_layer_norm_before": True, "activation_function": "relu",
               "enable_bias": True, "layer_norm_elementwise_affine": True, "_remove_final_layer_norm": False}
    (tmp_path / "config.json").write_text(json.dumps(opt125m))
    mc = model_config_from_hf(tmp_path, None)
    assert mc == PRESETS["opt-125m"]
    assert model_config_from_hf(tmp_path, 512).max_model_len == 512
    with pytest.raises(ValueError, match="max_position_embeddings"):
        model_config_from_hf(tmp_path, 4096)
    opt350m = {**opt125m, "hidden_size": 1024, "num_attention_heads": 16, "ffn_dim": 4096, "num_hidden_layers": 24,
               "word_embed_proj_dim": 512, "do_layer_norm_before": False}
    (tmp_path / "config.json").write_text(json.dumps(opt350m))
    with pytest.raises(ValueError, match="unsupported OPT variant"):
        model_config_from_hf(tmp_path, None)


def _vllm_request_sets(vocab):
    rng = np.random.RandomState(0)
    greedy = [rng.randint(3, vocab, size=n).tolist() for n in (5, 33, 64, 100, 17, 250)]
    rng = np.random.RandomState(7)
    plp = [rng.randint(3, vocab, size=96).tolist() for _ in range(4)]
    return greedy, plp


@pytest.mark.parametrize("name,top_logit", [("opt-tiny", 1.0), ("opt-125m", 2.0)])
def test_opt_oracle_matches_vllm_fixture(name, top_logit):
    """The OPT oracle against the reference's REAL engine path: vLLM 0.22.0 (its own OPTForCausalLM, FlashInfer) on a GPU
    over the same seeded checkpoint and requests (tests/golden/vllm_<name>.json, scripts/vllm_crosscheck.py check --configs
    opt-tiny opt-125m).  Teacher-forced on vLLM's tokens, in bf16 ulps of the logits, like the Llama fixtures."""
    import math

    path = GOLD / f"vllm_{name}.json"
    if not path.exists():
        pytest.skip(f"{path.name} not generated yet (scripts/vllm_crosscheck.py check on the GPU box)")
    fx = json.loads(path.read_text())
    cfg = dataclasses.replace(OPT_CONFIGS[name], max_model_len=1024) if name == "opt-125m" else OPT_CONFIGS[name]
    ora = OPTOracle(cfg, synthetic_opt_weights(cfg, seed=fx["meta"]["weights_seed"]))
    u = 2.0 ** (math.floor(math.log2(top_logit)) - 7)
    greedy, plp = _vllm_request_sets(cfg.vocab)
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
    assert float(diffs.max()) <= 3 * u + 1e-4 and float(diffs.mean()) <= 0.6 * u, (float(diffs.max()), float(diffs.mean()))
    assert flips_ok <= steps // 10
    pd = []
    for p, v in zip(plp, fx["plp"]):
        lp = torch.log_softmax(ora.step([(ora.new_seq(), p)], want_all_logits=True), -1)
        for i, vp in zip(range(1, len(p)), v["positions"]):
            pd.append(abs(float(lp[i - 1, p[i]]) - vp["logprob"]))
    pd = np.array(pd)
    assert float(pd.max()) <= 3 * u + 1e-4 and float(pd.mean()) <= 0.6 * u, (float(pd.max()), float(pd.mean()))


def test_loader_streams_a_pytorch_model_bin_directory(tmp_path):
    """facebook/opt-125m ships `pytorch_model.bin` (no safetensors): the loader must stream it tensor by tensor under the
    checkpoint's own names, and refuse a directory with neither format."""
    from vllm_tgis_adapter_b200.engine.loader import load_safetensors_dir

    class Recorder:
        def __init__(self):
            self.seen = {}

        def load_weight(self, name, t):
            self.seen[name] = tuple(t.shape)

    cfg = OPT_CONFIGS["opt-tiny"]
    w = synthetic_opt_weights(cfg, seed=3)
    torch.save({**w, "lm_head.weight": w["model.decoder.embed_tokens.weight"]}, tmp_path / "pytorch_model.bin")
    rec = Recorder()
    load_safetensors_dir(rec, tmp_path)
    assert set(rec.seen) == set(w) | {"lm_head.weight"}
    assert rec.seen["model.decoder.embed_positions.weight"] == (cfg.max_positions + 2, cfg.hidden)
    assert rec.seen["model.decoder.layers.1.fc1.bias"] == (cfg.ffn,)
    (tmp_path / "pytorch_model.bin").unlink()
    with pytest.raises(ValueError, match="safetensors or pytorch_model"):
        load_safetensors_dir(rec, tmp_path)
