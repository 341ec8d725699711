"""Phi-3 on the host side: config.json mapping (both rope spellings, the three LongRoPE type names, the window), the
refusals, the fused-tensor split, the LongRoPE table (the short / long choice at max_model_len = original and
original + 1, and mscale), the test oracle against transformers' Phi3ForCausalLM (tests/golden/phi3_hf_*.json,
scripts/gen_phi3_golden.py), and the ABI.  No GPU."""
import argparse
import ctypes as C
import dataclasses
import json
import math
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

from phi3_oracle import Phi3Config, Phi3Oracle, fuse, longrope_table, synthetic_weights

ROOT = Path(__file__).resolve().parent.parent
GOLD = ROOT / "tests" / "golden"
LONG = [1.0 + 0.1 * i for i in range(48)]
SHORT = [1.0 + 0.01 * i for i in range(48)]


def _phi3_json(**over) -> dict:
    """microsoft/Phi-3-mini-128k-instruct's config.json (transformers 4 spelling), as recalled, with stand-in factors"""
    cfg = {"architectures": ["Phi3ForCausalLM"], "model_type": "phi3", "hidden_size": 3072, "num_attention_heads": 32,
           "num_key_value_heads": 32, "num_hidden_layers": 32, "intermediate_size": 8192, "vocab_size": 32064,
           "max_position_embeddings": 131072, "original_max_position_embeddings": 4096, "rms_norm_eps": 1e-5,
           "rope_theta": 10000.0, "sliding_window": 262144, "tie_word_embeddings": False,
           "rope_scaling": {"type": "longrope", "long_factor": LONG, "short_factor": SHORT}}
    cfg.update(over)
    return cfg


def _read(tmp_path, cfg, max_model_len=None):
    from vllm_tgis_adapter_b200.engine.loader import model_config_from_hf

    (tmp_path / "config.json").write_text(json.dumps(cfg))
    return model_config_from_hf(tmp_path, max_model_len)


# ------------------------------------------------------------------------------------------------ config.json mapping
@pytest.mark.parametrize("kind", ["longrope", "su", "yarn"])
@pytest.mark.parametrize("spelling", ["rope_scaling", "rope_parameters"])
def test_loader_maps_longrope_in_every_spelling(tmp_path, kind, spelling):
    rope = {"rope_type": kind, "long_factor": LONG, "short_factor": SHORT}
    cfg = _phi3_json(rope_scaling=None)
    if spelling == "rope_parameters":   # transformers 5: theta and the original length inside rope_parameters
        del cfg["rope_theta"], cfg["original_max_position_embeddings"]
        rope.update(rope_theta=10000.0, original_max_position_embeddings=4096)
    cfg[spelling] = rope
    mc = _read(tmp_path, cfg)
    assert (mc.head_dim, mc.n_q_heads, mc.n_kv_heads, mc.vocab, mc.rope_theta) == (96, 32, 32, 32064, 10000.0)
    assert mc.rope_long_factor == tuple(LONG) and mc.rope_short_factor == tuple(SHORT)
    assert (mc.rope_original_max_pos, mc.rope_max_position_embeddings) == (4096, 131072)
    assert mc.rope_longrope and mc.rope_scaled and mc.fused_projections
    assert mc.max_model_len == 8192 and mc.sliding_window == 262144


def test_loader_maps_phi3_mini_4k_onto_the_preset(tmp_path):
    from vllm_tgis_adapter_b200.engine.core import PRESETS

    cfg = _phi3_json(max_position_embeddings=4096, sliding_window=2047, rope_scaling=None)
    mc = _read(tmp_path, cfg)
    assert mc == dataclasses.replace(PRESETS["phi3-mini-4k"], sliding_window=2047)   # the presets carry no window
    assert not mc.rope_longrope and not mc.rope_scaled


def test_phi4_and_medium_shapes_and_a_null_window(tmp_path):
    from vllm_tgis_adapter_b200.engine.core import PRESETS

    cfg = _phi3_json(hidden_size=5120, num_attention_heads=40, num_key_value_heads=10, num_hidden_layers=40,
                     intermediate_size=17920, vocab_size=100352, max_position_embeddings=16384, rope_theta=250000.0,
                     sliding_window=None, rope_scaling=None)
    mc = _read(tmp_path, cfg, 16384)
    assert mc == PRESETS["phi-4"]
    assert PRESETS["phi3-medium-4k"].head_dim == 128 and PRESETS["phi3-medium-4k"].n_q_heads // 10 == 4


@pytest.mark.parametrize("over,reason", [
    (dict(partial_rotary_factor=0.75), "partial_rotary_factor"),
    (dict(rope_scaling={"type": "longrope", "long_factor": LONG, "short_factor": SHORT, "short_mscale": 1.1}),
     "short_mscale"),
    (dict(rope_scaling={"type": "longrope", "long_factor": LONG, "short_factor": SHORT, "long_mscale": 1.2}),
     "long_mscale"),
    (dict(rope_scaling={"type": "longrope", "long_factor": LONG, "short_factor": SHORT, "attention_factor": 1.2}),
     "attention_factor"),
    (dict(layer_types=["full_attention", "sliding_attention"]), "layer_types"),
    (dict(hidden_size=2560), "head_dim 80"),
    (dict(rope_scaling={"type": "dynamic", "factor": 2.0}), "'dynamic'"),
])
def test_loader_refuses_phi3_variants_it_would_serve_wrongly(tmp_path, over, reason):
    with pytest.raises(ValueError, match=reason):
        _read(tmp_path, _phi3_json(**over))


def test_loader_refuses_phi3_under_tensor_parallelism():
    from vllm_tgis_adapter_b200.engine.loader import build_engine

    args = argparse.Namespace(model="phi3-mini-4k", synthetic_weights=True, max_model_len=None, tensor_parallel_size=2)
    with pytest.raises(ValueError, match="single GPU only"):
        build_engine(args)


@pytest.mark.parametrize("model_type,arch", [("phi3small", "Phi3SmallForCausalLM"), ("phimoe", "PhiMoEForCausalLM"),
                                             ("phi3_v", "Phi3VForCausalLM")])
def test_other_phi_families_stay_unrecognised(tmp_path, model_type, arch):
    with pytest.raises(ValueError, match="unsupported model architecture"):
        _read(tmp_path, _phi3_json(model_type=model_type, architectures=[arch]))


def test_llama_loader_still_refuses_96_dim_heads_and_longrope(tmp_path):
    cfg = _phi3_json(model_type="llama", architectures=["LlamaForCausalLM"], rope_scaling=None)
    with pytest.raises(ValueError, match="head_dim 96"):
        _read(tmp_path, cfg)


# ------------------------------------------------------------------------------------------------ fused tensors
def test_fused_tensors_split_into_the_separate_projections():
    from vllm_tgis_adapter_b200.engine.core import PRESETS
    from vllm_tgis_adapter_b200.engine.loader import split_fused

    mc = PRESETS["phi3-tiny"]
    cfg = Phi3Config(n_layers=1, hidden=mc.hidden, n_q_heads=4, n_kv_heads=2, ffn=mc.ffn, vocab=mc.vocab, head_dim=96)
    w = synthetic_weights(cfg, seed=3)
    fused = fuse(w)
    assert "model.layers.0.self_attn.qkv_proj.weight" in fused and "model.layers.0.mlp.up_proj.weight" not in fused
    mc2 = dataclasses.replace(mc, n_kv_heads=2)
    back = {}
    for name, t in fused.items():
        for n, part in split_fused(name, t, mc2):
            back[n] = part
    assert back.keys() == w.keys() and all(torch.equal(back[k], w[k]) for k in w)
    with pytest.raises(ValueError, match="rows"):
        split_fused("model.layers.0.mlp.gate_up_proj.weight", torch.zeros(3, 4), mc2)


# ------------------------------------------------------------------------------------------------ LongRoPE table
def _mc(max_model_len, **over):
    from vllm_tgis_adapter_b200.engine.core import ModelConfig

    d = dict(n_layers=1, hidden=384, n_q_heads=4, n_kv_heads=4, ffn=512, vocab=1021, head_dim=96, rope_theta=10000.0,
             max_model_len=max_model_len, rope_long_factor=tuple(LONG), rope_short_factor=tuple(SHORT),
             rope_original_max_pos=64, rope_max_position_embeddings=512)
    d.update(over)
    return ModelConfig(**d)


def test_longrope_factor_choice_is_made_by_max_model_len():
    from vllm_tgis_adapter_b200.engine.rope import longrope_factors

    assert longrope_factors(_mc(64)) == ("short", tuple(SHORT))
    assert longrope_factors(_mc(65)) == ("long", tuple(LONG))


def test_longrope_mscale_and_table_match_the_oracle_restatement():
    from vllm_tgis_adapter_b200.engine.rope import longrope_mscale, rope_cos_sin

    assert longrope_mscale(_mc(64)) == pytest.approx(math.sqrt(1 + math.log(8) / math.log(64)))
    assert longrope_mscale(_mc(64, rope_max_position_embeddings=64)) == 1.0
    for n, regime in ((64, "short"), (65, "long")):
        cfg = Phi3Config(n_layers=1, hidden=384, n_q_heads=4, n_kv_heads=4, ffn=512, vocab=1021, head_dim=96,
                         max_model_len=n, rope_theta=10000.0, long_factor=tuple(LONG), short_factor=tuple(SHORT),
                         original_max_pos=64, max_position_embeddings=512)
        assert torch.equal(rope_cos_sin(_mc(n)), longrope_table(cfg, regime))
    # the two regimes differ, and the mscale is in the table (cos at position 0 is mscale, rounded)
    assert not torch.equal(rope_cos_sin(_mc(65))[:64], rope_cos_sin(_mc(64)))
    assert float(rope_cos_sin(_mc(64))[0, 0]) == float(torch.tensor(longrope_mscale(_mc(64))).bfloat16())


def test_presets_without_longrope_keep_their_tables():
    from vllm_tgis_adapter_b200.engine.core import PRESETS

    for name, mc in PRESETS.items():
        if not name.startswith("phi"):
            assert not mc.rope_longrope and mc.rope_long_factor == () and mc.rope_short_factor == ()


# ------------------------------------------------------------------------------------------------ oracle vs HF
def _fixture(name):
    fx = json.loads((GOLD / name).read_text())
    return fx, Phi3Config(**fx["config"])


def _run(ora, run):
    s = ora.new_seq()
    logits = ora.step([(s, run["prompt"])], want_all_logits=True).float()
    steps = [ora.step([(s, [t])])[0].float() for t in run.get("decode_tokens", [])]
    return logits, steps


@pytest.mark.parametrize("regime", ["short", "long"])
def test_phi3_oracle_matches_hf_fixture_fp32(regime):
    fx, cfg = _fixture("phi3_hf_fp32.json")
    assert cfg.head_dim == 96 and cfg.n_q_heads // cfg.n_kv_heads == 2 and cfg.vocab % 2 == 1
    w = synthetic_weights(cfg, seed=fx["weights_seed"], dtype=torch.float32)
    run = fx[regime]
    assert (len(run["prompt"]) <= cfg.original_max_pos) == (regime == "short")
    logits, steps = _run(Phi3Oracle(cfg, w, regime=regime, dtype=torch.float32), run)
    assert logits.argmax(-1).tolist() == run["argmax_per_pos"]
    np.testing.assert_allclose(torch.logsumexp(logits, -1).numpy(), np.array(run["logsumexp_per_pos"]), atol=2e-4)
    np.testing.assert_allclose(logits[-1].numpy(), np.array(run["last_logits"]), atol=2e-4)
    for got, want in zip(steps, run.get("decode_logits", [])):
        np.testing.assert_allclose(got.numpy(), np.array(want), atol=2e-4)
    # the other regime's factors, or no window, visibly miss it
    other = "long" if regime == "short" else "short"
    lo, _ = _run(Phi3Oracle(cfg, w, regime=other, dtype=torch.float32), run)
    assert float((lo[-1] - torch.tensor(run["last_logits"])).abs().max()) > 1e-2
    lw, _ = _run(Phi3Oracle(cfg, w, regime=regime, window=None, dtype=torch.float32), run)
    assert float((lw[-1] - torch.tensor(run["last_logits"])).abs().max()) > 1e-2


@pytest.mark.parametrize("regime", ["short", "long"])
def test_phi3_oracle_bf16_rounding_points_match_hf_bf16_fixture(regime):
    """the bars of tests/test_mistral_cpu.py: within 2 bf16 ulps of the row's largest logit"""
    fx, cfg = _fixture("phi3_hf_bf16.json")
    assert cfg.n_q_heads == cfg.n_kv_heads
    run = fx[regime]
    logits, steps = _run(Phi3Oracle(cfg, synthetic_weights(cfg, seed=fx["weights_seed"]), regime=regime), run)
    pairs = [(logits[-1], torch.tensor(run["last_logits"]))]
    pairs += [(s, torch.tensor(w)) for s, w in zip(steps, run.get("decode_logits", []))]
    for got, want in pairs:
        d = (got - want).abs()
        ulp_row = 2.0 ** (torch.floor(torch.log2(want.abs().max())).item() - 7)
        assert float(d.max()) <= 2.0 * ulp_row, (float(d.max()), ulp_row)
        assert float(d.mean()) < 0.5 * ulp_row
    np.testing.assert_allclose(torch.logsumexp(logits, -1).numpy(), np.array(run["logsumexp_per_pos"]), atol=1e-2)
    for pos, (a, b, m) in enumerate(zip(logits.argmax(-1).tolist(), run["argmax_per_pos"], run["top2_margin_per_pos"])):
        if m > 0.04:
            assert a == b, (pos, a, b, m)


# ------------------------------------------------------------------------------------------------ ABI and build
def test_the_abi_is_unchanged():
    from vllm_tgis_adapter_b200.engine import _lib

    lib = _lib.load_library()
    assert _lib.ABI_VERSION == 9 and lib.tgis_abi_version() == 9
    assert C.sizeof(_lib.TgisConfig) == 336 and C.sizeof(_lib.TgisSamplingParams) == 120


def test_the_library_holds_sm_90a_code_with_96_dim_kernels():
    from vllm_tgis_adapter_b200.engine import _lib

    _lib.load_library()
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(tool).exists():
        pytest.skip("cuobjdump is not installed")
    out = subprocess.run([tool, "--list-elf", str(_lib.library_path())], capture_output=True, text=True).stdout
    assert "sm_90a" in out
    syms = subprocess.run([tool, "-symbols", str(_lib.library_path())], capture_output=True, text=True).stdout
    for k in ("attn_decode_kernelILi96ELi1E", "attn_decode_kernelILi96ELi8E", "attn_prefill_kernelILi96ELb1E",
              "rope_kvwrite_kernelILi96E"):
        assert k in syms, k
