"""Granite (GraniteForCausalLM) without a GPU: the oracle against transformers' fixtures, the config.json mapping and
its refusals, and the C ABI additions."""
import ctypes as C
import json
from pathlib import Path

import numpy as np
import pytest
import torch

from granite_oracle import CONFIGS, GraniteConfig, GraniteOracle, synthetic_weights
from oracle.llama_oracle import CONFIGS as LLAMA_CONFIGS
from oracle.llama_oracle import LlamaOracle
from oracle.llama_oracle import synthetic_weights as llama_synthetic_weights

GOLD = Path(__file__).parent / "golden"


def _oracle_logits(g: dict, dtype: torch.dtype) -> torch.Tensor:
    cfg = GraniteConfig(**g["config"])
    w = synthetic_weights(cfg, seed=g["weights_seed"], dtype=dtype)
    assert "lm_head.weight" not in w   # tied
    ora = GraniteOracle(cfg, w, dtype=dtype)
    return ora.step([(ora.new_seq(), g["prompt"])], want_all_logits=True)


def test_granite_oracle_matches_hf_fp32():
    g = json.loads((GOLD / "granite_hf_fp32.json").read_text())
    assert g["config"]["vocab"] % 8 != 0 and g["config"]["tie_word_embeddings"]
    logits = _oracle_logits(g, torch.float32)
    assert logits.shape[-1] == g["config"]["vocab"]
    assert logits.argmax(-1).tolist() == g["argmax_per_pos"]
    np.testing.assert_allclose(torch.logsumexp(logits, -1).numpy(), np.array(g["logsumexp_per_pos"]), atol=2e-4)
    np.testing.assert_allclose(logits[-1].numpy(), np.array(g["last_logits"]), atol=2e-4)


def test_granite_oracle_bf16_rounding_points_match_hf_bf16():
    """bf16: the multipliers' rounding points (bf16(e*m), bf16(r + bf16(x*m)), the scaled bf16 logits) are HF's: the last
    row's logits agree within 2 bf16 ulps of the row's magnitude."""
    g = json.loads((GOLD / "granite_hf_bf16.json").read_text())
    logits = _oracle_logits(g, torch.bfloat16)
    assert torch.equal(logits, logits.to(torch.bfloat16).float())
    last = torch.tensor(g["last_logits"])
    ulp_row = 2.0 ** (torch.floor(torch.log2(last.abs().max())).item() - 7)
    d = (logits[-1] - last).abs()
    assert float(d.max()) <= 2.0 * ulp_row, (float(d.max()), ulp_row)
    assert float(d.mean()) < 0.5 * ulp_row
    for pos, (a, b, m) in enumerate(zip(logits.argmax(-1).tolist(), g["argmax_per_pos"], g["top2_margin_per_pos"])):
        if m > 4 * ulp_row:
            assert a == b, (pos, a, b, m)


def test_granite_scalars_at_defaults_are_the_llama_oracle():
    """bf16(x * 1) = x: the Granite oracle with every scalar at its default computes the Llama logits bit for bit."""
    import dataclasses

    base = LLAMA_CONFIGS["tiny"]
    cfg = GraniteConfig(**dataclasses.asdict(base), tie_word_embeddings=False)
    w = llama_synthetic_weights(base, seed=5)
    prompt = [5, 9, 300, 44, 17, 1000, 3]
    ora0 = LlamaOracle(base, w)
    a = ora0.step([(ora0.new_seq(), prompt)], want_all_logits=True)
    ora = GraniteOracle(cfg, w)
    b = ora.step([(ora.new_seq(), prompt)], want_all_logits=True)
    assert torch.equal(a, b)


def test_granite_logit_scale_is_one_bf16_rounding_of_the_bf16_logits():
    cfg = CONFIGS["granite-tiny"]
    w = synthetic_weights(cfg, seed=3)
    ora = GraniteOracle(cfg, w)
    x = torch.randn(3, cfg.hidden).to(torch.bfloat16)
    got = ora.head(x)
    acc = (ora._rms(x, ora.norm).float() @ ora.lm_head.float().t()).to(torch.bfloat16)
    want = (acc.float() * torch.tensor(1.0 / 3.0, dtype=torch.float32)).to(torch.bfloat16).float()
    assert torch.equal(got, want)


# ------------------------------------------------------------------------------------------------ config.json mapping
def _granite_json(**over) -> dict:
    cfg = {"architectures": ["GraniteForCausalLM"], "model_type": "granite", "hidden_size": 4096,
           "num_attention_heads": 32, "num_key_value_heads": 8, "num_hidden_layers": 40, "intermediate_size": 12800,
           "vocab_size": 49155, "max_position_embeddings": 131072, "rms_norm_eps": 1e-5, "rope_theta": 10000000.0,
           "tie_word_embeddings": True, "embedding_multiplier": 12.0, "residual_multiplier": 0.22,
           "attention_multiplier": 0.0078125, "logits_scaling": 16.0, "attention_bias": False, "mlp_bias": False}
    cfg.update(over)
    return cfg


def _read(tmp_path, cfg, max_model_len=None):
    from vllm_tgis_adapter_b200.engine.loader import model_config_from_hf

    (tmp_path / "config.json").write_text(json.dumps(cfg))
    return model_config_from_hf(tmp_path, max_model_len)


def test_model_config_from_hf_reads_granite(tmp_path):
    mc = _read(tmp_path, _granite_json())
    assert (mc.n_layers, mc.hidden, mc.n_q_heads, mc.n_kv_heads, mc.ffn, mc.vocab) == (40, 4096, 32, 8, 12800, 49155)
    assert mc.arch == "llama" and mc.head_dim == 128 and mc.rope_theta == 1e7 and mc.max_model_len == 8192
    assert mc.tie_word_embeddings and mc.is_granite
    assert (mc.embedding_multiplier, mc.residual_multiplier, mc.attention_multiplier, mc.logits_scaling) == (
        12.0, 0.22, 0.0078125, 16.0)
    # transformers 5 writes the rotary settings as rope_parameters
    mc = _read(tmp_path, _granite_json(rope_theta=None, rope_parameters={"rope_type": "default", "rope_theta": 5e6}))
    assert mc.rope_theta == 5e6
    # model_type alone is enough
    mc = _read(tmp_path, _granite_json(architectures=None))
    assert mc.is_granite


@pytest.mark.parametrize("over,needle", [
    ({"attention_bias": True}, "attention_bias"),
    ({"mlp_bias": True}, "mlp_bias"),
    ({"rope_scaling": {"type": "linear", "factor": 2.0}}, "rope_scaling"),
    ({"rope_parameters": {"rope_type": "llama3", "rope_theta": 1e7, "factor": 8.0}}, "rope_parameters"),
    ({"hidden_size": 2048, "num_attention_heads": 32}, "head_dim 64"),
])
def test_model_config_from_hf_refuses_unsupported_granite(tmp_path, over, needle):
    with pytest.raises(ValueError, match="unsupported Granite variant") as ei:
        _read(tmp_path, _granite_json(**over))
    assert needle in str(ei.value)


def test_granite_presets_agree_with_the_oracle_configs():
    from vllm_tgis_adapter_b200.engine.core import PRESETS

    for name in ("granite-tiny", "granite-3-8b"):
        mc, oc = PRESETS[name], CONFIGS[name]
        for f in ("n_layers", "hidden", "n_q_heads", "n_kv_heads", "ffn", "vocab", "rope_theta", "embedding_multiplier",
                  "residual_multiplier", "attention_multiplier", "logits_scaling", "tie_word_embeddings"):
            assert getattr(mc, f) == getattr(oc, f), (name, f)
        assert mc.vocab % 8 != 0 and mc.is_granite
    # granite-3-8b's expected weight bytes per decode step (tied lm_head padded to 49 160 rows)
    c = PRESETS["granite-3-8b"]
    per_layer = c.hidden * (c.n_q_heads + 2 * c.n_kv_heads) * 128 + c.hidden * c.n_q_heads * 128 + 3 * c.hidden * c.ffn
    assert per_layer + 2 * c.hidden == 199_237_632
    assert abs(2 * (c.n_layers * (per_layer + 2 * c.hidden) + 49160 * c.hidden) / 1e9 - 16.34) < 0.01


# ------------------------------------------------------------------------------------------------ C ABI
def test_abi_v8_exports_the_model_scalars_call_and_keeps_struct_sizes():
    from vllm_tgis_adapter_b200.engine import _lib

    lib = _lib.load_library()
    assert _lib.ABI_VERSION == 8 == lib.tgis_abi_version()
    for sym in ("tgis_engine_set_model_scalars", "tgis_k_rmsnorm_mult", "tgis_k_embed", "tgis_k_sampler_scaled"):
        assert hasattr(lib, sym), sym
    assert C.sizeof(_lib.TgisConfig) == 304
    assert C.sizeof(_lib.TgisSamplingParams) == 120
    assert lib.tgis_k_sizeof_sample_row() == 64 and lib.tgis_k_sizeof_sample_out() == 112
    # a null engine is an error, not a crash
    assert lib.tgis_engine_set_model_scalars(None, 1.0, 1.0, 0.0, 1.0) != 0


def test_granite_under_tensor_parallelism_is_refused_before_any_rank_starts():
    from vllm_tgis_adapter_b200.engine.core import PRESETS, EngineError, NativeEngine

    with pytest.raises(EngineError, match="Granite.*tensor parallelism"):
        NativeEngine(PRESETS["granite-3-8b"], tp_size=2, tp_rank=0, nccl_id=bytes(128))


def test_granite_hf_checkpoint_config_round_trip(tmp_path):
    """config.json as transformers' save_pretrained writes it for a GraniteForCausalLM."""
    from transformers import GraniteConfig

    GraniteConfig(vocab_size=1021, hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2,
                  num_key_value_heads=1, max_position_embeddings=512, tie_word_embeddings=True, embedding_multiplier=12.0,
                  residual_multiplier=0.22, attention_multiplier=1.0 / 128, logits_scaling=3.0).save_pretrained(tmp_path)
    from vllm_tgis_adapter_b200.engine.loader import model_config_from_hf

    mc = model_config_from_hf(tmp_path, None)
    assert (mc.vocab, mc.head_dim, mc.n_q_heads, mc.n_kv_heads, mc.max_model_len) == (1021, 128, 2, 1, 512)
    assert mc.tie_word_embeddings and mc.logits_scaling == 3.0 and mc.attention_multiplier == 1.0 / 128
