"""Qwen2 / Qwen2.5 on the host side: config.json mapping (the 0.5B, 1.5B, 7B and 14B shapes, both rope spellings), vLLM's
defaults where they differ from transformers', the refusals, the test oracle against transformers' Qwen2ForCausalLM
(tests/golden/qwen2_hf_*.json, scripts/gen_qwen2_golden.py: teacher-forced logits and a KV-cache decode step), and the
new C-ABI symbols.  No GPU."""
import ctypes as C
import json
import re
from pathlib import Path

import numpy as np
import pytest
import torch

from qwen2_oracle import CONFIGS, Qwen2Config, Qwen2Oracle, synthetic_weights

ROOT = Path(__file__).resolve().parent.parent
GOLD = ROOT / "tests" / "golden"


def _qwen2_json(**over) -> dict:
    """Qwen/Qwen2.5-7B-Instruct's config.json (transformers 4 spelling), as recalled"""
    cfg = {"architectures": ["Qwen2ForCausalLM"], "model_type": "qwen2", "hidden_size": 3584,
           "num_attention_heads": 28, "num_key_value_heads": 4, "num_hidden_layers": 28, "intermediate_size": 18944,
           "vocab_size": 152064, "max_position_embeddings": 32768, "rms_norm_eps": 1e-6, "rope_theta": 1000000.0,
           "rope_scaling": None, "use_sliding_window": False, "sliding_window": 131072, "max_window_layers": 28,
           "tie_word_embeddings": False, "hidden_act": "silu", "attention_dropout": 0.0, "torch_dtype": "bfloat16"}
    cfg.update(over)
    return cfg


def _v5(cfg: dict) -> dict:
    """the transformers 5 spelling of the same config: rope_parameters holds rope_theta, layer_types is written out"""
    cfg = dict(cfg)
    theta = cfg.pop("rope_theta")
    cfg.pop("rope_scaling", None)
    cfg["rope_parameters"] = {"rope_type": "default", "rope_theta": theta}
    cfg["layer_types"] = ["full_attention"] * cfg["num_hidden_layers"]
    return cfg


def _read(tmp_path, cfg, max_model_len=None):
    from vllm_tgis_adapter_b200.engine.loader import model_config_from_hf

    (tmp_path / "config.json").write_text(json.dumps(cfg))
    return model_config_from_hf(tmp_path, max_model_len)


SHAPES = {
    "qwen2.5-7b": ({}, 7),
    "qwen2.5-0.5b": (dict(hidden_size=896, num_attention_heads=14, num_key_value_heads=2, num_hidden_layers=24,
                          intermediate_size=4864, vocab_size=151936, max_window_layers=21, tie_word_embeddings=True), 7),
    "qwen2.5-1.5b": (dict(hidden_size=1536, num_attention_heads=12, num_key_value_heads=2, num_hidden_layers=28,
                          intermediate_size=8960, vocab_size=151936, max_window_layers=21, tie_word_embeddings=True), 6),
    "qwen2.5-14b": (dict(hidden_size=5120, num_attention_heads=40, num_key_value_heads=8, num_hidden_layers=48,
                         intermediate_size=13824, rms_norm_eps=1e-5, max_window_layers=70, max_position_embeddings=131072),
                    5),
}


# ------------------------------------------------------------------------------------------------ config.json mapping
@pytest.mark.parametrize("preset", sorted(SHAPES))
@pytest.mark.parametrize("spelling", ["rope_theta", "rope_parameters"])
def test_loader_maps_qwen2_configs_onto_the_presets(tmp_path, preset, spelling):
    from vllm_tgis_adapter_b200.engine.core import PRESETS

    over, group = SHAPES[preset]
    cfg = _qwen2_json(**over)
    mc = _read(tmp_path, cfg if spelling == "rope_theta" else _v5(cfg))
    assert mc == PRESETS[preset]
    assert mc.qkv_bias and not mc.qk_norm and mc.arch == "llama" and not mc.rope_scaled and not mc.is_granite
    assert mc.sliding_window is None and mc.n_q_heads // mc.n_kv_heads == group
    assert mc.head_dim == (64 if preset == "qwen2.5-0.5b" else 128)
    # max_model_len policy: min(max_position_embeddings, 8192) unless asked for
    assert mc.max_model_len == 8192 and _read(tmp_path, cfg, 16384).max_model_len == 16384
    with pytest.raises(ValueError, match="exceeds the model's max_position_embeddings"):
        _read(tmp_path, cfg, cfg["max_position_embeddings"] + 1)
    # the default epsilon of Qwen2 is 1e-6 (Llama's is 1e-5)
    del cfg["rms_norm_eps"]
    assert _read(tmp_path, cfg).rms_eps == 1e-6


def test_vllm_defaults_where_they_differ_from_transformers(tmp_path):
    # no rotary theta at all: vLLM's qwen2.py sets 1e6 (transformers' Llama-style default would be 1e4)
    cfg = _qwen2_json()
    del cfg["rope_theta"]
    assert _read(tmp_path, cfg).rope_theta == 1000000.0
    v5 = _v5(_qwen2_json())
    v5["rope_parameters"] = {"rope_type": "default"}
    assert _read(tmp_path, v5).rope_theta == 1000000.0
    assert _read(tmp_path, _qwen2_json(rope_theta=10000.0)).rope_theta == 10000.0
    # head_dim is hidden_size // num_attention_heads; a head_dim key that agrees is fine
    assert _read(tmp_path, _qwen2_json(head_dim=128)).head_dim == 128
    # tie_word_embeddings is honoured both ways
    assert _read(tmp_path, _qwen2_json(tie_word_embeddings=True)).tie_word_embeddings


def test_qwen2_is_recognised_by_architecture_name_alone(tmp_path):
    from vllm_tgis_adapter_b200.engine.core import PRESETS

    cfg = _qwen2_json()
    del cfg["model_type"]
    assert _read(tmp_path, cfg) == PRESETS["qwen2.5-7b"]


def test_presets_agree_with_the_oracle_configs():
    from vllm_tgis_adapter_b200.engine.core import PRESETS

    for name in ("qwen2-tiny", "qwen2-tiny-hd64"):
        mc, oc = PRESETS[name], CONFIGS[name]
        for f in ("n_layers", "hidden", "n_q_heads", "n_kv_heads", "ffn", "vocab", "head_dim", "rope_theta", "rms_eps",
                  "max_model_len", "tie_word_embeddings"):
            assert getattr(mc, f) == getattr(oc, f), (name, f)
        assert mc.qkv_bias and mc.vocab % 2 == 1 and mc.hidden // mc.n_q_heads == mc.head_dim
    assert PRESETS["qwen2-tiny"].n_q_heads // PRESETS["qwen2-tiny"].n_kv_heads == 6
    assert PRESETS["qwen2-tiny-hd64"].n_q_heads // PRESETS["qwen2-tiny-hd64"].n_kv_heads == 7
    assert not PRESETS["qwen2.5-7b"].tie_word_embeddings and PRESETS["qwen2.5-0.5b"].tie_word_embeddings
    assert not any(p.qkv_bias for name, p in PRESETS.items() if not name.startswith("qwen2"))


# ------------------------------------------------------------------------------------------------ refusals
@pytest.mark.parametrize("over,reason", [
    (dict(use_sliding_window=True), "use_sliding_window"),
    (dict(layer_types=["full_attention"] * 27 + ["sliding_attention"]), r"layer_types \['sliding_attention'\]"),
    (dict(qk_norm=True), "qk_norm"),
    (dict(is_causal=False), "is_causal"),
    (dict(dual_chunk_attention_config={"chunk_size": 262144, "local_size": 8192}), "dual_chunk_attention_config"),
    (dict(head_dim=64), r"head_dim 64 != hidden_size // num_attention_heads = 128"),
    (dict(hidden_size=2560, num_attention_heads=32), "head_dim 80"),
    (dict(rope_scaling={"rope_type": "yarn", "factor": 4.0, "original_max_position_embeddings": 32768}),
     "'yarn' is not supported"),
])
def test_loader_refuses_qwen2_variants_it_would_serve_wrongly(tmp_path, over, reason):
    with pytest.raises(ValueError, match=reason):
        _read(tmp_path, _qwen2_json(**over))


def test_loader_refuses_qwen2_under_tensor_parallelism():
    from vllm_tgis_adapter_b200.engine.loader import build_engine
    from vllm_tgis_adapter_b200.tgis_utils.args import parse_args

    args = parse_args(["--model", "qwen2.5-7b", "--synthetic-weights", "--tensor-parallel-size", "2"])
    with pytest.raises(ValueError, match=r"Qwen2\) is supported on a single GPU only \(tp_size must be 1\)"):
        build_engine(args)


@pytest.mark.parametrize("by", ["model_type", "architectures"])
def test_a_config_declaring_bias_free_projections_is_not_qwen2(tmp_path, by):
    """Qwen2ForCausalLM hard-codes bias=True on q / k / v (transformers and vLLM) and Qwen2Config has no attention_bias
    key: a config with attention_bias false was written for another architecture and has no bias tensors to load"""
    cfg = _qwen2_json(attention_bias=False, head_dim=128)
    if by == "model_type":
        del cfg["architectures"]
    else:
        del cfg["model_type"]
    with pytest.raises(ValueError, match="unsupported model architecture.*attention_bias false"):
        _read(tmp_path, cfg)
    # transformers' own Qwen2Config writes no attention_bias key, and such a config maps
    from transformers import Qwen2Config as HFQwen2Config

    assert "attention_bias" not in HFQwen2Config().to_dict()
    cfg.pop("attention_bias")
    assert _read(tmp_path, cfg).qkv_bias


@pytest.mark.parametrize("model_type,arch", [("qwen2_moe", "Qwen2MoeForCausalLM"),
                                             ("qwen2_vl", "Qwen2VLForConditionalGeneration"),
                                             ("qwen2_5_vl", "Qwen2_5_VLForConditionalGeneration"),
                                             ("qwen2_audio", "Qwen2AudioForConditionalGeneration")])
def test_other_qwen2_families_stay_unrecognised(tmp_path, model_type, arch):
    with pytest.raises(ValueError, match="unsupported model architecture"):
        _read(tmp_path, _qwen2_json(model_type=model_type, architectures=[arch]))


# ------------------------------------------------------------------------------------------------ oracle vs transformers
def _fixture(name):
    fx = json.loads((GOLD / name).read_text())
    return fx, Qwen2Config(**fx["config"])


def _run(ora, fx):
    s = ora.new_seq()
    logits = ora.step([(s, fx["prompt"])], want_all_logits=True)
    step = ora.step([(s, [fx["decode_token"]])])[0]
    return logits, step


def _no_bias(w):
    return {k: (torch.zeros_like(v) if k.endswith("_proj.bias") else v) for k, v in w.items()}


def test_qwen2_oracle_matches_hf_fixture_fp32():
    fx, cfg = _fixture("qwen2_hf_fp32.json")
    assert fx["preset"] == "qwen2-tiny" and cfg.n_q_heads // cfg.n_kv_heads == 6 and cfg.head_dim == 128
    assert cfg.tie_word_embeddings and cfg.vocab % 2 == 1
    w = synthetic_weights(cfg, seed=fx["weights_seed"], dtype=torch.float32)
    logits, step = _run(Qwen2Oracle(cfg, w, dtype=torch.float32), fx)
    assert logits.argmax(-1).tolist() == fx["argmax_per_pos"]
    np.testing.assert_allclose(torch.logsumexp(logits, -1).numpy(), np.array(fx["logsumexp_per_pos"]), atol=2e-4)
    np.testing.assert_allclose(logits[-1].numpy(), np.array(fx["last_logits"]), atol=2e-4)
    np.testing.assert_allclose(step.numpy(), np.array(fx["decode_logits"]), atol=2e-4)
    # without the biases the logits are visibly different: the fixture does pin them
    lo, _ = _run(Qwen2Oracle(cfg, _no_bias(w), dtype=torch.float32), fx)
    assert float((lo[-1] - torch.tensor(fx["last_logits"])).abs().max()) > 1e-2


def test_qwen2_oracle_bf16_rounding_points_match_hf_bf16_fixture():
    """64-dim heads, GQA group 7; the bars of tests/test_oracle_cpu.py for llama_hf_bf16.json: within 2 bf16 ulps of the
    row's largest logit"""
    fx, cfg = _fixture("qwen2_hf_bf16.json")
    assert fx["preset"] == "qwen2-tiny-hd64" and cfg.n_q_heads // cfg.n_kv_heads == 7 and cfg.head_dim == 64
    w = synthetic_weights(cfg, seed=fx["weights_seed"])
    logits, step = _run(Qwen2Oracle(cfg, w), fx)
    assert torch.equal(logits, logits.to(torch.bfloat16).float())
    for got, want in ((logits[-1], torch.tensor(fx["last_logits"])), (step, torch.tensor(fx["decode_logits"]))):
        d = (got - want).abs()
        ulp_row = 2.0 ** (torch.floor(torch.log2(want.abs().max())).item() - 7)
        assert float(d.max()) <= 2.0 * ulp_row, (float(d.max()), ulp_row)
        assert float(d.mean()) < 0.5 * ulp_row
        assert float((d == 0).float().mean()) > 0.15
    np.testing.assert_allclose(torch.logsumexp(logits, -1).numpy(), np.array(fx["logsumexp_per_pos"]), atol=1e-2)
    for pos, (a, b, m) in enumerate(zip(logits.argmax(-1).tolist(), fx["argmax_per_pos"], fx["top2_margin_per_pos"])):
        if m > 0.04:
            assert a == b, (pos, a, b, m)
    # the biases dropped: visibly off the fixture
    lo, _ = _run(Qwen2Oracle(cfg, _no_bias(w)), fx)
    want = torch.tensor(fx["last_logits"])
    ulp_row = 2.0 ** (torch.floor(torch.log2(want.abs().max())).item() - 7)
    assert float((lo[-1] - want).abs().max()) > 8 * ulp_row


# ------------------------------------------------------------------------------------------------ ABI
def test_new_symbols_are_declared_and_exported_and_the_abi_is_unchanged():
    from vllm_tgis_adapter_b200.engine import _lib

    lib = _lib.load_library()
    new = {"tgis_kernels.h": ["tgis_k_rope_kv_bias"]}
    for header, syms in new.items():
        text = re.sub(r"/\*.*?\*/", "", (ROOT / "include" / header).read_text(), flags=re.S)
        for sym in syms:
            assert re.search(rf"\b{sym}\s*\(", text), (header, sym)
            assert hasattr(lib, sym), sym
            assert sym in _lib.ENGINE_SYMBOLS + _lib.KERNEL_SYMBOLS
    # the qkv bias is a tgis_config field (ABI v9), not a call of its own
    header = (ROOT / "include" / "tgis_engine.h").read_text()
    assert "qkv_bias" in [f for f, _ in _lib.TgisConfig._fields_] and "int32_t qkv_bias;" in header
    assert _lib.ABI_VERSION == 9 and lib.tgis_abi_version() == 9
    assert C.sizeof(_lib.TgisConfig) == 336 and C.sizeof(_lib.TgisSamplingParams) == 120
    assert re.search(r"#define TGIS_ABI_VERSION 9\b", header)
