"""Qwen3 on the host side: config.json mapping (the tiny, 0.6B and 8B shapes, both rope spellings), the refusals, the test
oracle against transformers' Qwen3ForCausalLM (tests/golden/qwen3_hf_*.json, scripts/gen_qwen3_golden.py: teacher-forced
logits and a KV-cache decode step), and the new C-ABI symbols.  No GPU."""
import argparse
import ctypes as C
import json
import re
from pathlib import Path

import numpy as np
import pytest
import torch

from qwen3_oracle import CONFIGS, Qwen3Config, Qwen3Oracle, synthetic_weights

ROOT = Path(__file__).resolve().parent.parent
GOLD = ROOT / "tests" / "golden"


def _qwen3_json(**over) -> dict:
    """Qwen/Qwen3-8B's config.json (transformers 4 spelling), as recalled"""
    cfg = {"architectures": ["Qwen3ForCausalLM"], "model_type": "qwen3", "hidden_size": 4096, "num_attention_heads": 32,
           "num_key_value_heads": 8, "num_hidden_layers": 36, "intermediate_size": 12288, "vocab_size": 151936,
           "head_dim": 128, "max_position_embeddings": 40960, "rms_norm_eps": 1e-6, "rope_theta": 1000000.0,
           "rope_scaling": None, "attention_bias": False, "use_sliding_window": False, "sliding_window": None,
           "max_window_layers": 36, "tie_word_embeddings": False}
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
    "qwen3-8b": {},
    "qwen3-0.6b": dict(hidden_size=1024, num_attention_heads=16, num_hidden_layers=28, intermediate_size=3072,
                       max_window_layers=28, tie_word_embeddings=True),
    "qwen3-tiny": dict(hidden_size=256, num_attention_heads=4, num_key_value_heads=2, num_hidden_layers=2,
                       intermediate_size=512, vocab_size=1021, max_position_embeddings=2048, tie_word_embeddings=True),
}


# ------------------------------------------------------------------------------------------------ config.json mapping
@pytest.mark.parametrize("preset", sorted(SHAPES))
@pytest.mark.parametrize("spelling", ["rope_theta", "rope_parameters"])
def test_loader_maps_qwen3_configs_onto_the_presets(tmp_path, preset, spelling):
    from vllm_tgis_adapter_b200.engine.core import PRESETS

    cfg = _qwen3_json(**SHAPES[preset])
    mc = _read(tmp_path, cfg if spelling == "rope_theta" else _v5(cfg))
    assert mc == PRESETS[preset]
    assert mc.qk_norm and mc.arch == "llama" and mc.head_dim == 128 and not mc.rope_scaled and not mc.is_granite
    assert mc.n_q_heads * mc.head_dim != mc.hidden or preset == "qwen3-8b"
    # max_model_len policy: min(max_position_embeddings, 8192) unless asked for
    if preset == "qwen3-tiny":
        with pytest.raises(ValueError, match="exceeds the model's max_position_embeddings 2048"):
            _read(tmp_path, cfg, 4096)
    else:
        assert _read(tmp_path, cfg, 16384).max_model_len == 16384
    # the default epsilon of Qwen3 is 1e-6 (Llama's is 1e-5)
    del cfg["rms_norm_eps"]
    assert _read(tmp_path, cfg).rms_eps == 1e-6


def test_qwen3_is_recognised_by_architecture_name_alone(tmp_path):
    from vllm_tgis_adapter_b200.engine.core import PRESETS

    cfg = _qwen3_json()
    del cfg["model_type"]
    assert _read(tmp_path, cfg) == PRESETS["qwen3-8b"]


def test_presets_agree_with_the_oracle_config():
    from vllm_tgis_adapter_b200.engine.core import PRESETS

    mc, oc = PRESETS["qwen3-tiny"], CONFIGS["qwen3-tiny"]
    for f in ("n_layers", "hidden", "n_q_heads", "n_kv_heads", "ffn", "vocab", "head_dim", "rope_theta", "rms_eps",
              "max_model_len", "tie_word_embeddings"):
        assert getattr(mc, f) == getattr(oc, f), f
    assert mc.qk_norm and mc.vocab % 2 == 1 and oc.q_dim != oc.hidden
    assert not PRESETS["qwen3-8b"].tie_word_embeddings and PRESETS["qwen3-0.6b"].tie_word_embeddings
    assert not any(p.qk_norm for name, p in PRESETS.items() if not name.startswith("qwen3"))


# ------------------------------------------------------------------------------------------------ refusals
@pytest.mark.parametrize("over,reason", [
    (dict(attention_bias=True), "attention_bias"),
    (dict(use_sliding_window=True, sliding_window=4096), "use_sliding_window"),
    (dict(layer_types=["full_attention"] * 35 + ["sliding_attention"]), r"layer_types \['sliding_attention'\]"),
    (dict(head_dim=64), "head_dim 64"),
    (dict(head_dim=None, hidden_size=2560, num_attention_heads=32), "head_dim 80"),
    (dict(rope_scaling={"rope_type": "yarn", "factor": 4.0, "original_max_position_embeddings": 32768}),
     "'yarn' is not supported"),
])
def test_loader_refuses_qwen3_variants_it_would_serve_wrongly(tmp_path, over, reason):
    with pytest.raises(ValueError, match=reason):
        _read(tmp_path, _qwen3_json(**over))


def test_loader_refuses_qwen3_under_tensor_parallelism():
    from vllm_tgis_adapter_b200.engine.loader import build_engine

    args = argparse.Namespace(model="qwen3-0.6b", synthetic_weights=True, max_model_len=None, tensor_parallel_size=2)
    with pytest.raises(ValueError, match="single GPU only: tensor_parallel_size 2"):
        build_engine(args)


@pytest.mark.parametrize("model_type,arch", [("qwen3_moe", "Qwen3MoeForCausalLM"), ("qwen3_next", "Qwen3NextForCausalLM"),
                                             ("qwen2", "Qwen2ForCausalLM")])
def test_other_qwen_families_stay_unrecognised(tmp_path, model_type, arch):
    with pytest.raises(ValueError, match="unsupported model architecture"):
        _read(tmp_path, _qwen3_json(model_type=model_type, architectures=[arch]))


# ------------------------------------------------------------------------------------------------ oracle vs transformers
def _fixture(name):
    fx = json.loads((GOLD / name).read_text())
    return fx, Qwen3Config(**fx["config"])


def _run(ora, fx):
    s = ora.new_seq()
    logits = ora.step([(s, fx["prompt"])], want_all_logits=True)
    step = ora.step([(s, [fx["decode_token"]])])[0]
    return logits, step


def test_qwen3_oracle_matches_hf_fixture_fp32():
    fx, cfg = _fixture("qwen3_hf_fp32.json")
    assert cfg.q_dim != cfg.hidden and cfg.tie_word_embeddings and cfg.vocab % 2 == 1
    w = synthetic_weights(cfg, seed=fx["weights_seed"], dtype=torch.float32)
    logits, step = _run(Qwen3Oracle(cfg, w, dtype=torch.float32), fx)
    assert logits.argmax(-1).tolist() == fx["argmax_per_pos"]
    np.testing.assert_allclose(torch.logsumexp(logits, -1).numpy(), np.array(fx["logsumexp_per_pos"]), atol=2e-4)
    np.testing.assert_allclose(logits[-1].numpy(), np.array(fx["last_logits"]), atol=2e-4)
    np.testing.assert_allclose(step.numpy(), np.array(fx["decode_logits"]), atol=2e-4)
    # without the per-head norm (the plain Llama stack on the same weights) the logits are visibly different: the fixture
    # does pin the norm and its weights
    from oracle.llama_oracle import LlamaOracle

    plain = LlamaOracle(cfg, w, dtype=torch.float32)
    lp = plain.step([(plain.new_seq(), fx["prompt"])], want_all_logits=True)
    assert float((lp[-1] - torch.tensor(fx["last_logits"])).abs().max()) > 1e-2
    ones = dict(w)
    for k in ones:
        if k.endswith("_norm.weight") and "self_attn" in k:
            ones[k] = torch.ones_like(ones[k])
    lo, _ = _run(Qwen3Oracle(cfg, ones, dtype=torch.float32), fx)
    assert float((lo[-1] - torch.tensor(fx["last_logits"])).abs().max()) > 1e-2


def test_qwen3_oracle_bf16_rounding_points_match_hf_bf16_fixture():
    """the bars of tests/test_oracle_cpu.py for llama_hf_bf16.json: within 2 bf16 ulps of the row's largest logit"""
    fx, cfg = _fixture("qwen3_hf_bf16.json")
    logits, step = _run(Qwen3Oracle(cfg, synthetic_weights(cfg, seed=fx["weights_seed"])), fx)
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


# ------------------------------------------------------------------------------------------------ ABI
def test_new_symbols_are_declared_and_exported_and_the_abi_is_unchanged():
    from vllm_tgis_adapter_b200.engine import _lib

    lib = _lib.load_library()
    new = {"tgis_engine.h": ["tgis_engine_set_qk_norm"], "tgis_kernels.h": ["tgis_k_rope_kv_qknorm"]}
    for header, syms in new.items():
        text = re.sub(r"/\*.*?\*/", "", (ROOT / "include" / header).read_text(), flags=re.S)
        for sym in syms:
            assert re.search(rf"\b{sym}\s*\(", text), (header, sym)
            assert hasattr(lib, sym), sym
            assert sym in _lib.ENGINE_SYMBOLS + _lib.KERNEL_SYMBOLS
    # the config struct did not grow and the version did not move: the q/k norm is a call of its own
    assert _lib.ABI_VERSION == 8 and lib.tgis_abi_version() == 8
    assert C.sizeof(_lib.TgisConfig) == 304 and C.sizeof(_lib.TgisSamplingParams) == 120
    assert re.search(r"#define TGIS_ABI_VERSION 8\b", (ROOT / "include" / "tgis_engine.h").read_text())
