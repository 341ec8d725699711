"""tgis_config_check without a GPU: which model descriptions the engine refuses, with which reason, and that the ones it
serves pass.  tgis_engine_create runs the same check before it looks for a device, and build_engine runs it before it
spawns tensor-parallel ranks, so these refusals are the ones a user sees."""
import ctypes as C
import dataclasses
import math
import re

import pytest

from vllm_tgis_adapter_b200.engine import _lib
from vllm_tgis_adapter_b200.engine.core import PRESETS, config_error, engine_config

GRANITE = dict(embedding_multiplier=12.0, residual_multiplier=0.22, attention_multiplier=1.0 / 128, logits_scaling=3.0)


def _cfg(preset: str, model: dict | None = None, fields: dict | None = None, **options) -> _lib.TgisConfig:
    """preset with ModelConfig overrides, NativeEngine options, and raw tgis_config fields set last"""
    cfg = engine_config(dataclasses.replace(PRESETS[preset], **(model or {})), **options)
    for name, value in (fields or {}).items():
        setattr(cfg, name, value)
    return cfg


REFUSED = [
    # OPT and GPTBigCode take none of the Llama stack's model variants
    *[(arch, model, fields, {}, reason) for arch in ("opt-tiny", "gpt-bigcode-tiny") for model, fields, reason in [
        (GRANITE, None, r"model scalars \(Granite\) apply to the Llama layer stack only, not OPT"),
        (None, dict(rope_table_from_host=1), "OPT has learned positions, no rotary table"),
        (dict(qk_norm=True), None, r"q/k norm \(Qwen3\) applies to the Llama layer stack only, not OPT"),
        (dict(qkv_bias=True), None, r"qkv bias \(Qwen2\) applies to the Llama layer stack only: OPT has its own bias"),
        (dict(sliding_window=40), None, "sliding-window attention applies to the Llama layer stack only, not OPT"),
    ]],
    # head dims
    ("llama-tiny-hd64", dict(qk_norm=True), None, {}, r"q/k norm \(Qwen3\) needs head_dim 128"),
    ("phi3-tiny", dict(qk_norm=True), None, {}, r"q/k norm \(Qwen3\) needs head_dim 128"),
    ("phi3-tiny", dict(qkv_bias=True), None, {}, r"qkv bias \(Qwen2\) needs head_dim 128 or 64"),
    ("qwen3-tiny", dict(qkv_bias=True), None, {}, r"qkv bias \(Qwen2\) and q/k norm \(Qwen3\) cannot be combined"),
    ("llama-tiny-hd64", GRANITE, None, {}, r"model scalars \(Granite\) need head_dim 128: Granite with 64-dim heads"),
    ("phi3-tiny", GRANITE, None, {}, r"model scalars \(Granite\) need head_dim 128: Granite with 96-dim heads"),
    ("llama-tiny-hd64", dict(embedding_multiplier=2.0), None, {}, "Granite with 64-dim heads"),
    ("llama-tiny-hd64", dict(attention_multiplier=0.125), None, {}, "Granite with 64-dim heads"),
    # tensor parallelism
    ("granite-tiny", dict(vocab=1024), None, dict(tp_size=2),
     r"Granite \(residual_multiplier != 1\) is not supported with tensor parallelism"),
    ("qwen3-tiny", dict(vocab=1024), None, dict(tp_size=2), r"q/k norm \(Qwen3\) is supported on a single GPU only"),
    ("qwen2.5-7b", None, None, dict(tp_size=2), r"qkv bias \(Qwen2\) is supported on a single GPU only"),
    ("mistral-7b-v0.1", None, None, dict(tp_size=2), "sliding-window attention is supported on a single GPU only"),
    ("phi3-mini-4k", None, None, dict(tp_size=2), "head_dim 96 is supported on a single GPU only"),
    ("llama3.2-1b", None, None, dict(tp_size=2), "head_dim 64 is supported on a single GPU only"),
    ("opt-125m", None, None, dict(tp_size=2), r"OPT runs on a single GPU only \(tp_size must be 1\)"),
    ("starcoder-15b", None, None, dict(tp_size=2), r"GPTBigCode runs on a single GPU only \(tp_size must be 1\)"),
    # LoRA
    ("gpt-bigcode-tiny", None, None, dict(max_loras=2), "GPTBigCode: LoRA adapter slots are not supported"),
    ("opt-tiny", None, None, dict(max_loras=2), "OPT: LoRA adapter slots are not supported"),
    ("phi3-tiny", None, None, dict(max_loras=2), "head_dim 96: LoRA adapter slots are not supported"),
    # values
    ("mistral-tiny", dict(sliding_window=-1), None, {}, r"sliding window must be >= 0"),
    *[("granite-tiny", None, {name: value}, {}, "model scalars must be finite and non-negative")
      for name in ("embedding_multiplier", "residual_multiplier", "attention_multiplier", "logit_scale")
      for value in (-1.0, math.nan, math.inf)],
    ("tiny", None, dict(abi_version=8), {}, "ABI version mismatch"),
]


@pytest.mark.parametrize("preset,model,fields,options,reason", REFUSED)
def test_refused_with_its_reason(preset, model, fields, options, reason):
    err = config_error(_cfg(preset, model, fields, **options))
    assert err is not None, (preset, model, fields, options)
    assert re.search(reason, err), err


@pytest.mark.parametrize("preset", sorted(PRESETS))
@pytest.mark.parametrize("caching", [False, True])
def test_every_preset_passes_on_one_gpu(preset, caching):
    assert config_error(_cfg(preset, enable_prefix_caching=caching)) is None


@pytest.mark.parametrize("preset,model,fields,options", [
    ("llama3-8b", None, None, dict(tp_size=2)),
    ("llama3-70b", None, None, dict(tp_size=8, tp_rank=7, enable_prefix_caching=True)),
    ("phi3-medium-4k", None, None, dict(tp_size=2)),              # the library serves it; the loader refuses Phi-3
    ("granite-tiny", dict(vocab=1024, residual_multiplier=1.0), None, dict(tp_size=2)),  # no residual multiplier
    ("llama3.1-8b", None, None, dict(tp_size=4)),                 # a scaled rotary table under TP
    ("granite-tiny", None, dict(embedding_multiplier=0.0, residual_multiplier=0.0, attention_multiplier=0.0,
                                logit_scale=0.0), {}),            # 0: the Llama default
    ("llama-tiny-hd64", dict(embedding_multiplier=1.0, residual_multiplier=1.0, logits_scaling=1.0), None, {}),
    ("qwen2-tiny-hd64", None, None, {}),
    ("mistral-tiny", dict(sliding_window=0), None, {}),
    ("phi3-tiny", dict(sliding_window=40), None, {}),
    ("tiny", None, None, dict(max_loras=4, max_lora_rank=64)),
])
def test_valid_configs_pass(preset, model, fields, options):
    assert config_error(_cfg(preset, model, fields, **options)) is None


def test_engine_config_describes_the_model():
    g = engine_config(PRESETS["granite-tiny"])
    assert (g.embedding_multiplier, g.attention_multiplier) == (12.0, C.c_float(1.0 / 128).value)
    assert g.residual_multiplier == C.c_float(0.22).value and g.logit_scale == C.c_float(1.0 / 3.0).value
    assert engine_config(PRESETS["llama3.1-8b"]).rope_table_from_host == 1
    assert engine_config(PRESETS["llama3-8b"]).rope_table_from_host == 0
    assert engine_config(PRESETS["qwen3-tiny"]).qk_norm == 1 and engine_config(PRESETS["qwen2-tiny"]).qkv_bias == 1
    assert engine_config(PRESETS["mistral-tiny"]).sliding_window == 40
    assert engine_config(PRESETS["mistral-7b-v0.3"]).sliding_window == 0
    assert engine_config(PRESETS["tiny"], enable_prefix_caching=True).enable_prefix_caching == 1
    lib = _lib.load_library()
    assert lib.tgis_config_check(None) != 0 and "null" in _lib.last_error(lib)
