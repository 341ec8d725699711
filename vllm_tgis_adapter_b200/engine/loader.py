"""Build the engine the way `build_async_engine_client(args)` does for the reference
(/root/reference/src/vllm_tgis_adapter/__main__.py:48): read the HF model directory (config.json + *.safetensors),
stream each tensor into libtgis_engine.so ("PyTorch tensors for weights only"), attach a tokenizer.

Offline builds have no checkpoints (SURVEY.md §0): `--model <preset> --synthetic-weights` creates seeded N(0, 0.02)
weights of the named architecture on the device instead."""
from __future__ import annotations

import dataclasses
import json
import logging
from pathlib import Path

from .async_engine import AsyncTGISEngine
from .core import PRESETS, ModelConfig, NativeEngine, config_error, engine_config
from .rope import rope_cos_sin, rope_inv_freq  # noqa: F401  (the table every Llama engine is given: rope.py)
from .tokenizer import load_tokenizer

logger = logging.getLogger("vllm_tgis_adapter.engine")


def model_config_from_hf(path: Path, max_model_len: int | None) -> ModelConfig:
    cfg = json.loads((path / "config.json").read_text())
    archs = cfg.get("architectures") or []
    if cfg.get("model_type") == "opt" or any("OPT" in a for a in archs):
        return _opt_model_config(cfg, max_model_len)
    if cfg.get("model_type") == "gpt_bigcode" or "GPTBigCodeForCausalLM" in archs:
        return _gpt_bigcode_model_config(cfg, max_model_len)
    if cfg.get("model_type") == "granite" or "GraniteForCausalLM" in archs:
        return _granite_model_config(cfg, max_model_len)
    if cfg.get("model_type") == "qwen3" or "Qwen3ForCausalLM" in archs:
        return _qwen3_model_config(cfg, max_model_len)
    if cfg.get("model_type") == "mistral" or "MistralForCausalLM" in archs:
        return _mistral_model_config(cfg, max_model_len)
    if cfg.get("model_type") == "phi3" or "Phi3ForCausalLM" in archs:
        return _phi3_model_config(cfg, max_model_len)
    if cfg.get("model_type") == "qwen2" or "Qwen2ForCausalLM" in archs:
        if cfg.get("attention_bias") is False:
            # Qwen2's q / k / v projections always carry a bias (transformers and vLLM hard-code bias=True; Qwen2Config
            # has no attention_bias key).  A config that declares bias-free projections was written for another
            # architecture (a Llama- or Qwen3-style one) and its checkpoint has no bias tensors to load.
            raise ValueError(f"unsupported model architecture {archs or cfg.get('model_type')}: attention_bias false "
                             "declares projections without biases, but Qwen2ForCausalLM always has q/k/v biases")
        return _qwen2_model_config(cfg, max_model_len)
    if cfg.get("model_type") != "llama" and not any("Llama" in a for a in archs):
        raise ValueError(f"unsupported model architecture {archs or cfg.get('model_type')}: only Llama-family "
                         "decoders (RMSNorm, RoPE, GQA, SwiGLU) and OPT are implemented")
    hidden, heads = cfg["hidden_size"], cfg["num_attention_heads"]
    head_dim = cfg.get("head_dim") or hidden // heads
    if head_dim not in (64, 128):
        raise ValueError(f"head_dim {head_dim} unsupported (the attention kernels exist for 64 and 128)")
    theta, scaling = _llama_rope(cfg)
    derived = cfg.get("max_position_embeddings", 8192)
    if max_model_len is not None and max_model_len > derived:
        raise ValueError(f"max_model_len {max_model_len} exceeds the model's max_position_embeddings {derived}")
    return ModelConfig(n_layers=cfg["num_hidden_layers"], hidden=hidden, n_q_heads=heads,
                       n_kv_heads=cfg.get("num_key_value_heads", heads), ffn=cfg["intermediate_size"],
                       vocab=cfg["vocab_size"], head_dim=head_dim, rope_theta=theta,
                       rms_eps=float(cfg.get("rms_norm_eps", 1e-5)), max_model_len=max_model_len or min(derived, 8192),
                       tie_word_embeddings=bool(cfg.get("tie_word_embeddings", False)), **scaling)


def _llama_rope(cfg: dict) -> tuple[float, dict]:
    """(rope_theta, ModelConfig rope_* fields) of a Llama config.json, from either spelling: `rope_scaling` beside a
    top-level `rope_theta` (transformers 4), or `rope_parameters` holding both (transformers 5).  Only the default rotary
    embedding and rope_type "llama3" (Llama-3.1 / 3.2) are implemented; every other type is refused by name."""
    rope = cfg.get("rope_parameters") or cfg.get("rope_scaling") or {}
    theta = float(rope.get("rope_theta") or cfg.get("rope_theta") or 10000.0)
    kind = rope.get("rope_type") or rope.get("type") or "default"
    if kind == "default":
        return theta, {}
    if kind != "llama3":
        raise ValueError(f"rope scaling type {kind!r} is not supported (only 'default' and 'llama3' are implemented)")
    missing = [k for k in ("factor", "low_freq_factor", "high_freq_factor", "original_max_position_embeddings")
               if k not in rope]
    if missing:
        raise ValueError(f"rope scaling type 'llama3' needs {', '.join(missing)}")
    return theta, dict(rope_scaling_factor=float(rope["factor"]), rope_low_freq_factor=float(rope["low_freq_factor"]),
                       rope_high_freq_factor=float(rope["high_freq_factor"]),
                       rope_original_max_pos=int(rope["original_max_position_embeddings"]))


def _granite_model_config(cfg: dict, max_model_len: int | None) -> ModelConfig:
    """ibm-granite GraniteForCausalLM config.json -> the Llama stack plus its four scalars (vllm
    model_executor/models/granite.py).  Variants the engine would serve wrongly are refused, each with its reason."""
    hidden, heads = cfg["hidden_size"], cfg["num_attention_heads"]
    head_dim = cfg.get("head_dim") or hidden // heads
    problems = []
    if cfg.get("attention_bias") or cfg.get("mlp_bias"):
        problems.append("attention_bias / mlp_bias (the Llama stack has no projection biases)")
    if cfg.get("rope_scaling"):
        problems.append("rope_scaling")
    rope = cfg.get("rope_parameters") or {}
    if rope.get("rope_type", "default") != "default" or set(rope) - {"rope_type", "rope_theta"}:
        problems.append(f"rope_parameters {rope} (only the default rotary embedding is implemented)")
    if head_dim != 128:
        problems.append(f"head_dim {head_dim} (the attention kernels need 128; zero-padding smaller heads does not "
                        "commute with RoPE)")
    if problems:
        raise ValueError("unsupported Granite variant: " + "; ".join(problems))
    derived = cfg.get("max_position_embeddings", 4096)
    if max_model_len is not None and max_model_len > derived:
        raise ValueError(f"max_model_len {max_model_len} exceeds the model's max_position_embeddings {derived}")
    theta = rope.get("rope_theta", cfg.get("rope_theta", 10000.0))
    return ModelConfig(n_layers=cfg["num_hidden_layers"], hidden=hidden, n_q_heads=heads,
                       n_kv_heads=cfg.get("num_key_value_heads", heads), ffn=cfg["intermediate_size"],
                       vocab=cfg["vocab_size"], head_dim=head_dim, rope_theta=float(theta),
                       rms_eps=float(cfg.get("rms_norm_eps", 1e-6)), max_model_len=max_model_len or min(derived, 8192),
                       tie_word_embeddings=bool(cfg.get("tie_word_embeddings", True)),
                       embedding_multiplier=float(cfg.get("embedding_multiplier", 1.0)),
                       residual_multiplier=float(cfg.get("residual_multiplier", 1.0)),
                       attention_multiplier=float(cfg.get("attention_multiplier") or 0.0),
                       logits_scaling=float(cfg.get("logits_scaling", 1.0)))


def _qwen3_model_config(cfg: dict, max_model_len: int | None) -> ModelConfig:
    """Qwen/Qwen3-* Qwen3ForCausalLM config.json -> the Llama stack plus the per-head q / k RMSNorm (vllm
    model_executor/models/qwen3.py).  Variants the engine would serve wrongly are refused, each with its reason; the
    rotary embedding is read as for Llama (_llama_rope: yarn and the other scaled types are refused by name)."""
    hidden, heads = cfg["hidden_size"], cfg["num_attention_heads"]
    head_dim = cfg.get("head_dim") or hidden // heads
    problems = []
    if cfg.get("attention_bias"):
        problems.append("attention_bias (the Llama stack has no projection biases)")
    if cfg.get("use_sliding_window"):
        problems.append("use_sliding_window (every layer attends to the whole context here)")
    other = sorted({t for t in cfg.get("layer_types") or [] if t != "full_attention"})
    if other:
        problems.append(f"layer_types {other} (only full_attention is implemented)")
    if head_dim != 128:
        problems.append(f"head_dim {head_dim} (the q/k norm is implemented for 128-dim heads)")
    if problems:
        raise ValueError("unsupported Qwen3 variant: " + "; ".join(problems))
    theta, scaling = _llama_rope(cfg)
    derived = cfg.get("max_position_embeddings", 40960)
    if max_model_len is not None and max_model_len > derived:
        raise ValueError(f"max_model_len {max_model_len} exceeds the model's max_position_embeddings {derived}")
    return ModelConfig(n_layers=cfg["num_hidden_layers"], hidden=hidden, n_q_heads=heads,
                       n_kv_heads=cfg.get("num_key_value_heads", heads), ffn=cfg["intermediate_size"],
                       vocab=cfg["vocab_size"], head_dim=head_dim, rope_theta=theta,
                       rms_eps=float(cfg.get("rms_norm_eps", 1e-6)), max_model_len=max_model_len or min(derived, 8192),
                       tie_word_embeddings=bool(cfg.get("tie_word_embeddings", False)), qk_norm=True, **scaling)


def _mistral_model_config(cfg: dict, max_model_len: int | None) -> ModelConfig:
    """mistralai MistralForCausalLM config.json -> the Llama stack with a sliding window in every layer (vLLM applies a
    model-wide window to each layer).  transformers' MistralConfig defaults sliding_window to 4096, so a config.json
    without the key is windowed; null or 0 is no window.  Variants the engine would serve wrongly are refused, each with
    its reason; the rotary embedding is read as for Llama (_llama_rope: yarn and the other scaled types are refused)."""
    hidden, heads = cfg["hidden_size"], cfg["num_attention_heads"]
    head_dim = cfg.get("head_dim") or hidden // heads
    window = cfg.get("sliding_window", 4096)
    problems = []
    if cfg.get("attention_bias") or cfg.get("mlp_bias"):
        problems.append("attention_bias / mlp_bias (the Llama stack has no projection biases)")
    if cfg.get("llama_4_scaling"):
        problems.append("llama_4_scaling (position-dependent query scaling is not implemented)")
    kinds = sorted(set(cfg.get("layer_types") or []))
    if len(kinds) > 1:
        problems.append(f"layer_types mixing {kinds} (per-layer windows are not implemented: one window serves every "
                        "layer)")
    if window is not None and (not isinstance(window, int) or isinstance(window, bool) or window < 0):
        problems.append(f"sliding_window {window!r} (a non-negative integer or null)")
    if head_dim not in (64, 128):
        problems.append(f"head_dim {head_dim} (the attention kernels exist for 64 and 128)")
    if problems:
        raise ValueError("unsupported Mistral variant: " + "; ".join(problems))
    theta, scaling = _llama_rope(cfg)
    derived = cfg.get("max_position_embeddings", 32768)
    if max_model_len is not None and max_model_len > derived:
        raise ValueError(f"max_model_len {max_model_len} exceeds the model's max_position_embeddings {derived}")
    return ModelConfig(n_layers=cfg["num_hidden_layers"], hidden=hidden, n_q_heads=heads,
                       n_kv_heads=cfg.get("num_key_value_heads", heads), ffn=cfg["intermediate_size"],
                       vocab=cfg["vocab_size"], head_dim=head_dim, rope_theta=theta,
                       rms_eps=float(cfg.get("rms_norm_eps", 1e-6)), max_model_len=max_model_len or min(derived, 8192),
                       tie_word_embeddings=bool(cfg.get("tie_word_embeddings", False)), sliding_window=window or None,
                       **scaling)


def _qwen2_model_config(cfg: dict, max_model_len: int | None) -> ModelConfig:
    """Qwen/Qwen2-* and Qwen2.5-* Qwen2ForCausalLM config.json -> the Llama stack with a bias on the q, k and v
    projections (vllm model_executor/models/qwen2.py).  Where vLLM and transformers' defaults differ, vLLM's are taken:
    head_dim is hidden_size // num_attention_heads, and a config without a rotary theta gets 1e6.  Variants the engine
    would serve wrongly are refused, each with its reason; the rotary embedding is read as for Llama (_llama_rope: yarn
    and the other scaled types are refused by name)."""
    hidden, heads = cfg["hidden_size"], cfg["num_attention_heads"]
    head_dim = hidden // heads
    problems = []
    if cfg.get("head_dim") not in (None, head_dim):
        problems.append(f"head_dim {cfg['head_dim']} != hidden_size // num_attention_heads = {head_dim} (vLLM computes "
                        "the latter, transformers reads the former: the two would build different models)")
    if head_dim not in (64, 128):
        problems.append(f"head_dim {head_dim} (the attention kernels exist for 64 and 128)")
    if cfg.get("use_sliding_window"):
        problems.append("use_sliding_window (every layer attends to the whole context here)")
    other = sorted({t for t in cfg.get("layer_types") or [] if t != "full_attention"})
    if other:
        problems.append(f"layer_types {other} (only full_attention is implemented)")
    if cfg.get("qk_norm"):
        problems.append("qk_norm (a q/k norm together with the qkv bias is not implemented)")
    if cfg.get("is_causal") is False:
        problems.append("is_causal false (bidirectional embedding models are not generative)")
    if cfg.get("dual_chunk_attention_config"):
        problems.append("dual_chunk_attention_config (dual-chunk attention is not implemented)")
    if problems:
        raise ValueError("unsupported Qwen2 variant: " + "; ".join(problems))
    rope = cfg.get("rope_parameters") or cfg.get("rope_scaling") or {}
    if not (rope.get("rope_theta") or cfg.get("rope_theta")):
        cfg = {**cfg, "rope_theta": 1000000.0}   # vllm qwen2.py: set_default_rope_theta(config, 1000000)
    theta, scaling = _llama_rope(cfg)
    derived = cfg.get("max_position_embeddings", 32768)
    if max_model_len is not None and max_model_len > derived:
        raise ValueError(f"max_model_len {max_model_len} exceeds the model's max_position_embeddings {derived}")
    return ModelConfig(n_layers=cfg["num_hidden_layers"], hidden=hidden, n_q_heads=heads,
                       n_kv_heads=cfg.get("num_key_value_heads", heads), ffn=cfg["intermediate_size"],
                       vocab=cfg["vocab_size"], head_dim=head_dim, rope_theta=theta,
                       rms_eps=float(cfg.get("rms_norm_eps", 1e-6)), max_model_len=max_model_len or min(derived, 8192),
                       tie_word_embeddings=bool(cfg.get("tie_word_embeddings", False)), qkv_bias=True, **scaling)


def _phi3_model_config(cfg: dict, max_model_len: int | None) -> ModelConfig:
    """microsoft Phi-3 / Phi-3.5 / Phi-4 Phi3ForCausalLM config.json -> the Llama stack (vLLM's Phi3ForCausalLM is a plain
    subclass of LlamaForCausalLM), with head_dim 96, 128 or 64, rope_type "longrope" (legacy spellings "su" and "yarn",
    as transformers' Phi3Config normalises them) and a model-wide sliding window (null: none).  The checkpoint's fused
    qkv_proj / gate_up_proj tensors are split at load (split_fused).  Variants the engine would serve wrongly are refused,
    each with its reason."""
    hidden, heads = cfg["hidden_size"], cfg["num_attention_heads"]
    head_dim = cfg.get("head_dim") or hidden // heads
    window = cfg.get("sliding_window")
    rope = cfg.get("rope_scaling") or cfg.get("rope_parameters") or {}   # transformers' Phi3Config: rope_scaling first
    kind = rope.get("rope_type") or rope.get("type") or "default"
    problems = []
    partial = rope.get("partial_rotary_factor", cfg.get("partial_rotary_factor", 1.0))
    if partial != 1.0:
        problems.append(f"partial_rotary_factor {partial} (only full-width rotary embeddings are implemented)")
    for key in ("short_mscale", "long_mscale", "attention_factor"):
        if rope.get(key) is not None:
            problems.append(f"rope {key} {rope[key]} (only the default LongRoPE scale sqrt(1 + ln s / ln original) is "
                            "implemented)")
    kinds = sorted(set(cfg.get("layer_types") or []))
    if len(kinds) > 1:
        problems.append(f"layer_types mixing {kinds} (per-layer windows are not implemented: one window serves every "
                        "layer)")
    if window is not None and (not isinstance(window, int) or isinstance(window, bool) or window < 0):
        problems.append(f"sliding_window {window!r} (a non-negative integer or null)")
    if head_dim not in (64, 96, 128):
        problems.append(f"head_dim {head_dim} (the attention kernels exist for 64, 96 and 128)")
    if kind not in ("default", "longrope", "su", "yarn"):
        problems.append(f"rope scaling type {kind!r} (only 'default' and 'longrope' are implemented)")
    if problems:
        raise ValueError("unsupported Phi-3 variant: " + "; ".join(problems))
    theta = float(rope.get("rope_theta") or cfg.get("rope_theta") or 10000.0)
    derived = cfg.get("max_position_embeddings", 4096)
    if max_model_len is not None and max_model_len > derived:
        raise ValueError(f"max_model_len {max_model_len} exceeds the model's max_position_embeddings {derived}")
    scaling = {}
    if kind != "default":
        orig = rope.get("original_max_position_embeddings") or cfg.get("original_max_position_embeddings")
        long_f, short_f = rope.get("long_factor"), rope.get("short_factor")
        if not orig or not long_f or not short_f:
            raise ValueError("rope scaling type 'longrope' needs long_factor, short_factor and "
                             "original_max_position_embeddings")
        if len(long_f) != head_dim // 2 or len(short_f) != head_dim // 2:
            raise ValueError(f"longrope long_factor / short_factor must have head_dim / 2 = {head_dim // 2} entries, got "
                             f"{len(long_f)} / {len(short_f)}")
        scaling = dict(rope_long_factor=tuple(float(x) for x in long_f),
                       rope_short_factor=tuple(float(x) for x in short_f), rope_original_max_pos=int(orig),
                       rope_max_position_embeddings=int(derived))
    return ModelConfig(n_layers=cfg["num_hidden_layers"], hidden=hidden, n_q_heads=heads,
                       n_kv_heads=cfg.get("num_key_value_heads") or heads, ffn=cfg["intermediate_size"],
                       vocab=cfg["vocab_size"], head_dim=head_dim, rope_theta=theta,
                       rms_eps=float(cfg.get("rms_norm_eps", 1e-5)), max_model_len=max_model_len or min(derived, 8192),
                       tie_word_embeddings=bool(cfg.get("tie_word_embeddings", False)), sliding_window=window or None,
                       fused_projections=True, **scaling)


def split_fused(name: str, t, mc: ModelConfig) -> list:
    """[(name, tensor)] to load for one checkpoint tensor: Phi-3's self_attn.qkv_proj.weight as its q | k | v rows and
    mlp.gate_up_proj.weight as gate (rows [0, ffn)) | up (rows [ffn, 2 ffn)) under the separate projections' names
    (HF Phi3MLP's chunk order, vLLM's merged column order); every other tensor as it is"""
    if name.endswith("self_attn.qkv_proj.weight"):
        base = name[: -len("qkv_proj.weight")]
        q, kv = mc.n_q_heads * mc.head_dim, mc.n_kv_heads * mc.head_dim
        if t.shape[0] != q + 2 * kv:
            raise ValueError(f"{name}: {t.shape[0]} rows, expected (n_q + 2 n_kv) * head_dim = {q + 2 * kv}")
        return [(base + "q_proj.weight", t[:q]), (base + "k_proj.weight", t[q:q + kv]),
                (base + "v_proj.weight", t[q + kv:])]
    if name.endswith("mlp.gate_up_proj.weight"):
        base = name[: -len("gate_up_proj.weight")]
        if t.shape[0] != 2 * mc.ffn:
            raise ValueError(f"{name}: {t.shape[0]} rows, expected 2 * intermediate_size = {2 * mc.ffn}")
        return [(base + "gate_proj.weight", t[:mc.ffn]), (base + "up_proj.weight", t[mc.ffn:])]
    return [(name, t)]


def _opt_model_config(cfg: dict, max_model_len: int | None) -> ModelConfig:
    """facebook/opt-* config.json -> ModelConfig(arch="opt").  The variants vLLM's OPT model handles with extra modules
    (opt-350m: post-LayerNorm + project_in/out) are refused rather than silently mis-served."""
    hidden, heads = cfg["hidden_size"], cfg["num_attention_heads"]
    head_dim = hidden // heads
    problems = []
    if head_dim not in (64, 128):
        problems.append(f"head_dim {head_dim} (64 or 128)")
    if not cfg.get("do_layer_norm_before", True):
        problems.append("do_layer_norm_before=false")
    if cfg.get("word_embed_proj_dim", hidden) != hidden:
        problems.append("word_embed_proj_dim != hidden_size")
    if cfg.get("activation_function", "relu") != "relu":
        problems.append(f"activation_function {cfg.get('activation_function')}")
    if not cfg.get("enable_bias", True) or not cfg.get("layer_norm_elementwise_affine", True):
        problems.append("enable_bias / layer_norm_elementwise_affine = false")
    if cfg.get("_remove_final_layer_norm", False):
        problems.append("_remove_final_layer_norm")
    if problems:
        raise ValueError("unsupported OPT variant: " + ", ".join(problems))
    derived = cfg.get("max_position_embeddings", 2048)
    if max_model_len is not None and max_model_len > derived:
        raise ValueError(f"max_model_len {max_model_len} exceeds the model's max_position_embeddings {derived}")
    return ModelConfig(n_layers=cfg["num_hidden_layers"], hidden=hidden, n_q_heads=heads, n_kv_heads=heads,
                       ffn=cfg["ffn_dim"], vocab=cfg["vocab_size"], head_dim=head_dim, rms_eps=1e-5,  # nn.LayerNorm default
                       max_model_len=max_model_len or derived, arch="opt")


def _gpt_bigcode_model_config(cfg: dict, max_model_len: int | None) -> ModelConfig:
    """bigcode / ibm-granite GPTBigCodeForCausalLM config.json -> ModelConfig(arch="gpt_bigcode"), read as vLLM's
    gpt_bigcode.py reads it: n_inner None is 4 n_embd, multi_query is one kv head, n_positions bounds max_model_len and
    is its default.  Variants the engine would serve wrongly are refused, each with its reason."""
    hidden, heads = cfg.get("n_embd", 768), cfg.get("n_head", 12)
    head_dim = hidden // heads
    problems = []
    act = cfg.get("activation_function", "gelu_pytorch_tanh")
    if act != "gelu_pytorch_tanh":
        problems.append(f"activation_function {act!r} (only gelu_pytorch_tanh is implemented)")
    if cfg.get("scale_attn_weights", True) is False:
        problems.append("scale_attn_weights false (the attention kernels scale the scores by 1 / sqrt(head_dim))")
    if head_dim != 128 or hidden != heads * head_dim:
        problems.append(f"head_dim {hidden} / {heads} (the GPTBigCode attention path needs 128-dim heads)")
    if problems:
        raise ValueError("unsupported GPTBigCode variant: " + "; ".join(problems))
    derived = cfg.get("n_positions", 1024)
    if max_model_len is not None and max_model_len > derived:
        raise ValueError(f"max_model_len {max_model_len} exceeds the model's n_positions {derived}")
    return ModelConfig(n_layers=cfg.get("n_layer", 12), hidden=hidden, n_q_heads=heads,
                       n_kv_heads=1 if cfg.get("multi_query", True) else heads,
                       ffn=cfg.get("n_inner") or 4 * hidden, vocab=cfg.get("vocab_size", 50257), head_dim=head_dim,
                       rms_eps=float(cfg.get("layer_norm_epsilon", 1e-5)), max_model_len=max_model_len or derived,
                       arch="gpt_bigcode", tie_word_embeddings=bool(cfg.get("tie_word_embeddings", True)))


def skip_tensor(name: str) -> bool:
    """checkpoint tensors that are not weights: rotary inverse frequencies, and GPTBigCode's causal-mask buffers
    (.attn.bias / .attn.masked_bias, which older checkpoints saved; vLLM skips them too).  c_attn.bias is a weight, and
    no other architecture here names a tensor "attn.bias" (theirs are self_attn.*_proj.bias)."""
    return name.endswith(("rotary_emb.inv_freq", ".attn.bias", ".attn.masked_bias"))


def load_synthetic_weights(eng: NativeEngine, mc: ModelConfig, seed: int, device: int) -> None:
    import torch

    gen = torch.Generator(device=f"cuda:{device}").manual_seed(seed)

    def rnd(r, c):
        return (torch.randn(r, c, generator=gen, device=f"cuda:{device}", dtype=torch.float32) * 0.02).to(torch.bfloat16)

    if mc.arch == "opt":
        # HF OPT parameter names; LayerNorm weights around 1, small random biases (HF's init has zeros: random ones exercise
        # the bias paths).  lm_head is tied to embed_tokens (not loaded).
        H = mc.hidden

        def vec(n, s=0.02, base=0.0):
            return (base + torch.randn(n, generator=gen, device=f"cuda:{device}", dtype=torch.float32) * s).to(torch.bfloat16)

        eng.load_weight("model.decoder.embed_tokens.weight", rnd(mc.vocab, H))
        eng.load_weight("model.decoder.embed_positions.weight", rnd(mc.max_model_len + 2, H))
        eng.load_weight("model.decoder.final_layer_norm.weight", vec(H, 0.05, 1.0))
        eng.load_weight("model.decoder.final_layer_norm.bias", vec(H))
        for i in range(mc.n_layers):
            p = f"model.decoder.layers.{i}."
            for m in ("q_proj", "k_proj", "v_proj", "out_proj"):
                eng.load_weight(p + f"self_attn.{m}.weight", rnd(H, H))
                eng.load_weight(p + f"self_attn.{m}.bias", vec(H))
            eng.load_weight(p + "fc1.weight", rnd(mc.ffn, H))
            eng.load_weight(p + "fc1.bias", vec(mc.ffn))
            eng.load_weight(p + "fc2.weight", rnd(H, mc.ffn))
            eng.load_weight(p + "fc2.bias", vec(H))
            for ln in ("self_attn_layer_norm", "final_layer_norm"):
                eng.load_weight(p + ln + ".weight", vec(H, 0.05, 1.0))
                eng.load_weight(p + ln + ".bias", vec(H))
        return

    if mc.arch == "gpt_bigcode":
        # HF GPTBigCode parameter names, LayerNorms and biases as for OPT above; c_attn is q | k | v rows
        H, kv_dim = mc.hidden, mc.n_kv_heads * mc.head_dim

        def vec(n, s=0.02, base=0.0):
            return (base + torch.randn(n, generator=gen, device=f"cuda:{device}", dtype=torch.float32) * s).to(torch.bfloat16)

        eng.load_weight("transformer.wte.weight", rnd(mc.vocab, H))
        eng.load_weight("transformer.wpe.weight", rnd(mc.max_model_len, H))
        eng.load_weight("transformer.ln_f.weight", vec(H, 0.05, 1.0))
        eng.load_weight("transformer.ln_f.bias", vec(H))
        if not mc.tie_word_embeddings:
            eng.load_weight("lm_head.weight", rnd(mc.vocab, H))
        for i in range(mc.n_layers):
            p = f"transformer.h.{i}."
            eng.load_weight(p + "attn.c_attn.weight", rnd(H + 2 * kv_dim, H))
            eng.load_weight(p + "attn.c_attn.bias", vec(H + 2 * kv_dim))
            eng.load_weight(p + "attn.c_proj.weight", rnd(H, H))
            eng.load_weight(p + "attn.c_proj.bias", vec(H))
            eng.load_weight(p + "mlp.c_fc.weight", rnd(mc.ffn, H))
            eng.load_weight(p + "mlp.c_fc.bias", vec(mc.ffn))
            eng.load_weight(p + "mlp.c_proj.weight", rnd(H, mc.ffn))
            eng.load_weight(p + "mlp.c_proj.bias", vec(H))
            for ln in ("ln_1", "ln_2"):
                eng.load_weight(p + ln + ".weight", vec(H, 0.05, 1.0))
                eng.load_weight(p + ln + ".bias", vec(H))
        return

    q_dim, kv_dim = mc.n_q_heads * mc.head_dim, mc.n_kv_heads * mc.head_dim
    ones = torch.ones(mc.hidden, dtype=torch.bfloat16, device=f"cuda:{device}")
    eng.load_weight("model.embed_tokens.weight", rnd(mc.vocab, mc.hidden))
    if not mc.tie_word_embeddings:   # tied (Granite, Llama-3.2): the engine copies embed_tokens into the lm_head at start
        eng.load_weight("lm_head.weight", rnd(mc.vocab, mc.hidden))
    eng.load_weight("model.norm.weight", ones)
    for i in range(mc.n_layers):
        p = f"model.layers.{i}."
        if mc.fused_projections:   # Phi-3: the checkpoint's fused tensors, through the loader's split
            for n, t in split_fused(p + "self_attn.qkv_proj.weight", rnd(q_dim + 2 * kv_dim, mc.hidden), mc):
                eng.load_weight(n, t)
            for n, t in split_fused(p + "mlp.gate_up_proj.weight", rnd(2 * mc.ffn, mc.hidden), mc):
                eng.load_weight(n, t)
        else:
            eng.load_weight(p + "self_attn.q_proj.weight", rnd(q_dim, mc.hidden))
            eng.load_weight(p + "self_attn.k_proj.weight", rnd(kv_dim, mc.hidden))
            eng.load_weight(p + "self_attn.v_proj.weight", rnd(kv_dim, mc.hidden))
            eng.load_weight(p + "mlp.gate_proj.weight", rnd(mc.ffn, mc.hidden))
            eng.load_weight(p + "mlp.up_proj.weight", rnd(mc.ffn, mc.hidden))
        eng.load_weight(p + "self_attn.o_proj.weight", rnd(mc.hidden, q_dim))
        eng.load_weight(p + "mlp.down_proj.weight", rnd(mc.hidden, mc.ffn))
        eng.load_weight(p + "input_layernorm.weight", ones)
        eng.load_weight(p + "post_attention_layernorm.weight", ones)
        if mc.qk_norm:   # Qwen3: per-head norm weights of one head's width
            eng.load_weight(p + "self_attn.q_norm.weight", ones[:mc.head_dim])
            eng.load_weight(p + "self_attn.k_norm.weight", ones[:mc.head_dim])
        if mc.qkv_bias:  # Qwen2: projection biases (random: HF's init has zeros, which would not exercise the bias path)
            for m, n in (("q_proj", q_dim), ("k_proj", kv_dim), ("v_proj", kv_dim)):
                b = torch.randn(n, generator=gen, device=f"cuda:{device}", dtype=torch.float32) * 0.1
                eng.load_weight(p + f"self_attn.{m}.bias", b.to(torch.bfloat16))


def load_safetensors_dir(eng: NativeEngine, path: Path) -> None:
    from safetensors import safe_open

    files = sorted(path.glob("*.safetensors"))
    if not files:
        bins = sorted(path.glob("pytorch_model*.bin"))   # facebook/opt-125m ships pytorch_model.bin
        if not bins:
            raise ValueError(f"no *.safetensors or pytorch_model*.bin files under {path}")
        import torch

        for f in bins:
            for name, t in torch.load(str(f), map_location="cpu", weights_only=True).items():
                if not skip_tensor(name):
                    eng.load_weight(name, t)
        return
    for f in files:
        with safe_open(str(f), framework="pt", device="cpu") as sf:
            for name in sf.keys():  # noqa: SIM118
                if skip_tensor(name):
                    continue
                for n, t in split_fused(name, sf.get_tensor(name), eng.model):
                    eng.load_weight(n, t)


def _resolve_model(args):
    """(ModelConfig, checkpoint dir or None) from --model: a HF-format directory or a preset name + --synthetic-weights."""
    if not args.model:
        raise ValueError("--model / --model-name is required")
    path = Path(args.model)
    if path.is_dir():
        return model_config_from_hf(path, args.max_model_len), path
    if args.model in PRESETS:
        if not args.synthetic_weights:
            raise ValueError(f"--model {args.model} is a preset name: pass --synthetic-weights or a model directory")
        mc = dataclasses.replace(PRESETS[args.model])
        if args.max_model_len:
            mc.max_model_len = args.max_model_len
        return mc, None
    raise ValueError(f"model path {args.model} does not exist (no network access: hub ids cannot be resolved)")


def _engine_options(args, device: int, **tp_kw) -> dict:
    """NativeEngine's keyword arguments (engine_config's options) from the server's arguments"""
    return dict(max_num_seqs=args.max_num_seqs, max_batched_tokens=args.max_num_batched_tokens,
                gpu_mem_fraction=args.gpu_memory_utilization, device=device, seed=args.seed,
                max_loras=args.max_loras if getattr(args, "enable_lora", False) else 0,
                max_lora_rank=getattr(args, "max_lora_rank", 16),
                enable_prefix_caching=bool(getattr(args, "enable_prefix_caching", False)), **tp_kw)


def _make_native_engine(args, mc: ModelConfig, path, device: int, **tp_kw) -> NativeEngine:
    eng = NativeEngine(mc, **_engine_options(args, device, **tp_kw))
    if path is not None:
        load_safetensors_dir(eng, path)      # full tensors: a tensor-parallel engine keeps its rank's shard
    else:
        load_synthetic_weights(eng, mc, args.seed, device)
    if mc.arch == "llama":   # OPT and GPTBigCode have learned positions (part of the checkpoint), no rotary table
        eng.load_weight("tgis.rope_cos_sin", rope_cos_sin(mc))
    return eng


def _tp_worker_main(args, rank: int, tp: int, nccl_id: bytes, shm_name: str) -> None:
    """Ranks 1..tp-1 of a tensor-parallel server (one spawned process per GPU): build the rank's shard of the same
    model and follow rank 0's step plans (shared-memory control block, csrc/engine.cu worker_loop) until it shuts down."""
    import torch  # noqa: F401  (first: resolves libnccl for the engine library)

    mc, path = _resolve_model(args)
    eng = _make_native_engine(args, mc, path, args.device + rank, tp_size=tp, tp_rank=rank, nccl_id=nccl_id,
                              shm_name=shm_name)
    try:
        eng.worker_run()
    finally:
        eng.close()


def build_engine(args) -> AsyncTGISEngine:
    """`--tensor-parallel-size N` (reference: tgis_utils/args.py:139-148 maps --num-gpus / --num-shard onto it): this
    process is rank 0 (scheduler, sampler, gRPC); ranks 1..N-1 are spawned here, one process per GPU."""
    tp = args.tensor_parallel_size or 1
    mc, path = _resolve_model(args)
    tp_kw = {}
    # Phi-3's fused projections are split on the host into full tensors, which no rank shards
    if tp > 1 and mc.fused_projections:
        raise ValueError(f"Phi-3 is supported on a single GPU only: tensor_parallel_size {tp}")
    # every other refusal is the library's, made here before any rank is spawned or device touched
    err = config_error(engine_config(mc, **_engine_options(args, args.device, tp_size=tp)))
    if err:
        raise ValueError(err)
    if tp > 1:
        import multiprocessing as mp
        import os

        import torch  # noqa: F401

        nccl_id = NativeEngine.nccl_unique_id()
        shm_name = f"/tgis_tp_{os.getpid()}"
        ctx = mp.get_context("spawn")
        workers = [ctx.Process(target=_tp_worker_main, args=(args, r, tp, nccl_id, shm_name), daemon=True,
                               name=f"tgis-tp-rank{r}") for r in range(1, tp)]
        for w in workers:
            w.start()
        tp_kw = dict(tp_size=tp, tp_rank=0, nccl_id=nccl_id, shm_name=shm_name)
    eng = _make_native_engine(args, mc, path, args.device, **tp_kw)
    # the synthetic vocabulary only for synthetic models (preset + --synthetic-weights); a checkpoint directory without
    # tokenizer files is a start-up error
    tokenizer = load_tokenizer(args.tokenizer or (str(path) if path is not None else None), mc.vocab,
                               allow_synthetic=path is None)
    logger.info("engine ready: %s (tensor_parallel_size=%d)", mc, tp)
    return AsyncTGISEngine(eng, tokenizer, mc)
