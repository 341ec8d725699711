"""The rotary table of the Llama stack, computed on the host and handed to the engine as the weight "tgis.rope_cos_sin"
([max_model_len][head_dim] bf16 = cos | sin).  The engine's built-in table is the unscaled one; a model with rope_type
"llama3" frequency scaling (Llama-3.1 / 3.2) or LongRoPE (Phi-3 128k) gets this one, and the engine refuses to start
without it."""
from __future__ import annotations

import logging

logger = logging.getLogger("vllm_tgis_adapter.engine")


def longrope_factors(mc) -> tuple[str, tuple[float, ...]]:
    """("long" | "short", the rescale factors [head_dim / 2]) of a LongRoPE model.  As vLLM's
    Phi3LongRoPEScaledRotaryEmbedding, the choice is made once per engine, for every position: the long factors when
    max_model_len exceeds original_max_position_embeddings, the short ones otherwise.  (transformers instead switches per
    forward pass, by the largest position in it.)"""
    if mc.max_model_len > mc.rope_original_max_pos:
        return "long", mc.rope_long_factor
    return "short", mc.rope_short_factor


def longrope_mscale(mc) -> float:
    """cos / sin multiplier of a LongRoPE model: sqrt(1 + ln(s) / ln(original)) with s = max_position_embeddings /
    original_max_position_embeddings, or 1 when s <= 1 (vLLM Phi3LongRoPEScaledRotaryEmbedding; transformers
    _compute_longrope_parameters' attention_factor)"""
    import math

    s = mc.rope_max_position_embeddings / mc.rope_original_max_pos
    return 1.0 if s <= 1.0 else math.sqrt(1 + math.log(s) / math.log(mc.rope_original_max_pos))


def rope_inv_freq(mc):
    """fp32 rotary frequencies [head_dim / 2].  rope_type "llama3" (HF modeling_rope_utils `_compute_llama3_parameters`;
    vllm rotary_embedding Llama3RotaryEmbedding): a frequency whose wavelength exceeds original_max_pos / low_freq_factor
    is divided by `factor`, one below original_max_pos / high_freq_factor is kept, and the band between is interpolated."""
    import math

    import torch

    d = mc.head_dim
    if mc.rope_longrope:   # LongRoPE: 1 / (factor_i * theta^(2i / d)), in fp32
        _, factor = longrope_factors(mc)
        ext = torch.tensor(factor, dtype=torch.float32)
        return 1.0 / (ext * mc.rope_theta ** (torch.arange(0, d, 2, dtype=torch.float32) / d))
    inv_freq = 1.0 / (mc.rope_theta ** (torch.arange(0, d, 2, dtype=torch.float32) / d))
    if not mc.rope_scaled:
        return inv_freq
    factor, lo, hi, orig = (mc.rope_scaling_factor, mc.rope_low_freq_factor, mc.rope_high_freq_factor,
                            mc.rope_original_max_pos)
    wavelen = 2 * math.pi / inv_freq
    scaled = torch.where(wavelen > orig / lo, inv_freq / factor, inv_freq)
    smooth = (orig / wavelen - lo) / (hi - lo)
    smoothed = (1 - smooth) * scaled / factor + smooth * scaled
    medium = ~(wavelen < orig / hi) * ~(wavelen > orig / lo)
    return torch.where(medium, smoothed, scaled)


def rope_cos_sin(mc):
    """HF LlamaRotaryEmbedding / vllm rotary_embedding base.py: fp32 table -> bf16.  LongRoPE: cos and sin are multiplied
    by longrope_mscale in fp32 before the rounding."""
    import torch

    inv_freq = rope_inv_freq(mc)
    freqs = torch.outer(torch.arange(mc.max_model_len, dtype=torch.float32), inv_freq)
    if mc.rope_longrope:
        which, _ = longrope_factors(mc)
        mscale = longrope_mscale(mc)
        logger.warning("LongRoPE: using the %s factors for every position (max_model_len %d %s "
                       "original_max_position_embeddings %d), mscale %.6f", which, mc.max_model_len,
                       ">" if which == "long" else "<=", mc.rope_original_max_pos, mscale)
        return torch.cat([freqs.cos() * mscale, freqs.sin() * mscale], dim=-1).to(torch.bfloat16)
    return torch.cat([freqs.cos(), freqs.sin()], dim=-1).to(torch.bfloat16)
