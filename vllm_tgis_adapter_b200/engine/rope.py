"""The rotary table of the Llama stack, computed on the host and handed to the engine as the weight "tgis.rope_cos_sin"
([max_model_len][head_dim] bf16 = cos | sin).  The engine's built-in table is the unscaled one; a model with rope_type
"llama3" frequency scaling (Llama-3.1 / 3.2) gets this one, and the engine refuses to start without it."""
from __future__ import annotations


def rope_inv_freq(mc):
    """fp32 rotary frequencies [head_dim / 2].  rope_type "llama3" (HF modeling_rope_utils `_compute_llama3_parameters`;
    vllm rotary_embedding Llama3RotaryEmbedding): a frequency whose wavelength exceeds original_max_pos / low_freq_factor
    is divided by `factor`, one below original_max_pos / high_freq_factor is kept, and the band between is interpolated."""
    import math

    import torch

    d = mc.head_dim
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
    """HF LlamaRotaryEmbedding / vllm rotary_embedding base.py: fp32 table -> bf16."""
    import torch

    inv_freq = rope_inv_freq(mc)
    freqs = torch.outer(torch.arange(mc.max_model_len, dtype=torch.float32), inv_freq)
    return torch.cat([freqs.cos(), freqs.sin()], dim=-1).to(torch.bfloat16)
