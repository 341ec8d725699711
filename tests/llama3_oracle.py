"""Llama-3.1 / 3.2 oracle for the tests: oracle/llama_oracle.py's Llama restatement with the rope_type "llama3" frequency
scaling and tied embeddings.

The rule (transformers modeling_rope_utils `_compute_llama3_parameters`; vllm rotary_embedding Llama3RotaryEmbedding),
per rotary frequency f with wavelength w = 2 pi / f, all in fp32:

  w > original_max_pos / low_freq_factor    f / factor                        (long wavelengths: interpolated positions)
  w < original_max_pos / high_freq_factor   f                                 (short wavelengths: untouched)
  otherwise                                 (1 - s) * f / factor + s * f,  s = (original_max_pos / w - low) / (high - low)

It is written here one frequency at a time on numpy fp32 scalars, independently of the engine loader's tensor version
(vllm_tgis_adapter_b200/engine/loader.py rope_inv_freq); tests/test_llama3_cpu.py holds both to transformers' inv_freq
bit for bit (tests/golden/llama3_hd64_hf_*.json, scripts/gen_llama3_golden.py).
"""
from __future__ import annotations

import dataclasses
import math

import numpy as np
import torch

from oracle.llama_oracle import LlamaConfig, LlamaOracle, synthetic_weights as llama_synthetic_weights


@dataclasses.dataclass
class Llama3Config(LlamaConfig):
    rope_factor: float = 8.0
    rope_low_freq_factor: float = 1.0
    rope_high_freq_factor: float = 4.0
    rope_original_max_pos: int = 8192
    tie_word_embeddings: bool = False


# vllm_tgis_adapter_b200/engine/core.py PRESETS["llama-tiny-hd64"]
CONFIGS = {
    "llama-tiny-hd64": Llama3Config(n_layers=2, hidden=256, n_q_heads=4, n_kv_heads=2, ffn=512, vocab=1024, head_dim=64,
                                    rope_theta=10000.0, max_model_len=2048, rope_factor=8.0, rope_original_max_pos=64,
                                    tie_word_embeddings=True),
}


def llama3_inv_freq(cfg: Llama3Config) -> tuple[np.ndarray, list[str]]:
    """(fp32 frequencies [head_dim / 2], the band of each: "low" (divided), "mid" (interpolated), "high" (kept))"""
    f32 = np.float32
    d = cfg.head_dim
    two_pi = f32(2 * math.pi)
    factor, lo, hi = f32(cfg.rope_factor), f32(cfg.rope_low_freq_factor), f32(cfg.rope_high_freq_factor)
    orig = f32(cfg.rope_original_max_pos)
    out, bands = np.empty(d // 2, dtype=np.float32), []
    base = (1.0 / (cfg.rope_theta ** (torch.arange(0, d, 2, dtype=torch.float32) / d))).numpy()
    for i, f in enumerate(base):
        w = (f32(1.0) / f) * two_pi   # torch evaluates scalar / tensor as reciprocal(tensor) * scalar; so does this
        if w > orig / lo:
            out[i], band = f / factor, "low"
        elif w < orig / hi:
            out[i], band = f, "high"
        else:
            s = ((f32(1.0) / w) * orig - lo) / (hi - lo)
            out[i], band = (f32(1.0) - s) * f / factor + s * f, "mid"
        bands.append(band)
    return out, bands


def rope_table(cfg: Llama3Config, dtype: torch.dtype = torch.bfloat16) -> torch.Tensor:
    """[max_model_len, head_dim] = cos | sin of pos * scaled frequency, computed in fp32, in the model dtype"""
    inv_freq = torch.from_numpy(llama3_inv_freq(cfg)[0])
    freqs = torch.outer(torch.arange(cfg.max_model_len, dtype=torch.float32), inv_freq)
    return torch.cat([freqs.cos(), freqs.sin()], dim=-1).to(dtype)


def synthetic_weights(cfg: Llama3Config, seed: int = 0, dtype: torch.dtype = torch.bfloat16, **kw
                      ) -> dict[str, torch.Tensor]:
    """llama_oracle.synthetic_weights without lm_head.weight when the embeddings are tied"""
    w = llama_synthetic_weights(cfg, seed=seed, dtype=dtype, **kw)
    if cfg.tie_word_embeddings:
        del w["lm_head.weight"]
    return w


class Llama3Oracle(LlamaOracle):
    def __init__(self, cfg: Llama3Config, weights: dict[str, torch.Tensor], **kw):
        super().__init__(cfg, weights, **kw)   # (tied: self.lm_head is the embedding table)
        self.cos_sin = rope_table(cfg, self.dtype).to(self.device)
