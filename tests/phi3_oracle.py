"""Phi-3 oracle for the tests: tests/mistral_oracle.py's Llama restatement with the window, at any head_dim (96 for
Phi-3-mini), plus the LongRoPE rotary table and the fused checkpoint tensors.

LongRoPE (vllm rotary_embedding Phi3LongRoPEScaledRotaryEmbedding; transformers _compute_longrope_parameters), in fp32:

  inv_freq_i = 1 / (factor_i * theta^(2i / D))
  cos, sin   = cos(p * inv_freq) * mscale, sin(p * inv_freq) * mscale, then rounded to the model dtype
  mscale     = sqrt(1 + ln(s) / ln(original)),  s = max_position_embeddings / original (1 when s <= 1)

`factor` is the long list in the long regime and the short one otherwise.  vLLM picks the regime once per engine, by
max_model_len > original_max_position_embeddings; transformers picks it per forward pass, by the largest position in
it.  The oracle takes the regime as an argument, so it can follow either.

Phi-3 checkpoints store self_attn.qkv_proj.weight (q | k | v rows) and mlp.gate_up_proj.weight (gate | up rows);
`fuse` builds them from the separate projections.  The oracle is pinned to transformers' Phi3ForCausalLM by
tests/golden/phi3_hf_*.json (scripts/gen_phi3_golden.py).
"""
from __future__ import annotations

import dataclasses
import math

import torch

from mistral_oracle import MistralConfig, MistralOracle, synthetic_weights  # noqa: F401


@dataclasses.dataclass
class Phi3Config(MistralConfig):
    long_factor: tuple = ()
    short_factor: tuple = ()
    original_max_pos: int = 4096
    max_position_embeddings: int = 4096


def longrope_mscale(cfg: Phi3Config) -> float:
    s = cfg.max_position_embeddings / cfg.original_max_pos
    return 1.0 if s <= 1.0 else math.sqrt(1 + math.log(s) / math.log(cfg.original_max_pos))


def longrope_table(cfg: Phi3Config, regime: str, n_pos: int | None = None, dtype=torch.bfloat16) -> torch.Tensor:
    """[n_pos, head_dim] = cos | sin with the `regime` ("long" / "short") factors and the mscale, in the model dtype"""
    d = cfg.head_dim
    factor = torch.tensor(cfg.long_factor if regime == "long" else cfg.short_factor, dtype=torch.float32)
    inv_freq = 1.0 / (factor * cfg.rope_theta ** (torch.arange(0, d, 2, dtype=torch.float32) / d))
    freqs = torch.outer(torch.arange(n_pos or cfg.max_model_len, dtype=torch.float32), inv_freq)
    m = longrope_mscale(cfg)
    return torch.cat([freqs.cos() * m, freqs.sin() * m], dim=-1).to(dtype)


def engine_regime(cfg: Phi3Config, max_model_len: int) -> str:
    """vLLM's (and the engine's) choice: one regime for every position"""
    return "long" if max_model_len > cfg.original_max_pos else "short"


def fuse(weights: dict[str, torch.Tensor]) -> dict[str, torch.Tensor]:
    """separate q/k/v and gate/up projections -> Phi-3's fused checkpoint tensors"""
    out = {}
    for name, t in weights.items():
        if name.endswith(("self_attn.k_proj.weight", "self_attn.v_proj.weight", "mlp.up_proj.weight")):
            continue
        if name.endswith("self_attn.q_proj.weight"):
            p = name[: -len("q_proj.weight")]
            out[p + "qkv_proj.weight"] = torch.cat([t, weights[p + "k_proj.weight"], weights[p + "v_proj.weight"]])
        elif name.endswith("mlp.gate_proj.weight"):
            p = name[: -len("gate_proj.weight")]
            out[p + "gate_up_proj.weight"] = torch.cat([t, weights[p + "up_proj.weight"]])
        else:
            out[name] = t
    return out


class Phi3Oracle(MistralOracle):
    """MistralOracle (window None: full attention) with the LongRoPE table of `regime` when the config has factors"""

    def __init__(self, cfg: Phi3Config, weights: dict[str, torch.Tensor], regime: str | None = None, **kw):
        super().__init__(cfg, weights, **kw)
        if cfg.long_factor:
            self.cos_sin = longrope_table(cfg, regime or engine_regime(cfg, cfg.max_model_len),
                                          dtype=self.dtype).to(self.device)
