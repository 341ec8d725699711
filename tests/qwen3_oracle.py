"""Qwen3 oracle for the tests: oracle/llama_oracle.py's Llama restatement plus Qwen3's per-head RMSNorm of q and k.

Qwen3 (transformers Qwen3Attention; vllm model_executor/models/qwen3.py Qwen3Attention.forward) normalises each q head
and each k head over its head_dim after the qkv projection (LoRA deltas included) and before RoPE, with the model's
rms_norm_eps and the rounding points of every other RMSNorm in the stack: the fp32 mean of squares, x * rsqrt(...) rounded
to the model dtype, then a model-dtype multiply by the weight (q_norm / k_norm, [head_dim]).  V is not normalised.
Everything else is the Llama stack with tied or untied embeddings.

The oracle is pinned to transformers' Qwen3ForCausalLM by tests/golden/qwen3_hf_*.json (scripts/gen_qwen3_golden.py).
"""
from __future__ import annotations

import dataclasses

import torch

from oracle.llama_oracle import LlamaConfig, LlamaOracle, synthetic_weights as llama_synthetic_weights


@dataclasses.dataclass
class Qwen3Config(LlamaConfig):
    tie_word_embeddings: bool = False


# vllm_tgis_adapter_b200/engine/core.py PRESETS["qwen3-tiny"]: q width 4 x 128 = 512 != hidden 256, odd vocabulary
CONFIGS = {
    "qwen3-tiny": Qwen3Config(n_layers=2, hidden=256, n_q_heads=4, n_kv_heads=2, ffn=512, vocab=1021,
                              rope_theta=1000000.0, rms_eps=1e-6, max_model_len=2048, tie_word_embeddings=True),
}


def synthetic_weights(cfg: Qwen3Config, seed: int = 0, dtype: torch.dtype = torch.bfloat16, **kw
                      ) -> dict[str, torch.Tensor]:
    """llama_oracle.synthetic_weights plus q_norm / k_norm per layer, drawn from [0.25, 2.5) -- well away from 1, so the
    weight multiply and its rounding matter -- and without lm_head.weight when the embeddings are tied"""
    w = llama_synthetic_weights(cfg, seed=seed, dtype=dtype, **kw)
    g = torch.Generator().manual_seed(seed + 7919)
    device = w["model.embed_tokens.weight"].device
    for i in range(cfg.n_layers):
        for name in ("q_norm", "k_norm"):
            v = 0.25 + 2.25 * torch.rand(cfg.head_dim, generator=g, dtype=torch.float32)
            w[f"model.layers.{i}.self_attn.{name}.weight"] = v.to(device=device, dtype=dtype)
    if cfg.tie_word_embeddings:
        del w["lm_head.weight"]
    return w


class Qwen3Oracle(LlamaOracle):
    """LlamaOracle.step rotates q and then k of layer 0, 1, ... through `_rope`; this subclass counts those calls within
    a step to know which layer and which projection it is given, and normalises each head before the rotation."""

    def __init__(self, cfg: Qwen3Config, weights: dict[str, torch.Tensor], **kw):
        super().__init__(cfg, weights, **kw)   # (tied: self.lm_head is the embedding table)
        self.head_norms = [
            tuple(weights[f"model.layers.{i}.self_attn.{n}_norm.weight"].to(device=self.device, dtype=self.dtype)
                  for n in ("q", "k")) for i in range(cfg.n_layers)]
        self._rope_calls = 0

    def head_norm(self, x: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
        """x [T, heads, head_dim] in the model dtype: Qwen3RMSNorm over each head"""
        return self._rms(x, w)

    def _rope(self, x: torch.Tensor, pos: torch.Tensor) -> torch.Tensor:
        layer, which = divmod(self._rope_calls, 2)
        self._rope_calls += 1
        return super()._rope(self.head_norm(x, self.head_norms[layer][which]), pos)

    def step(self, *args, **kw) -> torch.Tensor:
        self._rope_calls = 0
        out = super().step(*args, **kw)
        assert self._rope_calls == 2 * self.cfg.n_layers
        return out
