"""Mistral oracle for the tests: oracle/llama_oracle.py's Llama restatement plus the sliding-window mask.

Mistral (transformers MistralForCausalLM; vllm model_executor/models/mistral.py) is the Llama stack with one window in
every layer: the query at position p attends to the keys at positions p - W < k <= p, W keys including itself
(transformers masking_utils.sliding_window_overlay: kv_idx > q_idx - sliding_window).  The window is integer logic: it
changes which scores take part in the softmax and nothing about how any value is rounded.  sliding_window None is the
plain causal mask.

The oracle is pinned to transformers' MistralForCausalLM by tests/golden/mistral_hf_*.json
(scripts/gen_mistral_golden.py).
"""
from __future__ import annotations

import dataclasses
import math

import torch

from oracle.llama_oracle import LlamaConfig, LlamaOracle, synthetic_weights as llama_synthetic_weights


@dataclasses.dataclass
class MistralConfig(LlamaConfig):
    tie_word_embeddings: bool = False
    sliding_window: int | None = None


# vllm_tgis_adapter_b200/engine/core.py PRESETS["mistral-tiny"]: q width 4 x 128 = 512 != hidden 256, GQA group 4, odd
# vocabulary, a window shorter than the test prompts and not a multiple of the 32-token KV block
CONFIGS = {
    "mistral-tiny": MistralConfig(n_layers=2, hidden=256, n_q_heads=4, n_kv_heads=1, ffn=512, vocab=1021,
                                  rope_theta=10000.0, rms_eps=1e-5, max_model_len=2048, sliding_window=40),
}


def synthetic_weights(cfg: MistralConfig, seed: int = 0, dtype: torch.dtype = torch.bfloat16, **kw
                      ) -> dict[str, torch.Tensor]:
    """llama_oracle.synthetic_weights, without lm_head.weight when the embeddings are tied"""
    w = llama_synthetic_weights(cfg, seed=seed, dtype=dtype, **kw)
    if cfg.tie_word_embeddings:
        del w["lm_head.weight"]
    return w


class MistralOracle(LlamaOracle):
    """LlamaOracle with the sliding-window mask in every layer's attention (window None: LlamaOracle itself)"""

    def __init__(self, cfg: MistralConfig, weights: dict[str, torch.Tensor], window: int | None = -1, **kw):
        super().__init__(cfg, weights, **kw)
        self.window = cfg.sliding_window if window == -1 else window

    def _attend(self, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, first_pos: int) -> torch.Tensor:
        if not self.window:
            return super()._attend(q, k, v, first_pos)
        # LlamaOracle._attend with the window beside the causal test
        cfg = self.cfg
        g = cfg.n_q_heads // cfg.n_kv_heads
        kf = k.float().repeat_interleave(g, dim=1)
        vf = v.float().repeat_interleave(g, dim=1)
        s = torch.einsum("qhd,khd->hqk", q.float(), kf) * (1.0 / math.sqrt(cfg.head_dim))
        tq, tk = q.shape[0], k.shape[0]
        qpos = first_pos + torch.arange(tq, device=q.device)[:, None]
        kpos = torch.arange(tk, device=q.device)[None, :]
        mask = (kpos <= qpos) & (kpos > qpos - self.window)
        s = s.masked_fill(~mask[None], float("-inf"))
        p = torch.softmax(s, dim=-1)
        o = torch.einsum("hqk,khd->qhd", p, vf)
        return o.to(self.dtype)
