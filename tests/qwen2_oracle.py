"""Qwen2 oracle for the tests: oracle/llama_oracle.py's Llama restatement with Qwen2's bias on the q, k and v projections.

Qwen2 (transformers Qwen2Attention; vllm model_executor/models/qwen2.py Qwen2Attention, QKVParallelLinear(bias=True)) is
the Llama stack with a bias on qkv_proj and nowhere else.  vLLM runs F.linear(x, W, b) in the model dtype, which adds the
bias to the fp32 accumulator and rounds once: qkv = bf16(x . W^T + b).  LoRA deltas land on that biased output (vllm
MergedQKVParallelLinearWithLoRA), then RoPE runs.  Everything else is the Llama stack with tied or untied embeddings.

The oracle is pinned to transformers' Qwen2ForCausalLM by tests/golden/qwen2_hf_*.json (scripts/gen_qwen2_golden.py).
"""
from __future__ import annotations

import dataclasses

import torch
import torch.nn.functional as F

import oracle.llama_oracle as llama_oracle
from oracle.llama_oracle import LlamaConfig, LlamaOracle, synthetic_weights as llama_synthetic_weights


@dataclasses.dataclass
class Qwen2Config(LlamaConfig):
    tie_word_embeddings: bool = False


# vllm_tgis_adapter_b200/engine/core.py PRESETS["qwen2-tiny"] (GQA group 6, 128-dim heads, q width 768 = hidden) and
# ["qwen2-tiny-hd64"] (group 7, 64-dim heads, q width 448 = hidden); both with an odd vocabulary and tied embeddings
CONFIGS = {
    "qwen2-tiny": Qwen2Config(n_layers=2, hidden=768, n_q_heads=6, n_kv_heads=1, ffn=1024, vocab=1021,
                              rope_theta=1000000.0, rms_eps=1e-6, max_model_len=2048, tie_word_embeddings=True),
    "qwen2-tiny-hd64": Qwen2Config(n_layers=2, hidden=448, n_q_heads=7, n_kv_heads=1, ffn=512, vocab=1021, head_dim=64,
                                   rope_theta=1000000.0, rms_eps=1e-6, max_model_len=2048, tie_word_embeddings=True),
}

BIAS_NAMES = ("q_proj", "k_proj", "v_proj")


def synthetic_weights(cfg: Qwen2Config, seed: int = 0, dtype: torch.dtype = torch.bfloat16, **kw
                      ) -> dict[str, torch.Tensor]:
    """llama_oracle.synthetic_weights plus q / k / v biases per layer, without lm_head.weight when the embeddings are tied.

    The projections are about 0.02 * sqrt(hidden) * |x| ~ 0.5 wide; the biases are N(0, 0.5) for q and v, and k's are
    N(0, 2) with every 16th entry at +-24 -- far above the projection's scale, as the k biases of the published Qwen2.5
    checkpoints are -- so that where the one rounding after the bias add sits shows in the logits."""
    w = llama_synthetic_weights(cfg, seed=seed, dtype=dtype, **kw)
    g = torch.Generator().manual_seed(seed + 104729)
    device = w["model.embed_tokens.weight"].device
    for i in range(cfg.n_layers):
        for name, n in zip(BIAS_NAMES, (cfg.q_dim, cfg.kv_dim, cfg.kv_dim)):
            b = torch.randn(n, generator=g, dtype=torch.float32) * (2.0 if name == "k_proj" else 0.5)
            if name == "k_proj":
                b[::16] = 24.0 * torch.sign(torch.randn(len(b[::16]), generator=g))
            w[f"model.layers.{i}.self_attn.{name}.bias"] = b.to(device=device, dtype=dtype)
    if cfg.tie_word_embeddings:
        del w["lm_head.weight"]
    return w


class _BiasedLinear:
    """Stands in for torch.nn.functional inside llama_oracle during a Qwen2 step: F.linear of a layer's fused qkv weight
    becomes bf16(x . W^T + b) -- the product and the bias add in fp32, one rounding to the model dtype; every other
    function is torch's."""

    def __init__(self, biases: dict[int, torch.Tensor]):
        self.biases = biases

    def linear(self, x, w, b=None):
        bias = self.biases.get(id(w))
        if bias is None:
            return F.linear(x, w, b)
        return (F.linear(x.float(), w.float()) + bias.float()).to(x.dtype)

    def __getattr__(self, name):
        return getattr(F, name)


class Qwen2Oracle(LlamaOracle):
    """LlamaOracle with the qkv bias: the qkv projection of each layer goes through _BiasedLinear."""

    def __init__(self, cfg: Qwen2Config, weights: dict[str, torch.Tensor], **kw):
        super().__init__(cfg, weights, **kw)   # (tied: self.lm_head is the embedding table)
        self.qkv_bias = [
            torch.cat([weights[f"model.layers.{i}.self_attn.{n}.bias"] for n in BIAS_NAMES]).to(
                device=self.device, dtype=self.dtype) for i in range(cfg.n_layers)]
        self._shim = _BiasedLinear({id(L["qkv"]): b for L, b in zip(self.layers, self.qkv_bias)})

    def step(self, *args, **kw) -> torch.Tensor:
        saved = llama_oracle.F
        llama_oracle.F = self._shim
        try:
            return super().step(*args, **kw)
        finally:
            llama_oracle.F = saved
