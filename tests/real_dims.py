"""The real-dimension presets and the map from a ModelConfig to its family's oracle.

tests/test_real_dims_gpu.py runs every preset of REAL_DIMS as a two-layer stack against the oracle that `family` picks;
tests/test_real_dims_cpu.py checks that every real preset is either in REAL_DIMS or accounted for below, and that
`family` carries every field that changes the numbers."""
from __future__ import annotations

import dataclasses
from typing import Callable

# Order matters: the GPU tests that run on a subset take a prefix of this list (WINDOW_CROSSED, then FUSED_ROPE), so
# that pytest keeps one preset's module-scoped stack for all of its checks (its grouping follows parameter indices).
REAL_DIMS = [
    # 128-dim heads, no qkv bias, no q/k norm, and a qkv projection of at most 66 weight tiles of 128 rows (half of an
    # H100's 132 SMs, so that decode steps cut every tile over several CTAs): the fused RoPE + KV-scatter epilogue runs
    "mistral-7b-v0.1", "llama3.1-8b", "granite-3-8b", "mistral-7b-v0.3", "mistral-nemo-12b", "phi3-medium-4k", "phi-4",
    # the rest; llama3-70b's qkv projection is 80 tiles, so its decode steps take rope_kvwrite
    "llama3-70b", "llama3.2-1b", "qwen3-0.6b", "qwen3-8b", "qwen2.5-0.5b", "qwen2.5-1.5b", "qwen2.5-7b", "qwen2.5-14b",
    "phi3-mini-4k", "starcoderbase-1b", "starcoder-15b",
]
WINDOW_CROSSED = REAL_DIMS[:1]
FUSED_ROPE = REAL_DIMS[:7]

# real presets checked against an oracle by another test
COVERED_ELSEWHERE = {
    "llama3-8b": "tests/test_parity_gpu.py (the 8b2l stack against the oracle and vLLM's outputs)",
    "opt-125m": "tests/test_zz_opt_gpu.py (opt-125m-2l against the oracle, opt-125m against vLLM's outputs)",
}
# real presets whose two-layer stack is another preset's, field for field
SAME_TWO_LAYER_STACK = {"granite-20b-code": "starcoder-15b", "granite-34b-code": "starcoder-15b"}

TEST_SIZED = ("tiny", "small", "125m")


def is_test_sized(name: str) -> bool:
    return name in TEST_SIZED or "-tiny" in name


def two_layer(name: str):
    from vllm_tgis_adapter_b200.engine.core import PRESETS

    return dataclasses.replace(PRESETS[name], n_layers=2)


@dataclasses.dataclass
class Family:
    name: str
    cfg: object                       # the oracle's config
    oracle: type                      # its oracle class: oracle(cfg, weights, device=...)
    synthetic_weights: Callable       # synthetic_weights(cfg, seed=...) under the names the engine loads


def family(mc) -> Family:
    """The oracle of `mc`'s family with `mc`'s dims and every field that changes the numbers.  A ModelConfig that
    combines features no single oracle restates is refused, not approximated."""
    common = dict(n_layers=mc.n_layers, hidden=mc.hidden, n_q_heads=mc.n_q_heads, n_kv_heads=mc.n_kv_heads, ffn=mc.ffn,
                  vocab=mc.vocab, head_dim=mc.head_dim, rope_theta=mc.rope_theta, rms_eps=mc.rms_eps,
                  max_model_len=mc.max_model_len)
    features = {k for k, on in (("granite", mc.is_granite), ("qk_norm", mc.qk_norm), ("qkv_bias", mc.qkv_bias),
                                ("window", mc.sliding_window is not None), ("phi3", mc.fused_projections),
                                ("longrope", mc.rope_longrope),
                                ("llama3", mc.rope_scaling_factor not in (0.0, 1.0))) if on}

    def only(*allowed):
        if features - set(allowed):
            raise ValueError(f"no oracle restates {sorted(features)} together")

    if mc.arch == "gpt_bigcode":
        from gpt_bigcode_oracle import GPTBigCodeConfig, GPTBigCodeOracle, synthetic_weights

        only()
        if not mc.tie_word_embeddings or mc.hidden != mc.n_q_heads * mc.head_dim:
            raise ValueError("the GPTBigCode oracle's synthetic weights are tied, with hidden = heads x head_dim")
        cfg = GPTBigCodeConfig(n_layers=mc.n_layers, hidden=mc.hidden, n_heads=mc.n_q_heads, n_kv_heads=mc.n_kv_heads,
                               ffn=mc.ffn, vocab=mc.vocab, ln_eps=mc.rms_eps, max_model_len=mc.max_model_len)
        return Family("gpt_bigcode", cfg, GPTBigCodeOracle, synthetic_weights)
    if mc.arch != "llama":
        raise ValueError(f"no real-dimension oracle map for arch {mc.arch!r}")
    if mc.is_granite:
        from granite_oracle import GraniteConfig, GraniteOracle, synthetic_weights

        only("granite")
        cfg = GraniteConfig(**common, embedding_multiplier=mc.embedding_multiplier,
                            residual_multiplier=mc.residual_multiplier, attention_multiplier=mc.attention_multiplier,
                            logits_scaling=mc.logits_scaling, tie_word_embeddings=mc.tie_word_embeddings)
        return Family("granite", cfg, GraniteOracle, synthetic_weights)
    if mc.qk_norm:
        from qwen3_oracle import Qwen3Config, Qwen3Oracle, synthetic_weights

        only("qk_norm")
        return Family("qwen3", Qwen3Config(**common, tie_word_embeddings=mc.tie_word_embeddings), Qwen3Oracle,
                      synthetic_weights)
    if mc.qkv_bias:
        from qwen2_oracle import Qwen2Config, Qwen2Oracle, synthetic_weights

        only("qkv_bias")
        return Family("qwen2", Qwen2Config(**common, tie_word_embeddings=mc.tie_word_embeddings), Qwen2Oracle,
                      synthetic_weights)
    if mc.fused_projections or mc.rope_longrope:
        from phi3_oracle import Phi3Config, Phi3Oracle, synthetic_weights

        only("phi3", "longrope", "window")
        longrope = dict(long_factor=tuple(mc.rope_long_factor), short_factor=tuple(mc.rope_short_factor),
                        original_max_pos=mc.rope_original_max_pos,
                        max_position_embeddings=mc.rope_max_position_embeddings) if mc.rope_longrope else {}
        cfg = Phi3Config(**common, tie_word_embeddings=mc.tie_word_embeddings, sliding_window=mc.sliding_window,
                         **longrope)
        return Family("phi3", cfg, Phi3Oracle, synthetic_weights)
    if "llama3" in features:
        from llama3_oracle import Llama3Config, Llama3Oracle, synthetic_weights

        only("llama3")
        cfg = Llama3Config(**common, rope_factor=mc.rope_scaling_factor, rope_low_freq_factor=mc.rope_low_freq_factor,
                           rope_high_freq_factor=mc.rope_high_freq_factor,
                           rope_original_max_pos=mc.rope_original_max_pos, tie_word_embeddings=mc.tie_word_embeddings)
        return Family("llama3", cfg, Llama3Oracle, synthetic_weights)
    if mc.sliding_window is not None:
        from mistral_oracle import MistralConfig, MistralOracle, synthetic_weights

        only("window")
        cfg = MistralConfig(**common, tie_word_embeddings=mc.tie_word_embeddings, sliding_window=mc.sliding_window)
        return Family("mistral", cfg, MistralOracle, synthetic_weights)
    from oracle.llama_oracle import LlamaConfig, LlamaOracle, synthetic_weights

    only()
    if mc.tie_word_embeddings:
        raise ValueError("oracle/llama_oracle.py's synthetic weights carry an lm_head: untied only")
    return Family("llama", LlamaConfig(**common), LlamaOracle, synthetic_weights)
