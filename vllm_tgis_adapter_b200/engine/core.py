"""Thin object wrapper over the C ABI (include/tgis_engine.h).  No arithmetic happens in Python."""
from __future__ import annotations

import ctypes as C
import dataclasses
from typing import Iterable

from . import _lib
from ._lib import TgisConfig, TgisSamplingParams, TgisStatus, TgisStepOutput


class EngineError(RuntimeError):
    pass


@dataclasses.dataclass
class ModelConfig:
    """Decoder dims (HF config.json names in comments).  arch "llama": RMSNorm / RoPE / GQA / SwiGLU; arch "opt": learned
    positions / LayerNorm / biased projections / ReLU (n_kv_heads == n_q_heads, head_dim 64 or 128, ffn = ffn_dim,
    rms_eps carries the LayerNorm epsilon, rope_theta unused) -- include/tgis_engine.h TGIS_ARCH_*.

    Granite (GraniteForCausalLM) is arch "llama" with the four scalars of its config.json set; their defaults are the
    Llama stack (tgis_engine_set_model_scalars).

    arch "llama" takes head_dim 128 or 64 (Llama-3.2-1B; single GPU, no LoRA slots, no Granite scalars), and the
    rope_type "llama3" frequency scaling of Llama-3.1 / 3.2 (rope_scaling_factor > 1; loader.rope_cos_sin).

    Qwen3 (Qwen3ForCausalLM) is arch "llama" with qk_norm set: an RMSNorm over each q and k head before RoPE, with the
    per-layer weights self_attn.q_norm / k_norm (tgis_engine_set_qk_norm; head_dim 128, single GPU).

    Mistral (MistralForCausalLM) is arch "llama" with sliding_window set: every layer's query at position p attends to
    the keys p - sliding_window < k <= p (tgis_engine_set_sliding_window; single GPU).

    Qwen2 / Qwen2.5 (Qwen2ForCausalLM) is arch "llama" with qkv_bias set: a bias on the q, k and v projections, added to
    the fp32 accumulators before the one rounding to bf16 (tgis_engine_set_qkv_bias; head_dim 128 or 64, single GPU).

    Phi-3 / Phi-3.5 / Phi-4 (Phi3ForCausalLM) is arch "llama", with head_dim 96 for Phi-3-mini / Phi-3.5-mini (single
    GPU, no LoRA slots), LongRoPE for the 128k variants (rope_long_factor / rope_short_factor) and the model-wide
    sliding_window of the 4k variants.  Its fused qkv_proj / gate_up_proj tensors are split on the host (loader.py).

    GPTBigCode (GPTBigCodeForCausalLM: StarCoder, SantaCoder, Granite-20B/34B-Code) is arch "gpt_bigcode": OPT's layer
    stack with positions from 0, GELU-tanh, head_dim 128 and n_kv_heads 1 (multi_query, up to 64 query heads) or n_q_heads
    (single GPU, no LoRA slots)."""

    n_layers: int        # num_hidden_layers
    hidden: int          # hidden_size
    n_q_heads: int       # num_attention_heads
    n_kv_heads: int      # num_key_value_heads
    ffn: int             # intermediate_size
    vocab: int           # vocab_size
    head_dim: int = 128
    rope_theta: float = 500000.0
    rms_eps: float = 1e-5
    max_model_len: int = 2048
    arch: str = "llama"
    tie_word_embeddings: bool = False   # no lm_head.weight: the engine copies embed_tokens
    embedding_multiplier: float = 1.0   # Granite: h = bf16(embed * m)
    residual_multiplier: float = 1.0    # Granite: r = bf16(r + bf16(x * m)) after o_proj and down_proj
    attention_multiplier: float = 0.0   # Granite: softmax scale; 0 = 1/sqrt(head_dim)
    logits_scaling: float = 1.0         # Granite: logits = bf16(logits * (1 / logits_scaling))
    rope_scaling_factor: float = 0.0    # rope_scaling / rope_parameters of rope_type "llama3": factor (0 or 1 = unscaled)
    rope_low_freq_factor: float = 1.0   # low_freq_factor
    rope_high_freq_factor: float = 4.0  # high_freq_factor
    rope_original_max_pos: int = 8192   # original_max_position_embeddings
    qk_norm: bool = False               # Qwen3: per-head RMSNorm of q and k (self_attn.q_norm / k_norm)
    sliding_window: int | None = None   # Mistral: keys per query, itself included, in every layer; None = all
    qkv_bias: bool = False              # Qwen2: self_attn.{q,k,v}_proj.bias
    # LongRoPE (Phi-3 128k, rope_type "longrope"): per-frequency rescale factors [head_dim / 2], long and short, with
    # rope_original_max_pos as original_max_position_embeddings; empty = no LongRoPE (rope.py)
    rope_long_factor: tuple[float, ...] = ()
    rope_short_factor: tuple[float, ...] = ()
    rope_max_position_embeddings: int = 0   # LongRoPE: max_position_embeddings (the mscale's numerator)
    fused_projections: bool = False     # Phi-3: checkpoints hold self_attn.qkv_proj and mlp.gate_up_proj (loader.py)

    @property
    def rope_longrope(self) -> bool:
        return bool(self.rope_long_factor)

    @property
    def rope_scaled(self) -> bool:
        """the rotary table is not the engine's built-in unscaled one (llama3 scaling or LongRoPE)"""
        return self.rope_scaling_factor not in (0.0, 1.0) or self.rope_longrope

    @property
    def is_granite(self) -> bool:
        return (self.embedding_multiplier, self.residual_multiplier, self.attention_multiplier,
                self.logits_scaling) != (1.0, 1.0, 0.0, 1.0)


# Named architectures (real dims; this offline build runs them on synthetic weights — SURVEY.md §0)
PRESETS: dict[str, ModelConfig] = {
    "tiny": ModelConfig(n_layers=2, hidden=256, n_q_heads=4, n_kv_heads=2, ffn=512, vocab=1024, max_model_len=512),
    "small": ModelConfig(n_layers=4, hidden=512, n_q_heads=4, n_kv_heads=1, ffn=1536, vocab=4096, max_model_len=1024),
    "125m": ModelConfig(n_layers=12, hidden=768, n_q_heads=6, n_kv_heads=2, ffn=3072, vocab=50272, max_model_len=2048),
    # facebook/opt-125m (the reference's own test model; BASELINE configs[0]) and a CPU-oracle-sized sibling
    "opt-125m": ModelConfig(n_layers=12, hidden=768, n_q_heads=12, n_kv_heads=12, ffn=3072, vocab=50272, head_dim=64,
                            max_model_len=2048, arch="opt"),
    "opt-tiny": ModelConfig(n_layers=2, hidden=256, n_q_heads=4, n_kv_heads=4, ffn=1024, vocab=1024, head_dim=64,
                            max_model_len=512, arch="opt"),
    "llama3-8b": ModelConfig(n_layers=32, hidden=4096, n_q_heads=32, n_kv_heads=8, ffn=14336, vocab=128256,
                             max_model_len=8192),
    "llama3-70b": ModelConfig(n_layers=80, hidden=8192, n_q_heads=64, n_kv_heads=8, ffn=28672, vocab=128256,
                              max_model_len=8192),
    # Llama-3.1 / 3.2: rope_type "llama3" frequency scaling; 3.2-1B has 64-dim heads and tied embeddings
    "llama3.1-8b": ModelConfig(n_layers=32, hidden=4096, n_q_heads=32, n_kv_heads=8, ffn=14336, vocab=128256,
                               max_model_len=8192, rope_scaling_factor=8.0, rope_low_freq_factor=1.0,
                               rope_high_freq_factor=4.0, rope_original_max_pos=8192),
    "llama3.2-1b": ModelConfig(n_layers=16, hidden=2048, n_q_heads=32, n_kv_heads=8, ffn=8192, vocab=128256, head_dim=64,
                               max_model_len=8192, tie_word_embeddings=True, rope_scaling_factor=32.0,
                               rope_low_freq_factor=1.0, rope_high_freq_factor=4.0, rope_original_max_pos=8192),
    # CPU-oracle-sized 64-dim-head stack; original_max_position_embeddings 64 puts its 32 rotary frequencies into all
    # three bands of the llama3 rule and lets short prompts run past it
    "llama-tiny-hd64": ModelConfig(n_layers=2, hidden=256, n_q_heads=4, n_kv_heads=2, ffn=512, vocab=1024, head_dim=64,
                                   rope_theta=10000.0, max_model_len=2048, tie_word_embeddings=True,
                                   rope_scaling_factor=8.0, rope_low_freq_factor=1.0, rope_high_freq_factor=4.0,
                                   rope_original_max_pos=64),
    # Granite: a CPU-oracle-sized stack with an odd vocabulary and scalars that round (1/3 is not a power of two), and
    # the Granite 3.x 8B shape.  The granite-3-8b values are those of the published ibm-granite/granite-3.1-8b config.json
    # as recalled; they could not be checked against the file when this preset was written.
    "granite-tiny": ModelConfig(n_layers=2, hidden=256, n_q_heads=4, n_kv_heads=2, ffn=512, vocab=1021,
                                max_model_len=512, tie_word_embeddings=True, embedding_multiplier=12.0,
                                residual_multiplier=0.22, attention_multiplier=1.0 / 128, logits_scaling=3.0),
    "granite-3-8b": ModelConfig(n_layers=40, hidden=4096, n_q_heads=32, n_kv_heads=8, ffn=12800, vocab=49155,
                                rope_theta=10000000.0, max_model_len=8192, tie_word_embeddings=True,
                                embedding_multiplier=12.0, residual_multiplier=0.22, attention_multiplier=0.0078125,
                                logits_scaling=16.0),
    # Qwen3: a CPU-oracle-sized stack whose q width (4 x 128) is not its hidden size, with an odd vocabulary, and the
    # Qwen3-0.6B and Qwen3-8B shapes.  The qwen3-0.6b / qwen3-8b values are those of the published Qwen/Qwen3-0.6B and
    # Qwen/Qwen3-8B config.json files as recalled; they could not be checked against the files when these presets were
    # written.
    "qwen3-tiny": ModelConfig(n_layers=2, hidden=256, n_q_heads=4, n_kv_heads=2, ffn=512, vocab=1021,
                              rope_theta=1000000.0, rms_eps=1e-6, max_model_len=2048, tie_word_embeddings=True,
                              qk_norm=True),
    "qwen3-0.6b": ModelConfig(n_layers=28, hidden=1024, n_q_heads=16, n_kv_heads=8, ffn=3072, vocab=151936,
                              rope_theta=1000000.0, rms_eps=1e-6, max_model_len=8192, tie_word_embeddings=True,
                              qk_norm=True),
    "qwen3-8b": ModelConfig(n_layers=36, hidden=4096, n_q_heads=32, n_kv_heads=8, ffn=12288, vocab=151936,
                            rope_theta=1000000.0, rms_eps=1e-6, max_model_len=8192, qk_norm=True),
    # Mistral: a CPU-oracle-sized stack whose q width (4 x 128) is not its hidden size, with an odd vocabulary and a
    # window of 40 (shorter than the test prompts, not a multiple of the 32-token KV block), and the Mistral-7B v0.1 /
    # v0.3 and Mistral-Nemo-12B shapes.  Those three are the published mistralai config.json values as recalled, not
    # checked against the files when these presets were written.
    "mistral-tiny": ModelConfig(n_layers=2, hidden=256, n_q_heads=4, n_kv_heads=1, ffn=512, vocab=1021,
                                rope_theta=10000.0, rms_eps=1e-5, max_model_len=2048, sliding_window=40),
    "mistral-7b-v0.1": ModelConfig(n_layers=32, hidden=4096, n_q_heads=32, n_kv_heads=8, ffn=14336, vocab=32000,
                                   rope_theta=10000.0, rms_eps=1e-5, max_model_len=8192, sliding_window=4096),
    "mistral-7b-v0.3": ModelConfig(n_layers=32, hidden=4096, n_q_heads=32, n_kv_heads=8, ffn=14336, vocab=32768,
                                   rope_theta=1000000.0, rms_eps=1e-5, max_model_len=8192),
    "mistral-nemo-12b": ModelConfig(n_layers=40, hidden=5120, n_q_heads=32, n_kv_heads=8, ffn=14336, vocab=131072,
                                    rope_theta=1000000.0, rms_eps=1e-5, max_model_len=8192),
    # Qwen2 / Qwen2.5: two CPU-oracle-sized stacks with GQA groups of 6 (128-dim heads) and 7 (64-dim heads), q widths
    # that are not their hidden sizes and an odd vocabulary, and the Qwen2.5 0.5B, 1.5B, 7B and 14B shapes.  Those four are
    # the published Qwen/Qwen2.5-* config.json values as recalled, not checked against the files when these presets were
    # written.
    "qwen2-tiny": ModelConfig(n_layers=2, hidden=768, n_q_heads=6, n_kv_heads=1, ffn=1024, vocab=1021,
                              rope_theta=1000000.0, rms_eps=1e-6, max_model_len=2048, tie_word_embeddings=True,
                              qkv_bias=True),
    "qwen2-tiny-hd64": ModelConfig(n_layers=2, hidden=448, n_q_heads=7, n_kv_heads=1, ffn=512, vocab=1021, head_dim=64,
                                   rope_theta=1000000.0, rms_eps=1e-6, max_model_len=2048, tie_word_embeddings=True,
                                   qkv_bias=True),
    "qwen2.5-0.5b": ModelConfig(n_layers=24, hidden=896, n_q_heads=14, n_kv_heads=2, ffn=4864, vocab=151936, head_dim=64,
                                rope_theta=1000000.0, rms_eps=1e-6, max_model_len=8192, tie_word_embeddings=True,
                                qkv_bias=True),
    "qwen2.5-1.5b": ModelConfig(n_layers=28, hidden=1536, n_q_heads=12, n_kv_heads=2, ffn=8960, vocab=151936,
                                rope_theta=1000000.0, rms_eps=1e-6, max_model_len=8192, tie_word_embeddings=True,
                                qkv_bias=True),
    "qwen2.5-7b": ModelConfig(n_layers=28, hidden=3584, n_q_heads=28, n_kv_heads=4, ffn=18944, vocab=152064,
                              rope_theta=1000000.0, rms_eps=1e-6, max_model_len=8192, qkv_bias=True),
    "qwen2.5-14b": ModelConfig(n_layers=48, hidden=5120, n_q_heads=40, n_kv_heads=8, ffn=13824, vocab=152064,
                               rope_theta=1000000.0, rms_eps=1e-5, max_model_len=8192, qkv_bias=True),
    # Phi-3: a CPU-oracle-sized stack with 96-dim heads, GQA group 1 and an odd vocabulary, and the
    # Phi-3-mini-4k, Phi-3-medium-4k and Phi-4 shapes.  Those three are the published microsoft/Phi-3-mini-4k-instruct,
    # Phi-3-medium-4k-instruct and phi-4 config.json values as recalled, not checked against the files when these
    # presets were written.  The 4k checkpoints' config.json sets sliding_window 2047, which the loader maps; the presets
    # leave it out (only the Mistral presets carry a window), which changes nothing below 2047 tokens.  Phi-4's
    # sliding_window is uncertain (recalled as null, i.e. none).
    "phi3-tiny": ModelConfig(n_layers=2, hidden=384, n_q_heads=4, n_kv_heads=4, ffn=512, vocab=1021, head_dim=96,
                             rope_theta=10000.0, rms_eps=1e-5, max_model_len=2048, fused_projections=True),
    "phi3-mini-4k": ModelConfig(n_layers=32, hidden=3072, n_q_heads=32, n_kv_heads=32, ffn=8192, vocab=32064,
                                head_dim=96, rope_theta=10000.0, rms_eps=1e-5, max_model_len=4096,
                                fused_projections=True),
    "phi3-medium-4k": ModelConfig(n_layers=40, hidden=5120, n_q_heads=40, n_kv_heads=10, ffn=17920, vocab=32064,
                                  rope_theta=10000.0, rms_eps=1e-5, max_model_len=4096, fused_projections=True),
    "phi-4": ModelConfig(n_layers=40, hidden=5120, n_q_heads=40, n_kv_heads=10, ffn=17920, vocab=100352,
                         rope_theta=250000.0, rms_eps=1e-5, max_model_len=16384, fused_projections=True),
    # GPTBigCode: two CPU-oracle-sized stacks, multi-query with 12 heads (a partial last head octet: 8 + 4) and multi-head,
    # with an odd vocabulary, and the StarCoderBase-1B, StarCoder-15B, Granite-20B-Code and Granite-34B-Code shapes.
    # Those four are the published bigcode/starcoderbase-1b, bigcode/starcoder, ibm-granite/granite-20b-code-base and
    # granite-34b-code-base config.json values as recalled, not checked against the files when these presets were written.
    "gpt-bigcode-tiny": ModelConfig(n_layers=2, hidden=1536, n_q_heads=12, n_kv_heads=1, ffn=2048, vocab=1021,
                                    rms_eps=1e-5, max_model_len=2048, arch="gpt_bigcode", tie_word_embeddings=True),
    "gpt-bigcode-tiny-mha": ModelConfig(n_layers=2, hidden=512, n_q_heads=4, n_kv_heads=4, ffn=1024, vocab=1021,
                                        rms_eps=1e-5, max_model_len=2048, arch="gpt_bigcode", tie_word_embeddings=True),
    "starcoderbase-1b": ModelConfig(n_layers=24, hidden=2048, n_q_heads=16, n_kv_heads=1, ffn=8192, vocab=49152,
                                    rms_eps=1e-5, max_model_len=8192, arch="gpt_bigcode", tie_word_embeddings=True),
    "starcoder-15b": ModelConfig(n_layers=40, hidden=6144, n_q_heads=48, n_kv_heads=1, ffn=24576, vocab=49152,
                                 rms_eps=1e-5, max_model_len=8192, arch="gpt_bigcode", tie_word_embeddings=True),
    "granite-20b-code": ModelConfig(n_layers=52, hidden=6144, n_q_heads=48, n_kv_heads=1, ffn=24576, vocab=49152,
                                    rms_eps=1e-5, max_model_len=8192, arch="gpt_bigcode", tie_word_embeddings=True),
    "granite-34b-code": ModelConfig(n_layers=88, hidden=6144, n_q_heads=48, n_kv_heads=1, ffn=24576, vocab=49152,
                                    rms_eps=1e-5, max_model_len=8192, arch="gpt_bigcode", tie_word_embeddings=True),
}


@dataclasses.dataclass
class StepOutput:
    request_id: str
    new_token: int | None
    logprob: float
    rank: int
    topn: list[tuple[int, float]]
    finish_reason: int
    stop_token_id: int
    n_prompt_tokens: int
    n_output_tokens: int
    ts_arrival: float
    ts_first_scheduled: float
    ts_first_token: float
    ts_last_token: float
    prompt_pos: int = -1   # >= 1: prompt-logprob record for that prompt position
    token_id: int = -1     # the token the record describes (generated token, or prompt token for prompt records)


def make_sampling_params(*, greedy: bool = True, temperature: float = 1.0, top_k: int = 0, top_p: float = 1.0,
                         typical_p: float = 0.0, repetition_penalty: float = 1.0,
                         length_penalty: tuple[int, float] | None = None, eos_token_id: int = 2, min_tokens: int = 0,
                         max_tokens: int = 16, num_logprobs: int = 0, prompt_logprobs: int = 0, seed: int | None = None,
                         stop_token_ids: Iterable[int] = (), guided: bool = False,
                         lora_slot: int = 0) -> TgisSamplingParams:
    sp = TgisSamplingParams()
    sp.greedy = 1 if greedy else 0
    sp.temperature = float(temperature)
    sp.top_k = int(top_k)
    sp.top_p = float(top_p)
    sp.typical_p = float(typical_p)
    sp.repetition_penalty = float(repetition_penalty)
    sp.has_length_penalty = 1 if length_penalty is not None else 0
    if length_penalty is not None:
        sp.lp_start_index = int(length_penalty[0])
        sp.lp_decay_factor = float(length_penalty[1])
    sp.eos_token_id = int(eos_token_id)
    sp.min_tokens = int(min_tokens)
    sp.max_tokens = int(max_tokens)
    sp.num_logprobs = int(num_logprobs)
    sp.prompt_logprobs = int(prompt_logprobs)
    sp.has_seed = 1 if seed is not None else 0
    sp.seed = int(seed or 0)
    ids = list(stop_token_ids)
    sp.n_stop_token_ids = len(ids)
    for i, t in enumerate(ids):
        sp.stop_token_ids[i] = int(t)
    sp.guided = 1 if guided else 0
    sp.lora_slot = int(lora_slot)
    return sp


class NativeEngine:
    """Owns one `tgis_engine*`."""

    def __init__(self, model: ModelConfig, *, max_num_seqs: int = 64, max_batched_tokens: int = 2048,
                 kv_cache_bytes: int = 0, gpu_mem_fraction: float = 0.85, device: int = 0, seed: int = 0,
                 debug_gemm_ref: bool = False, use_cuda_graphs: bool | None = None, tp_size: int = 1, tp_rank: int = 0,
                 nccl_id: bytes | None = None, shm_name: str = "", max_loras: int = 0, max_lora_rank: int = 16,
                 enable_prefix_caching: bool = False):
        self.lib = _lib.load_library()
        self.model = model
        if use_cuda_graphs is None:   # default on; TGIS_CUDA_GRAPHS=0 turns decode-step graph replay off
            import os

            use_cuda_graphs = os.environ.get("TGIS_CUDA_GRAPHS", "1") != "0"
        cfg = TgisConfig()
        cfg.abi_version = _lib.ABI_VERSION
        cfg.n_layers, cfg.hidden, cfg.n_q_heads, cfg.n_kv_heads = model.n_layers, model.hidden, model.n_q_heads, model.n_kv_heads
        cfg.head_dim, cfg.ffn, cfg.vocab = model.head_dim, model.ffn, model.vocab
        cfg.rope_theta, cfg.rms_eps, cfg.max_model_len = model.rope_theta, model.rms_eps, model.max_model_len
        cfg.max_num_seqs, cfg.max_batched_tokens = max_num_seqs, max_batched_tokens
        cfg.kv_cache_bytes, cfg.gpu_mem_fraction = kv_cache_bytes, gpu_mem_fraction
        cfg.device, cfg.tp_size, cfg.tp_rank = device, tp_size, tp_rank
        if tp_size > 1:
            import torch  # noqa: F401  (load torch's NCCL before the engine dlopens libnccl.so.2)

            if nccl_id is None or len(nccl_id) != 128:
                raise EngineError("tensor parallelism needs the 128-byte NCCL unique id of rank 0")
            C.memmove(cfg.nccl_id, nccl_id, 128)
            cfg.shm_name = shm_name.encode()
        cfg.use_cuda_graphs, cfg.debug_gemm_ref, cfg.seed = int(use_cuda_graphs), 1 if debug_gemm_ref else 0, seed
        cfg.max_loras, cfg.max_lora_rank = int(max_loras), int(max_lora_rank) if max_loras else 0
        if model.residual_multiplier != 1.0 and tp_size > 1:
            raise EngineError("Granite (residual_multiplier != 1) is not supported with tensor parallelism: the "
                              "row-parallel exchange kernels do not implement the multiplier (use tensor_parallel_size 1)")
        if model.qk_norm and tp_size > 1:
            raise EngineError("Qwen3 (qk_norm) is not supported with tensor parallelism: the q/k norm is implemented on a "
                              "single GPU only (use tensor_parallel_size 1)")
        if model.sliding_window and tp_size > 1:
            raise EngineError("sliding-window attention (Mistral) is not supported with tensor parallelism: it is "
                              "implemented on a single GPU only (use tensor_parallel_size 1)")
        if model.fused_projections and tp_size > 1:
            raise EngineError("Phi-3 is not supported with tensor parallelism: it is implemented on a single GPU only "
                              "(use tensor_parallel_size 1)")
        if model.qkv_bias and tp_size > 1:
            raise EngineError("Qwen2 (qkv_bias) is not supported with tensor parallelism: the qkv bias is implemented on a "
                              "single GPU only (use tensor_parallel_size 1)")
        if model.arch == "gpt_bigcode" and tp_size > 1:
            raise EngineError("GPTBigCode is not supported with tensor parallelism: it is implemented on a single GPU only "
                              "(use tensor_parallel_size 1)")
        if model.arch == "gpt_bigcode" and max_loras:
            raise EngineError("GPTBigCode is not supported with LoRA adapters (--enable-lora)")
        if model.arch not in ("llama", "opt", "gpt_bigcode"):
            raise EngineError(f"unknown architecture {model.arch!r}")
        if model.arch == "llama" and model.head_dim != 128 and model.is_granite:
            raise EngineError(f"Granite with head_dim {model.head_dim} is not supported yet (Granite needs head_dim 128)")
        cfg.arch = {"opt": _lib.ARCH_OPT, "gpt_bigcode": _lib.ARCH_GPT_BIGCODE}.get(model.arch, _lib.ARCH_LLAMA)
        self.max_loras, self.max_lora_rank = int(max_loras), int(max_lora_rank)
        self._h = C.c_void_p()
        if self.lib.tgis_engine_create(C.byref(cfg), C.byref(self._h)) != 0:
            raise EngineError(f"tgis_engine_create failed: {_lib.last_error(self.lib)}")
        if model.is_granite and self.lib.tgis_engine_set_model_scalars(
                self._h, model.embedding_multiplier, model.residual_multiplier, model.attention_multiplier,
                1.0 / model.logits_scaling) != 0:
            msg = _lib.last_error(self.lib)
            self.close()
            raise EngineError(f"tgis_engine_set_model_scalars failed: {msg}")
        if model.arch == "llama" and model.rope_scaled:
            # the engine's built-in rotary table is the unscaled one: mark the table as required (start fails without it)
            # and load the scaled one here, so that every way of building an engine gets it
            if self.lib.tgis_engine_require_rope_table(self._h) != 0:
                msg = _lib.last_error(self.lib)
                self.close()
                raise EngineError(f"tgis_engine_require_rope_table failed: {msg}")
            from .rope import rope_cos_sin

            self.load_weight("tgis.rope_cos_sin", rope_cos_sin(model))
        if model.qk_norm and self.lib.tgis_engine_set_qk_norm(self._h, 1) != 0:
            msg = _lib.last_error(self.lib)
            self.close()
            raise EngineError(f"tgis_engine_set_qk_norm failed: {msg}")
        if model.qkv_bias and self.lib.tgis_engine_set_qkv_bias(self._h, 1) != 0:
            msg = _lib.last_error(self.lib)
            self.close()
            raise EngineError(f"tgis_engine_set_qkv_bias failed: {msg}")
        if model.sliding_window and self.lib.tgis_engine_set_sliding_window(self._h, int(model.sliding_window)) != 0:
            msg = _lib.last_error(self.lib)
            self.close()
            raise EngineError(f"tgis_engine_set_sliding_window failed: {msg}")
        self.enable_prefix_caching = bool(enable_prefix_caching)
        if self.enable_prefix_caching and self.lib.tgis_engine_set_prefix_caching(self._h, 1) != 0:
            msg = _lib.last_error(self.lib)
            self.close()
            raise EngineError(f"tgis_engine_set_prefix_caching failed: {msg}")
        self._poll_buf = (TgisStepOutput * 512)()

    # -- weights ------------------------------------------------------------------------------------------------
    def load_weight(self, name: str, tensor) -> None:
        """tensor: contiguous torch bf16 tensor (host or device) — "PyTorch tensors for weights only"."""
        import torch

        t = tensor.detach()
        if t.dtype != torch.bfloat16:
            t = t.to(torch.bfloat16)
        t = t.contiguous()
        rows = t.shape[0]
        cols = t.numel() // rows if rows else 0
        if self.lib.tgis_engine_load_weight(self._h, name.encode(), C.c_void_p(t.data_ptr()), rows, cols, 0) != 0:
            raise EngineError(f"load_weight({name}) failed: {_lib.last_error(self.lib)}")

    def load_weights(self, weights: dict) -> None:
        for k, v in weights.items():
            self.load_weight(k, v)

    # -- control ------------------------------------------------------------------------------------------------
    def start(self) -> None:
        if self.lib.tgis_engine_start(self._h) != 0:
            raise EngineError(_lib.last_error(self.lib))

    def add_request(self, request_id: str, prompt_ids: list[int], params: TgisSamplingParams) -> None:
        arr = (C.c_int32 * len(prompt_ids))(*prompt_ids)
        if self.lib.tgis_engine_add_request(self._h, request_id.encode(), arr, len(prompt_ids), C.byref(params)) != 0:
            raise EngineError(f"add_request failed: {_lib.last_error(self.lib)}")

    def abort(self, request_id: str) -> None:
        self.lib.tgis_engine_abort(self._h, request_id.encode())

    def load_adapter(self, slot: int, weights: dict) -> None:
        """weights: {(layer, module): (A [r, in] bf16, B_scaled [out, r] bf16)} as engine/lora.py `read_adapter` returns
        them.  The slot is zeroed first (modules the adapter does not target contribute nothing)."""
        import torch

        if self.lib.tgis_engine_clear_adapter(self._h, slot) != 0:
            raise EngineError(f"clear_adapter({slot}) failed: {_lib.last_error(self.lib)}")
        for (layer, module), (a, b) in weights.items():
            for which, t in (("lora_A", a), ("lora_B", b)):
                t = t.detach().to(torch.bfloat16).contiguous()
                name = f"layers.{layer}.{module}.{which}".encode()
                if self.lib.tgis_engine_load_adapter_weight(self._h, slot, name, C.c_void_p(t.data_ptr()), t.shape[0],
                                                            t.shape[1]) != 0:
                    raise EngineError(f"load_adapter_weight({name.decode()}) failed: {_lib.last_error(self.lib)}")

    def set_mask_provider(self, callback) -> None:
        """callback: a `guided.MASK_FN` C function pointer (the caller keeps it alive), or None to remove it."""
        self._mask_cb = callback   # the engine stores the raw pointer: keep the ctypes object alive with the engine
        fn = C.cast(callback, C.c_void_p) if callback is not None else None
        if self.lib.tgis_engine_set_mask_provider(self._h, fn, None) != 0:
            raise EngineError(_lib.last_error(self.lib))

    def poll(self, timeout_ms: int = 0) -> list[StepOutput]:
        n = self.lib.tgis_engine_poll(self._h, self._poll_buf, len(self._poll_buf), timeout_ms)
        if n < 0:
            raise EngineError(_lib.last_error(self.lib))
        outs = []
        for i in range(n):
            o = self._poll_buf[i]
            outs.append(StepOutput(
                request_id=o.request_id.decode(), new_token=o.token_id if o.n_new_tokens else None,
                logprob=o.logprob, rank=o.rank,
                topn=[(o.topn_ids[j], o.topn_logprobs[j]) for j in range(o.n_topn)],
                finish_reason=o.finish_reason, stop_token_id=o.stop_token_id, n_prompt_tokens=o.n_prompt_tokens,
                n_output_tokens=o.n_output_tokens, ts_arrival=o.ts_arrival, ts_first_scheduled=o.ts_first_scheduled,
                ts_first_token=o.ts_first_token, ts_last_token=o.ts_last_token, prompt_pos=o.prompt_pos, token_id=o.token_id))
        return outs

    def run_until_idle(self) -> int:
        n = self.lib.tgis_engine_run_until_idle(self._h)
        if n < 0:
            raise EngineError(f"run_until_idle failed: {_lib.last_error(self.lib)}")
        return n

    def status(self) -> TgisStatus:
        st = TgisStatus()
        self.lib.tgis_engine_status(self._h, C.byref(st))
        return st

    def prefix_cache_stats(self) -> tuple[int, int, int]:
        """(tokens looked up in the prefix cache, tokens found there, keyed blocks now); all 0 with caching off."""
        q, h, n = C.c_int64(0), C.c_int64(0), C.c_int32(0)
        if self.lib.tgis_engine_prefix_cache_stats(self._h, C.byref(q), C.byref(h), C.byref(n)) != 0:
            raise EngineError(_lib.last_error(self.lib))
        return q.value, h.value, n.value

    @staticmethod
    def nccl_unique_id() -> bytes:
        import torch  # noqa: F401  (torch's bundled libnccl.so.2 must be the copy in the process: see csrc/engine.cu)

        buf = (C.c_uint8 * 128)()
        lib = _lib.load_library()
        if lib.tgis_nccl_unique_id(C.byref(buf)) != 0:
            raise EngineError(_lib.last_error(lib))
        return bytes(buf)

    def worker_run(self) -> None:
        """Tensor-parallel ranks > 0: execute rank 0's step plans until it shuts down (blocking)."""
        if self.lib.tgis_engine_worker_run(self._h) != 0:
            raise EngineError(f"worker_run failed: {_lib.last_error(self.lib)}")

    def set_profiling(self, on: bool | int) -> None:
        """True/1: time every GEMM launch; 2: only those of pure-decode steps."""
        self.lib.tgis_engine_set_profiling(self._h, int(on))

    @property
    def max_model_len(self) -> int:
        return self.lib.tgis_engine_max_model_len(self._h)

    def close(self) -> None:
        if self._h:
            self.lib.tgis_engine_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):  # noqa: D105
        try:
            self.close()
        except Exception:  # noqa: BLE001
            pass

    # -- convenience for tests / bench --------------------------------------------------------------------------
    def generate_sync(self, prompts: list[list[int]], params: list[TgisSamplingParams] | TgisSamplingParams
                      ) -> list[list[StepOutput]]:
        """Submit all prompts, drive the step loop on this thread, return per-request output records."""
        if not isinstance(params, list):
            params = [params] * len(prompts)
        for i, (p, sp) in enumerate(zip(prompts, params)):
            self.add_request(f"r{i}", p, sp)
        self.run_until_idle()
        res: list[list[StepOutput]] = [[] for _ in prompts]
        while True:
            outs = self.poll(0)
            if not outs:
                break
            for o in outs:
                res[int(o.request_id[1:])].append(o)
        return res
