"""ctypes binding of libtgis_engine.so (C ABI: include/tgis_engine.h, include/tgis_kernels.h).

This is the reference-side binding a maintainer would add next to `build_async_engine_client`
(/root/reference/src/vllm_tgis_adapter/__main__.py:48); see INTEGRATION.md.  There is no Python/CPU fallback: if the
library is missing it is built with nvcc, and if that is impossible the import fails loudly.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

ABI_VERSION = 9
ARCH_LLAMA, ARCH_OPT, ARCH_GPT_BIGCODE = 0, 1, 2
MAX_REQUEST_ID = 96
MAX_TOPN = 12
MAX_STOP_TOKEN_IDS = 8

FINISH_NONE, FINISH_LENGTH, FINISH_STOP_EOS, FINISH_STOP_TOKEN, FINISH_ABORT, FINISH_ERROR = range(6)


class TgisConfig(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int32), ("n_layers", C.c_int32), ("hidden", C.c_int32), ("n_q_heads", C.c_int32),
        ("n_kv_heads", C.c_int32), ("head_dim", C.c_int32), ("ffn", C.c_int32), ("vocab", C.c_int32),
        ("rope_theta", C.c_float), ("rms_eps", C.c_float), ("max_model_len", C.c_int32),
        ("max_num_seqs", C.c_int32), ("max_batched_tokens", C.c_int32), ("kv_cache_bytes", C.c_int64),
        ("gpu_mem_fraction", C.c_float), ("device", C.c_int32), ("tp_size", C.c_int32), ("tp_rank", C.c_int32),
        ("use_cuda_graphs", C.c_int32), ("debug_gemm_ref", C.c_int32), ("seed", C.c_uint64),
        ("nccl_id", C.c_uint8 * 128), ("shm_name", C.c_char * 64),
        ("max_loras", C.c_int32), ("max_lora_rank", C.c_int32), ("arch", C.c_int32),
        ("embedding_multiplier", C.c_float), ("residual_multiplier", C.c_float), ("attention_multiplier", C.c_float),
        ("logit_scale", C.c_float), ("qk_norm", C.c_int32), ("qkv_bias", C.c_int32), ("sliding_window", C.c_int32),
        ("rope_table_from_host", C.c_int32), ("enable_prefix_caching", C.c_int32),
    ]


class TgisSamplingParams(C.Structure):
    _fields_ = [
        ("greedy", C.c_int32), ("temperature", C.c_float), ("top_k", C.c_int32), ("top_p", C.c_float),
        ("typical_p", C.c_float), ("repetition_penalty", C.c_float), ("has_length_penalty", C.c_int32),
        ("lp_start_index", C.c_uint32), ("lp_decay_factor", C.c_float), ("eos_token_id", C.c_int32),
        ("min_tokens", C.c_int32), ("max_tokens", C.c_int32), ("num_logprobs", C.c_int32),
        ("prompt_logprobs", C.c_int32), ("has_seed", C.c_int32), ("seed", C.c_uint64),
        ("n_stop_token_ids", C.c_int32), ("stop_token_ids", C.c_int32 * MAX_STOP_TOKEN_IDS),
        ("guided", C.c_int32), ("lora_slot", C.c_int32),
    ]


class TgisStepOutput(C.Structure):
    _fields_ = [
        ("request_id", C.c_char * MAX_REQUEST_ID), ("n_new_tokens", C.c_int32), ("token_id", C.c_int32),
        ("logprob", C.c_float), ("rank", C.c_int32), ("n_topn", C.c_int32), ("topn_ids", C.c_int32 * MAX_TOPN),
        ("topn_logprobs", C.c_float * MAX_TOPN), ("finish_reason", C.c_int32), ("stop_token_id", C.c_int32),
        ("n_prompt_tokens", C.c_int32), ("n_output_tokens", C.c_int32), ("ts_arrival", C.c_double),
        ("ts_first_scheduled", C.c_double), ("ts_first_token", C.c_double), ("ts_last_token", C.c_double),
        ("prompt_pos", C.c_int32), ("reserved", C.c_int32),
    ]


class TgisStatus(C.Structure):
    _fields_ = [
        ("errored", C.c_int32), ("is_running", C.c_int32), ("n_running", C.c_int32), ("n_waiting", C.c_int32),
        ("free_blocks", C.c_int32), ("total_blocks", C.c_int32), ("steps", C.c_int64),
        ("tokens_generated", C.c_int64), ("kernel_launches", C.c_int64), ("gpu_busy_ms", C.c_double),
        ("gpu_decode_ms", C.c_double), ("gpu_mixed_ms", C.c_double), ("decode_steps", C.c_int64),
        ("decode_tokens", C.c_int64), ("h2d_bytes", C.c_int64), ("d2h_bytes", C.c_int64), ("gemm_ms", C.c_double),
        ("gemm_bytes", C.c_double), ("gemm_calls", C.c_int64), ("graph_launches", C.c_int64),
        ("exchange_ms", C.c_double), ("exchange_calls", C.c_int64), ("preemptions", C.c_int64),
    ]


# Every symbol include/tgis_engine.h and include/tgis_kernels.h declare (tests/test_abi_cpu.py checks the export list)
ENGINE_SYMBOLS = [
    "tgis_last_error", "tgis_abi_version", "tgis_config_check", "tgis_engine_create", "tgis_engine_load_weight",
    "tgis_engine_prefix_cache_stats", "tgis_engine_start",
    "tgis_engine_add_request", "tgis_engine_abort", "tgis_engine_set_mask_provider", "tgis_engine_load_adapter_weight", "tgis_engine_clear_adapter", "tgis_engine_poll", "tgis_engine_status",
    "tgis_engine_max_model_len", "tgis_engine_set_profiling", "tgis_nccl_unique_id", "tgis_engine_worker_run", "tgis_engine_shutdown", "tgis_engine_destroy", "tgis_engine_run_until_idle",
]
KERNEL_SYMBOLS = [
    "tgis_k_last_error", "tgis_k_gemm_timeline", "tgis_k_step_timeline_enable", "tgis_k_step_timeline_read", "tgis_k_gemm", "tgis_k_rmsnorm", "tgis_k_rmsnorm_mult", "tgis_k_embed", "tgis_k_opt_layernorm", "tgis_k_opt_bias_act", "tgis_k_opt_embed", "tgis_k_silu_mul", "tgis_k_rope_kv", "tgis_k_gemm_rope", "tgis_k_attention", "tgis_k_attention_split", "tgis_k_attention_split_bench", "tgis_k_rope_attention",
    "tgis_k_attention_bench", "tgis_k_decode_items", "tgis_k_gemm_plan", "tgis_k_gemm_schedule", "tgis_k_gemm_chain", "tgis_k_gemm_blocks_per_sm",
    "tgis_k_sampler", "tgis_k_sampler_ex", "tgis_k_sampler_masked", "tgis_k_sampler_scaled", "tgis_k_lora", "tgis_k_lora_group", "tgis_k_lora_bench", "tgis_k_silu_mul_interleaved", "tgis_k_sizeof_sample_row", "tgis_k_sizeof_sample_out", "tgis_k_kv_block",
    "tgis_k_rope_kv_hd", "tgis_k_attention_hd", "tgis_k_attention_split_hd", "tgis_k_attention_bench_hd",
    "tgis_k_rope_kv_qknorm", "tgis_k_tp_area_bytes", "tgis_k_tp_exchange", "tgis_k_logits_push", "tgis_k_logits_wait",
    "tgis_k_gather_relayout", "tgis_k_tp_exchange_check", "tgis_k_logits_wait_check",
    "tgis_k_attention_window", "tgis_k_attention_bench_window", "tgis_k_decode_items_window",
    "tgis_k_rope_kv_bias",
]

_LIB: C.CDLL | None = None


def library_path() -> Path:
    override = os.environ.get("TGIS_ENGINE_LIB")   # experiments: an alternative build of the same sources
    if override:
        return Path(override)
    return Path(__file__).resolve().parent.parent / "lib" / "libtgis_engine.so"


def load_library() -> C.CDLL:
    """Load (building first if needed) the native engine.  Raises if neither is possible — no fallback."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = library_path()
    if not os.environ.get("TGIS_ENGINE_LIB"):
        # build() is a digest compare when the library is current; it rebuilds after ANY source/header edit, so tests
        # and benchmarks can never validate a stale .so.  Without nvcc (a deployment box) an existing library is used.
        from vllm_tgis_adapter_b200.csrc.build import build, have_nvcc

        if have_nvcc() or not path.exists():
            build(force=bool(os.environ.get("TGIS_FORCE_BUILD")))
    if not path.exists():
        raise RuntimeError(f"{path} is missing and could not be built: the TGIS engine has no fallback path")
    lib = C.CDLL(str(path))
    vp, i32, i64, f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_float
    lib.tgis_last_error.restype = C.c_char_p
    lib.tgis_k_last_error.restype = C.c_char_p
    lib.tgis_config_check.argtypes = [C.POINTER(TgisConfig)]
    lib.tgis_engine_create.argtypes = [C.POINTER(TgisConfig), C.POINTER(vp)]
    lib.tgis_engine_load_weight.argtypes = [vp, C.c_char_p, vp, i64, i64, i32]
    lib.tgis_engine_prefix_cache_stats.argtypes = [vp, C.POINTER(i64), C.POINTER(i64), C.POINTER(i32)]
    lib.tgis_engine_start.argtypes = [vp]
    lib.tgis_engine_add_request.argtypes = [vp, C.c_char_p, C.POINTER(i32), i32, C.POINTER(TgisSamplingParams)]
    lib.tgis_engine_abort.argtypes = [vp, C.c_char_p]
    lib.tgis_engine_set_mask_provider.argtypes = [vp, vp, vp]
    lib.tgis_engine_load_adapter_weight.argtypes = [vp, i32, C.c_char_p, vp, i64, i64]
    lib.tgis_engine_clear_adapter.argtypes = [vp, i32]
    lib.tgis_engine_poll.argtypes = [vp, C.POINTER(TgisStepOutput), i32, i32]
    lib.tgis_engine_status.argtypes = [vp, C.POINTER(TgisStatus)]
    lib.tgis_engine_max_model_len.argtypes = [vp]
    lib.tgis_engine_set_profiling.argtypes = [vp, i32]
    lib.tgis_nccl_unique_id.argtypes = [C.POINTER(C.c_uint8 * 128)]
    lib.tgis_engine_worker_run.argtypes = [vp]
    lib.tgis_engine_shutdown.argtypes = [vp]
    lib.tgis_engine_destroy.argtypes = [vp]
    lib.tgis_engine_destroy.restype = None
    lib.tgis_engine_run_until_idle.argtypes = [vp]
    lib.tgis_k_gemm.argtypes = [vp, vp, vp, i32, i32, i32, i32, i32, i32, C.POINTER(f32), i32]
    lib.tgis_k_gemm_schedule.argtypes = [i32, i32, i32, i32, C.POINTER(i32), C.POINTER(i32), i32, C.POINTER(i32), C.POINTER(i32), i32, C.POINTER(i32),
                                         C.POINTER(i32), i32, C.POINTER(i32)]
    lib.tgis_k_gemm_chain.argtypes = [i32, C.POINTER(i32), C.POINTER(C.c_uint64), C.POINTER(i32)]
    lib.tgis_k_rmsnorm.argtypes = [vp, vp, vp, vp, i32, i32, f32]
    lib.tgis_k_rmsnorm_mult.argtypes = [vp, vp, vp, vp, i32, i32, f32, f32]
    lib.tgis_k_embed.argtypes = [vp, vp, vp, i32, i32, i32, f32]
    lib.tgis_k_silu_mul.argtypes = [vp, vp, i32, i32]
    lib.tgis_k_opt_layernorm.argtypes = [vp, vp, vp, vp, vp, vp, i32, i32, f32]
    lib.tgis_k_opt_bias_act.argtypes = [vp, vp, vp, i32, i32, i32]
    lib.tgis_k_opt_embed.argtypes = [vp, vp, vp, vp, vp, i32, i32, i32, i32, i32]
    lib.tgis_k_rope_kv.argtypes = [vp, C.POINTER(i32), C.POINTER(i32), vp, vp, vp, i32, i32, i32]
    lib.tgis_k_attention.argtypes = [vp, vp, vp, C.POINTER(i32), i32, C.POINTER(i32), i32, i32, vp, i32, i32, f32]
    lib.tgis_k_attention_split.argtypes = [vp, vp, vp, C.POINTER(i32), i32, C.POINTER(i32), i32, i32, vp, i32, i32, f32,
                                           i32]
    lib.tgis_k_attention_split_bench.argtypes = [vp, vp, vp, C.POINTER(i32), i32, C.POINTER(i32), i32, i32, vp, i32,
                                                 i32, f32, i32, i32, C.POINTER(f32)]
    lib.tgis_k_rope_kv_hd.argtypes = [i32, vp, C.POINTER(i32), C.POINTER(i32), vp, vp, vp, i32, i32, i32]
    lib.tgis_k_rope_kv_qknorm.argtypes = [vp, C.POINTER(i32), C.POINTER(i32), vp, vp, vp, i32, i32, i32, vp, vp, f32, i32,
                                          C.POINTER(f32)]
    lib.tgis_k_rope_kv_bias.argtypes = [i32, vp, vp, vp, C.POINTER(i32), C.POINTER(i32), vp, vp, vp, i32, i32, i32, i32,
                                        C.POINTER(f32)]
    lib.tgis_k_attention_hd.argtypes = [i32, vp, vp, vp, C.POINTER(i32), i32, C.POINTER(i32), i32, i32, vp, i32, i32, f32]
    lib.tgis_k_attention_split_hd.argtypes = [i32, vp, vp, vp, C.POINTER(i32), i32, C.POINTER(i32), i32, i32, vp, i32, i32,
                                              f32, i32]
    lib.tgis_k_attention_bench_hd.argtypes = [i32, vp, vp, vp, C.POINTER(i32), i32, C.POINTER(i32), i32, i32, vp, i32, i32,
                                              f32, i32, i64, i32, C.POINTER(f32)]
    lib.tgis_k_attention_window.argtypes = [i32, vp, vp, vp, C.POINTER(i32), i32, C.POINTER(i32), i32, i32, vp, i32,
                                            i32, f32, i32, i32]
    lib.tgis_k_attention_bench_window.argtypes = [i32, vp, vp, vp, C.POINTER(i32), i32, C.POINTER(i32), i32, i32, vp,
                                                  i32, i32, f32, i32, i64, i32, C.POINTER(f32), i32]
    lib.tgis_k_decode_items_window.argtypes = [C.POINTER(i32), i32, C.POINTER(i32), i32, C.POINTER(i32), i32, i32]
    lib.tgis_k_rope_attention.argtypes = [i32, vp, vp, i32, i32, vp, C.POINTER(i32), C.POINTER(i32), vp, vp, vp,
                                          C.POINTER(i32), i32, C.POINTER(i32), i32, i32, vp, i32, i32, f32]
    lib.tgis_k_sampler.argtypes = [vp, i32, i32, vp, i32, vp, vp]
    lib.tgis_k_sampler_ex.argtypes = [vp, i32, i32, i32, vp, i32, vp, vp, i32, C.POINTER(f32)]
    lib.tgis_k_lora.argtypes = [vp, i32, vp, vp, vp, i32, i32, i32, i32, vp, i32, i32]
    lib.tgis_k_lora_group.argtypes = [vp, i32, vp, vp, i32, C.POINTER(vp), C.POINTER(vp), C.POINTER(i32), i32, vp, i32, i32]
    lib.tgis_k_silu_mul_interleaved.argtypes = [vp, vp, i32, i32]
    lib.tgis_k_lora_bench.argtypes = [vp, i32, vp, vp, vp, i32, i32, i32, vp, i32, i32, i32, C.POINTER(f32), C.POINTER(f32)]
    lib.tgis_k_sampler_masked.argtypes = [vp, i32, i32, i32, vp, i32, vp, vp, vp, i32, C.POINTER(f32)]
    lib.tgis_k_sampler_scaled.argtypes = [vp, i32, i32, i32, vp, i32, vp, vp, vp, f32]
    u32 = C.c_uint32
    lib.tgis_k_tp_area_bytes.argtypes = [i32, i32, C.POINTER(i64)]
    lib.tgis_k_tp_exchange.argtypes = [i32, i32, i32, vp, C.POINTER(C.c_uint64), vp, vp, vp, i32, i32, f32, u32, u32]
    lib.tgis_k_logits_push.argtypes = [vp, vp, i32, i32, i32, i32, vp, vp, u32, u32]
    lib.tgis_k_logits_wait.argtypes = [vp, i32, u32, u32]
    lib.tgis_k_tp_exchange_check.argtypes = [i32, i32, i32, C.POINTER(C.c_uint64), i32, i32, u32, u32]
    lib.tgis_k_logits_wait_check.argtypes = [vp, i32, u32, u32]
    lib.tgis_k_gather_relayout.argtypes = [vp, vp, i32, i32, i32]
    _LIB = lib
    return lib


def last_error(lib: C.CDLL) -> str:
    return (lib.tgis_last_error() or b"").decode(errors="replace")
