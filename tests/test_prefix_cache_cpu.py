"""Automatic prefix caching, the parts that need no GPU: the vLLM flag pair, the Prometheus counters, and the two C ABI
calls (exported, null-safe, and additive: the ABI version and the struct sizes are unchanged)."""
import ctypes as C
import types

from vllm_tgis_adapter_b200.engine import _lib


def test_flag_parses_both_ways_and_defaults_off(monkeypatch):
    from vllm_tgis_adapter_b200.tgis_utils.args import parse_args

    monkeypatch.delenv("ENABLE_PREFIX_CACHING", raising=False)
    assert parse_args(["--model", "tiny"]).enable_prefix_caching is False
    assert parse_args(["--model", "tiny", "--enable-prefix-caching"]).enable_prefix_caching is True
    assert parse_args(["--model", "tiny", "--no-enable-prefix-caching"]).enable_prefix_caching is False
    assert parse_args(["--model", "tiny", "--enable-prefix-caching", "--no-enable-prefix-caching"]
                      ).enable_prefix_caching is False


def test_loader_threads_the_flag_into_the_engine(monkeypatch):
    from vllm_tgis_adapter_b200.engine import loader

    seen = {}

    class FakeNative:
        def __init__(self, mc, **kw):
            seen.update(kw)

        def load_weight(self, *a):
            pass

    monkeypatch.setattr(loader, "NativeEngine", FakeNative)
    monkeypatch.setattr(loader, "load_synthetic_weights", lambda *a: None)
    monkeypatch.setattr(loader, "rope_cos_sin", lambda mc: None)
    args = types.SimpleNamespace(max_num_seqs=4, max_num_batched_tokens=64, gpu_memory_utilization=0.5, seed=0,
                                 enable_lora=False, max_loras=0, max_lora_rank=16, enable_prefix_caching=True)
    mc = types.SimpleNamespace(arch="llama")
    loader._make_native_engine(args, mc, None, 0)
    assert seen["enable_prefix_caching"] is True
    args.enable_prefix_caching = False
    loader._make_native_engine(args, mc, None, 0)
    assert seen["enable_prefix_caching"] is False


def _status():
    return types.SimpleNamespace(n_running=0, n_waiting=0, free_blocks=10, total_blocks=10, steps=0,
                                 kernel_launches=0, gpu_busy_ms=0.0)


def _sample(text: str, name: str) -> float:
    for line in text.splitlines():
        if line.startswith(name + "{"):
            return float(line.rsplit(" ", 1)[1])
    raise AssertionError(f"{name} not in the exposition")


def test_metrics_render_prefix_cache_counters_from_engine_stats():
    from vllm_tgis_adapter_b200.metrics import EngineMetrics

    m = EngineMetrics("m")
    text = m.render(_status(), (0, 0)).decode()
    assert _sample(text, "vllm:prefix_cache_queries_total") == 0
    assert _sample(text, "vllm:prefix_cache_hits_total") == 0
    text = m.render(_status(), (1000, 768)).decode()
    assert _sample(text, "vllm:prefix_cache_queries_total") == 1000
    assert _sample(text, "vllm:prefix_cache_hits_total") == 768
    # the engine counters are cumulative: each scrape adds the increase since the previous one
    text = m.render(_status(), (1500, 768)).decode()
    assert _sample(text, "vllm:prefix_cache_queries_total") == 1500
    assert _sample(text, "vllm:prefix_cache_hits_total") == 768
    text = m.render(None).decode()   # engine gone: the counters keep their values
    assert _sample(text, "vllm:prefix_cache_queries_total") == 1500


def test_http_metrics_reads_the_stats_call():
    from vllm_tgis_adapter_b200 import http
    from vllm_tgis_adapter_b200.metrics import EngineMetrics

    class Native:
        def status(self):
            return _status()

        def prefix_cache_stats(self):
            return 640, 512, 16

    eng = types.SimpleNamespace(engine=Native(), metrics=EngineMetrics("m"))
    text = http._metrics(eng).decode()
    assert _sample(text, "vllm:prefix_cache_queries_total") == 640
    assert _sample(text, "vllm:prefix_cache_hits_total") == 512


def test_new_symbols_exported_and_null_safe():
    lib = _lib.load_library()
    for name in ("tgis_engine_prefix_cache_stats", "tgis_k_attention_split", "tgis_k_attention_split_bench"):
        assert hasattr(lib, name), name
    # prefix caching is a tgis_config field (ABI v9), not a call of its own
    assert "enable_prefix_caching" in [f for f, _ in _lib.TgisConfig._fields_]
    q, h, n = C.c_int64(-1), C.c_int64(-1), C.c_int32(-1)
    assert lib.tgis_engine_prefix_cache_stats(None, C.byref(q), C.byref(h), C.byref(n)) != 0
    assert "null" in _lib.last_error(lib)
    assert lib.tgis_k_attention_split(None, None, None, None, 0, None, 0, 0, None, 8, 2, 1.0, 3) != 0


def test_abi_version_and_struct_sizes_unchanged():
    lib = _lib.load_library()
    assert _lib.ABI_VERSION == 9 and lib.tgis_abi_version() == 9
    assert C.sizeof(_lib.TgisConfig) == 336
    assert C.sizeof(_lib.TgisStatus) == 4 * 6 + 8 * 17
