"""Request-level Prometheus metrics under vLLM's metric names, so dashboards built for the reference's /metrics keep
working (the reference re-exports vLLM's registry: /root/reference/src/vllm_tgis_adapter/http.py:41-99; names from
vllm v1/metrics/loggers.py `PrometheusStatLogger`).  Engine-level gauges are read from `tgis_engine_status` at scrape
time; the histograms are fed by AsyncTGISEngine when a request finishes, from the engine's own timestamps."""
from __future__ import annotations

from prometheus_client import CollectorRegistry, Counter, Gauge, Histogram, generate_latest

_LAT = (0.001, 0.005, 0.01, 0.02, 0.04, 0.06, 0.08, 0.1, 0.25, 0.5, 0.75, 1.0, 2.5, 5.0, 7.5, 10.0, 20.0, 40.0, 80.0)
_TPOT = (0.0025, 0.005, 0.0075, 0.01, 0.015, 0.02, 0.025, 0.03, 0.04, 0.05, 0.075, 0.1, 0.15, 0.2, 0.3, 0.4, 0.5, 0.75,
         1.0, 2.5)
_TOK = (1, 2, 5, 10, 20, 50, 100, 200, 500, 1000, 2000, 5000, 10000)


class EngineMetrics:
    def __init__(self, model_name: str = ""):
        self.registry = CollectorRegistry()
        lab, self._lv = ["model_name"], [model_name]

        def gauge(name, doc):
            return Gauge(name, doc, lab, registry=self.registry).labels(*self._lv)

        def hist(name, doc, buckets):
            return Histogram(name, doc, lab, buckets=buckets, registry=self.registry).labels(*self._lv)

        self.running = gauge("vllm:num_requests_running", "Number of requests in model execution batches.")
        self.waiting = gauge("vllm:num_requests_waiting", "Number of requests waiting to be processed.")
        self.kv_usage = gauge("vllm:kv_cache_usage_perc", "KV-cache usage. 1 means 100 percent usage.")
        self.gpu_cache_usage = gauge("vllm:gpu_cache_usage_perc", "GPU KV-cache usage (pre-V1 name).")
        self.prompt_tokens = Counter("vllm:prompt_tokens", "Number of prefill tokens processed.", lab,
                                     registry=self.registry).labels(*self._lv)
        self.generation_tokens = Counter("vllm:generation_tokens", "Number of generation tokens processed.", lab,
                                         registry=self.registry).labels(*self._lv)
        self._success = Counter("vllm:request_success", "Count of successfully processed requests.",
                                [*lab, "finished_reason"], registry=self.registry)
        self.ttft = hist("vllm:time_to_first_token_seconds", "Histogram of time to first token in seconds.", _LAT)
        self.tpot = hist("vllm:time_per_output_token_seconds", "Histogram of time per output token in seconds.", _TPOT)
        self.e2e = hist("vllm:e2e_request_latency_seconds", "Histogram of e2e request latency in seconds.", _LAT)
        self.queue_time = hist("vllm:request_queue_time_seconds", "Histogram of time spent in WAITING phase.", _LAT)
        self.req_prompt = hist("vllm:request_prompt_tokens", "Number of prefill tokens processed per request.", _TOK)
        self.req_gen = hist("vllm:request_generation_tokens", "Number of generation tokens processed per request.", _TOK)
        # prefix caching, in tokens (vLLM V1's names); fed at scrape time with the increase of the engine's counters.
        # As in vLLM, a request counts once: the recompute of a preempted request is not queried again.
        self.prefix_cache_queries = Counter(
            "vllm:prefix_cache_queries", "Prefix cache queries, in terms of number of queried tokens.", lab,
            registry=self.registry).labels(*self._lv)
        self.prefix_cache_hits = Counter(
            "vllm:prefix_cache_hits", "Prefix cache hits, in terms of number of cached tokens.", lab,
            registry=self.registry).labels(*self._lv)
        self._pc_seen = (0, 0)
        self.steps = gauge("tgis_engine_steps", "Engine steps executed.")
        self.launches = gauge("tgis_engine_kernel_launches", "CUDA kernels launched by the engine.")
        self.gpu_busy = gauge("tgis_engine_gpu_busy_seconds", "Device time spent in engine steps.")

    def observe_finished(self, *, n_prompt: int, n_generated: int, finish_reason: str | None, arrival: float,
                         first_scheduled: float, first_token: float, last_token: float) -> None:
        """One finished request; timestamps are the engine's (seconds on one monotonic clock, 0 = not reached)."""
        self.prompt_tokens.inc(n_prompt)
        self.generation_tokens.inc(n_generated)
        self.req_prompt.observe(n_prompt)
        self.req_gen.observe(n_generated)
        self._success.labels(*self._lv, finish_reason or "abort").inc()
        if first_scheduled and arrival:
            self.queue_time.observe(max(0.0, first_scheduled - arrival))
        if first_token and arrival:
            self.ttft.observe(max(0.0, first_token - arrival))
        if last_token and arrival:
            self.e2e.observe(max(0.0, last_token - arrival))
        if n_generated > 1 and last_token and first_token:
            self.tpot.observe(max(0.0, (last_token - first_token) / (n_generated - 1)))

    def render(self, status, prefix_cache: tuple[int, int] | None = None) -> bytes:
        """status: the engine's tgis_status (or None when the engine cannot be queried any more); prefix_cache: the
        engine's cumulative (queried tokens, hit tokens), or None."""
        if prefix_cache is not None:
            q, h = int(prefix_cache[0]), int(prefix_cache[1])
            self.prefix_cache_queries.inc(max(0, q - self._pc_seen[0]))
            self.prefix_cache_hits.inc(max(0, h - self._pc_seen[1]))
            self._pc_seen = (max(q, self._pc_seen[0]), max(h, self._pc_seen[1]))
        if status is not None:
            self.running.set(status.n_running)
            self.waiting.set(status.n_waiting)
            usage = 1.0 - status.free_blocks / max(status.total_blocks, 1)
            self.kv_usage.set(usage)
            self.gpu_cache_usage.set(usage)
            self.steps.set(status.steps)
            self.launches.set(status.kernel_launches)
            self.gpu_busy.set(status.gpu_busy_ms / 1e3)
        return generate_latest(self.registry)
